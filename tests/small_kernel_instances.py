"""Which template instance of the norm and RoPE kernels a call runs: a Python statement of the host-side choice in
csrc/elementwise.cu, and one shape per instance that reaches it.  No torch import, so the CPU test of the built library
(test_small_kernel_instances.py) can check the table against the instances the compiler emitted."""

KTHREADS = 256  # kThreads of elementwise.cu


def _block_nv(H: int) -> int:
    """vectors per thread of the block-per-row kernels (1, 2, 3 -> 4, >4 -> 8)"""
    nv = (H // 8 + KTHREADS - 1) // KTHREADS
    return nv if nv <= 2 else (4 if nv <= 4 else 8)


def rmsnorm_fwd_instance(T: int, H: int) -> str:
    H8 = H // 8
    if H8 <= 16 * 32 and T >= 64:  # one warp per row
        nvw = (H8 + 31) // 32
        return f"rmsnorm_fwd_warp_kernel<{4 if nvw <= 4 else 8 if nvw <= 8 else 10 if nvw <= 10 else 16}>"
    return f"rmsnorm_fwd_kernel<{_block_nv(H)}>"


def rmsnorm_bwd_instance(T: int, H: int) -> str:
    return f"rmsnorm_bwd_kernel<{_block_nv(H)}>"


def layernorm_fwd_instance(T: int, H: int) -> str:
    return f"layernorm_fwd_kernel<{_block_nv(H)}>"


def layernorm_bwd_instance(T: int, H: int) -> str:
    return f"layernorm_bwd_kernel<{_block_nv(H)}>"


def rope_threads(n_groups: int, q_per_group: int, head_dim: int) -> int:
    items = n_groups * (q_per_group + 1) * (head_dim // 16)
    return 1024 if items >= 1024 else (items + 31) // 32 * 32


def rope_instance(n_groups: int, q_per_group: int, head_dim: int, pos_dtype: str) -> str:
    max_threads = 512 if rope_threads(n_groups, q_per_group, head_dim) <= 512 else 1024
    return f"rope_kernel<{pos_dtype}, {max_threads}>"


# instance -> arguments of its family's choice rule: (T, H) for the norms, (n_groups, q_per_group, head_dim, position id
# type) for RoPE.  RMSNorm forward: the warp kernels need T >= 64, and (63, 2048) / (37, 4096) are the block kernels at
# the hidden sizes of warp<8> / warp<16>.  Backward: T below and far above the number of row partials (6 per SM).
INSTANCES = {
    "rmsnorm_fwd_warp_kernel<4>": (128, 1024),
    "rmsnorm_fwd_warp_kernel<8>": (64, 2048),
    "rmsnorm_fwd_warp_kernel<10>": (200, 2560),
    "rmsnorm_fwd_warp_kernel<16>": (300, 4096),
    "rmsnorm_fwd_kernel<1>": (63, 2048),
    "rmsnorm_fwd_kernel<2>": (37, 4096),
    "rmsnorm_fwd_kernel<4>": (200, 8192),
    "rmsnorm_fwd_kernel<8>": (70, 16384),
    "rmsnorm_bwd_kernel<1>": (2000, 1024),
    "rmsnorm_bwd_kernel<2>": (3, 4096),
    "rmsnorm_bwd_kernel<4>": (1000, 6144),
    "rmsnorm_bwd_kernel<8>": (5, 16384),
    "layernorm_fwd_kernel<1>": (1, 64),
    "layernorm_fwd_kernel<2>": (100, 4096),
    "layernorm_fwd_kernel<4>": (37, 6144),
    "layernorm_fwd_kernel<8>": (9, 16384),
    "layernorm_bwd_kernel<1>": (2000, 768),
    "layernorm_bwd_kernel<2>": (5, 2560),
    "layernorm_bwd_kernel<4>": (1000, 8192),
    "layernorm_bwd_kernel<8>": (3, 12288),
    "rope_kernel<int32_t, 512>": (4, 1, 64, "int32_t"),
    "rope_kernel<int64_t, 512>": (2, 4, 128, "int64_t"),
    "rope_kernel<int32_t, 1024>": (40, 1, 128, "int32_t"),
    "rope_kernel<int64_t, 1024>": (8, 8, 256, "int64_t"),
}

CHOICE = {
    "rmsnorm_fwd_warp_kernel": rmsnorm_fwd_instance,
    "rmsnorm_fwd_kernel": rmsnorm_fwd_instance,
    "rmsnorm_bwd_kernel": rmsnorm_bwd_instance,
    "layernorm_fwd_kernel": layernorm_fwd_instance,
    "layernorm_bwd_kernel": layernorm_bwd_instance,
    "rope_kernel": rope_instance,
}


def family(name: str) -> str:
    return name.split("<")[0]


def chosen_instance(name: str) -> str:
    """the instance the host rule picks for INSTANCES[name]"""
    return CHOICE[family(name)](*INSTANCES[name])


def instances_of(fam: str) -> list[str]:
    return [n for n in INSTANCES if family(n) == fam]
