"""The cases of tests/test_gpu_attention_wide.py and the template instances of the wide-head attention kernels
(csrc/attention_wide.cu) they reach.

No torch import, so the CPU test of the built library (test_attention_wide_instances.py) can check that the wide instances
the compiler emitted are exactly the keys of INSTANCES.

Each forward / backward case is one packed batch run through attn_varlen_fwd and attn_varlen_bwd; it reaches
attn_wide_fwd_kernel, attn_wide_bwd_kernel (dK / dV) and attn_wide_dq_kernel at its (head_dim, ALiBi).  Each decode case is
one attn_decode call and reaches attn_wide_decode_kernel.
"""

HEAD_DIMS = (160, 192, 256)

# (n_groups, q_per_group): MHA with 5 and 16 heads, GQA with g = 2, 3, 4, 5, MQA with 16 and 7 heads.  Cycled over the
# grid so that MQA with 16 heads falls on an ALiBi case.
HEAD_CONFIGS = [(5, 1), (3, 2), (2, 3), (1, 16), (3, 4), (2, 5), (16, 1), (1, 7)]
SCALES = ("rsqrt", "mup")  # 1 / sqrt(head_dim), 1 / head_dim
DISTS = ("normal", "peaked", "flat")

# document lengths on both sides of the 64-row tiles and halves and of the 128-row tiles, one of ~600; the order rotates
# per case and empty documents stand at the start, in the middle and at the end
RAGGED_LENGTHS = [1, 63, 64, 65, 127, 128, 129, 255, 257, 601]
DROPOUT_P = 0.15


def ragged_lens(i: int) -> list[int]:
    r = i % len(RAGGED_LENGTHS)
    rot = RAGGED_LENGTHS[r:] + RAGGED_LENGTHS[:r]
    return [0] + rot[:5] + [0] + rot[5:] + [0]


def _ragged_cases() -> dict:
    cases = {}
    i = 0
    for hd in HEAD_DIMS:
        for alibi in (False, True):
            for dropout in (0.0, DROPOUT_P):
                ng, g = HEAD_CONFIGS[i % len(HEAD_CONFIGS)]
                scale, dist = SCALES[(i + i // 4) % 2], DISTS[i % 3]
                name = f"wide-hd{hd}-{'alibi' if alibi else 'plain'}-p{dropout}-{ng}x{g}-{scale}-{dist}"
                cases[name] = dict(hd=hd, alibi=alibi, dropout=dropout, ng=ng, g=g, scale=scale, dist=dist,
                                   lens=ragged_lens(i), seed=500 + i)
                i += 1
    return cases


def _long_cases() -> dict:
    """one document of 2150 tokens between short ones per head_dim: the forward's and dQ's 64-key K / V rings and the
    dK / dV kernel's Q / dO ring wrap many times.  "late": the keys of the last 128-key tile are shifted along the mean
    query direction, so the rows of the last tile find their maximum logit in their last key tiles."""
    cases = {}
    grid = [(160, False, 2, 2, "rsqrt"), (192, True, 2, 3, "mup"), (256, False, 1, 4, "rsqrt")]
    for i, (hd, alibi, ng, g, scale) in enumerate(grid):
        name = f"wide-long-hd{hd}-{'alibi' if alibi else 'plain'}-{ng}x{g}-{scale}"
        cases[name] = dict(hd=hd, alibi=alibi, dropout=0.0, ng=ng, g=g, scale=scale, dist="late", lens=[3, 2150, 0, 130],
                           seed=600 + i)
    return cases


FWD_BWD_CASES = {**_ragged_cases(), **_long_cases()}

DECODE_LENS = [1, 127, 128, 129, 255, 256, 257, 700]  # on both sides of the 256-key chunk; L_max = 700 is not a multiple


def _decode_cases() -> dict:
    cases = {}
    i = 0
    for hd in HEAD_DIMS:
        for alibi in (False, True):
            ng, g = HEAD_CONFIGS[(i + 1) % len(HEAD_CONFIGS)]
            scale = SCALES[(i + i // 2) % 2]
            cases[f"wide-decode-hd{hd}-{'alibi' if alibi else 'plain'}-{ng}x{g}-{scale}"] = dict(
                hd=hd, alibi=alibi, ng=ng, g=g, scale=scale, lens=DECODE_LENS, seed=700 + i)
            i += 1
    return cases


DECODE_CASES = _decode_cases()


def _instances() -> dict:
    inst: dict = {}
    for name, c in FWD_BWD_CASES.items():
        a = int(c["alibi"])
        for fam in ("attn_wide_fwd_kernel", "attn_wide_bwd_kernel", "attn_wide_dq_kernel"):
            inst.setdefault(f"{fam}<{c['hd']}, {a}>", []).append(name)
    for name, c in DECODE_CASES.items():
        inst.setdefault(f"attn_wide_decode_kernel<{c['hd']}, {int(c['alibi'])}>", []).append(name)
    return inst


# instance -> the per-element cases that run it
INSTANCES = _instances()
