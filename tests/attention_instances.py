"""The cases of tests/test_gpu_attention_elementwise.py and the template instances of the attention kernels they reach.

No torch import, so the CPU test of the built library (test_attention_instances.py) can check that the instances the
compiler emitted are exactly the keys of INSTANCES: a new instance without a per-element GPU case fails there.

Each forward / backward case is one packed batch run through attn_varlen_fwd and attn_varlen_bwd; it reaches
attn_fwd_kernel, attn_bwd_kernel (dK / dV) and attn_dq_kernel at its (head_dim, ALiBi) and attn_delta_kernel.  Each decode
case is one attn_decode call.
"""

HEAD_DIMS = (16, 32, 64, 80, 96, 128)

# (n_groups, q_per_group): MHA with 5 and 16 heads, GQA with g = 2, 3, 4, 5, MQA with 16 and 7 heads.  Cycled over the
# grid so that (1, 16) and (16, 1) -- 16 heads, first ALiBi slope 2^-0.5 -- fall on ALiBi cases.
HEAD_CONFIGS = [(5, 1), (3, 2), (2, 3), (1, 16), (3, 4), (2, 5), (16, 1), (1, 7)]
SCALES = ("rsqrt", "mup")  # 1 / sqrt(head_dim), 1 / head_dim (the muP attention multiplier)
DISTS = ("normal", "peaked", "flat")

# document lengths on both sides of the 64-row backward step and the 128-row tile, one of ~600; the order rotates per case
# and empty documents stand at the start, in the middle and at the end
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
                name = f"hd{hd}-{'alibi' if alibi else 'plain'}-p{dropout}-{ng}x{g}-{scale}-{dist}"
                cases[name] = dict(hd=hd, alibi=alibi, dropout=dropout, ng=ng, g=g, scale=scale, dist=dist,
                                   lens=ragged_lens(i), seed=100 + i)
                i += 1
    return cases


def _long_cases() -> dict:
    """one document of 2150 tokens (16 full 128-key tiles and one of 102) between short ones: the forward's 2-stage K/V
    ring, the dK/dV Q/dO ring and the dQ K/V ring wrap many times.  "late": the keys of the last 128-key tile are shifted
    along the mean query direction, so the rows of the last tile find their maximum logit in their last key tile."""
    cases = {}
    grid = [(64, False, 2, 2, "rsqrt"), (64, True, 1, 16, "mup"), (80, False, 4, 1, "mup"), (80, True, 2, 3, "rsqrt"),
            (128, False, 1, 5, "rsqrt"), (128, True, 16, 1, "mup")]
    for i, (hd, alibi, ng, g, scale) in enumerate(grid):
        name = f"long-hd{hd}-{'alibi' if alibi else 'plain'}-{ng}x{g}-{scale}"
        cases[name] = dict(hd=hd, alibi=alibi, dropout=0.0, ng=ng, g=g, scale=scale, dist="late", lens=[3, 2150, 0, 130],
                           seed=200 + i)
    return cases


FWD_BWD_CASES = {**_ragged_cases(), **_long_cases()}

DECODE_LENS = [1, 127, 128, 129, 255, 256, 257, 700]  # L_max = 700 is not a multiple of the 128-key chunk


def _decode_cases() -> dict:
    cases = {}
    i = 0
    for hd in HEAD_DIMS:
        for alibi in (False, True):
            ng, g = HEAD_CONFIGS[i % len(HEAD_CONFIGS)]
            scale = SCALES[(i + i // 2) % 2]
            cases[f"decode-hd{hd}-{'alibi' if alibi else 'plain'}-{ng}x{g}-{scale}"] = dict(
                hd=hd, alibi=alibi, ng=ng, g=g, scale=scale, lens=DECODE_LENS, seed=300 + i)
            i += 1
    return cases


DECODE_CASES = _decode_cases()


def _instances() -> dict:
    inst: dict = {}
    for name, c in FWD_BWD_CASES.items():
        a = int(c["alibi"])
        for fam in ("attn_fwd_kernel", "attn_bwd_kernel", "attn_dq_kernel"):
            inst.setdefault(f"{fam}<{c['hd']}, {a}>", []).append(name)
        inst.setdefault("attn_delta_kernel", []).append(name)
    for name, c in DECODE_CASES.items():
        inst.setdefault(f"attn_decode_kernel<{c['hd']}, {int(c['alibi'])}>", []).append(name)
    return inst


# instance -> the per-element cases that run it
INSTANCES = _instances()
