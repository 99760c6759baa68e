"""The cases of tests/test_gpu_attention_cache.py and the template instances of the KV-cache attention kernel
(csrc/attention_cache.cu) they reach.

No torch import, so the CPU test of the built library (test_attention_cache_instances.py) can check that the instances the
compiler emitted are exactly the keys of INSTANCES.

Each case is one attn_cache call on a batch of sequences that pairs every cached length of PASTS with a count of new
tokens from NEWS; it reaches attn_cache_kernel at its (head_dim, ALiBi).
"""

HEAD_DIMS = (16, 32, 64, 80, 96, 128, 160, 192, 256)

# (n_groups, q_per_group): MHA, GQA with g = 2, 3, 4, 5, MQA with 7 and 16 heads
HEAD_CONFIGS = [(4, 1), (3, 2), (2, 3), (2, 4), (2, 5), (1, 7), (1, 16)]
SCALES = ("rsqrt", "mup")  # 1 / sqrt(head_dim), 1 / head_dim
DISTS = ("normal", "peaked", "flat")

# cached lengths on both sides of the 64-key tiles, and one of several tiles; new-token counts from none and one (a
# decode step) to more than two 64-row tiles of a CTA
PASTS = (0, 1, 63, 64, 65, 127, 128, 129, 700)
NEWS = (0, 1, 2, 17, 64, 65, 130)


def batch(i: int) -> tuple[list[int], list[int]]:
    """(past, n) per sequence of case i: every past once, the new-token counts rotated so that each appears"""
    return list(PASTS), [NEWS[(k + i) % len(NEWS)] for k in range(len(PASTS))]


def _cases() -> dict:
    cases = {}
    i = 0
    for hd in HEAD_DIMS:
        for alibi in (False, True):
            ng, g = HEAD_CONFIGS[i % len(HEAD_CONFIGS)]
            scale, dist = SCALES[(i + i // 4) % 2], DISTS[i % 3]
            past, n = batch(i)
            name = f"cache-hd{hd}-{'alibi' if alibi else 'plain'}-{ng}x{g}-{scale}-{dist}"
            cases[name] = dict(hd=hd, alibi=alibi, ng=ng, g=g, scale=scale, dist=dist, past=past, n=n, seed=900 + i)
            i += 1
    return cases


CASES = _cases()

# instance -> the per-element cases that run it
INSTANCES: dict = {}
for _name, _c in CASES.items():
    INSTANCES.setdefault(f"attn_cache_kernel<{_c['hd']}, {int(_c['alibi'])}>", []).append(_name)
