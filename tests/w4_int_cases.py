"""The exact-integer W4A16 kernels (kV3Variants x fused RMSNorm x v3_fusion in zhilight_b200/csrc/w4a16_gemm_v3.cu) and the
cases tests/test_w4_int_kernels_gpu.py runs them with.  tests/test_w4_int_kernels_cpu.py checks on the CPU, through the
planner of the built library, that the cases reach every kernel."""

import numpy as np

SMS = 132   # H100 SXM

# kV3Variants: (NT, warps per sub-CTA, sub-CTAs, ring stages, PACK)
SHAPES = [(1, 16, 1, 4, False), (1, 16, 1, 4, True), (1, 8, 2, 5, False), (1, 8, 2, 5, True), (1, 8, 2, 4, False),
          (1, 8, 2, 4, True), (2, 8, 2, 4, False)]
# v3_fusion: 0 plain, 1 act-order gather, 2 int8-KV epilogue, 3 reduce-in, 4 reduce-in + int8 KV, 5 push; the exchange
# fusions exist for the 4-stage shapes only
FUSIONS = ("plain", "gather", "kv8", "reduce_in", "reduce_in_kv8", "push")


def fusion(tp_mode, k_perm, kv8):
    if tp_mode:
        return 5 if tp_mode == 2 else 4 if kv8 else 3
    return 1 if k_perm else 2 if kv8 else 0


def kernels():
    """every compiled kernel: (shape index, NORM, fusion)"""
    return [(i, norm, f) for i, sh in enumerate(SHAPES) for norm in (0, 1) for f in range(6 if sh[3] == 4 else 3)]


def shape_of(plan_out):
    """index into SHAPES of a zl_w4_v3_plan result (nt, warps, subs, stages, rt, pack, ...)"""
    nt, warps, subs, stages, rt, pack = list(plan_out)[:6]
    assert rt == nt * 8
    return SHAPES.index((nt, warps, subs, stages, bool(pack)))


# (mc, N, K, epilogue, norm, fusion, sym, activations).  qkv cases use d = 128 heads, 8 kv heads and N / 128 - 16 q heads.
# Activations: rand (log-spread magnitudes), adv (power-of-two and (2 - 2^-10) 2^k maxima, all-zero, subnormal and flushed
# groups), headroom (one group of q = 15, z = 0 weights against activations all at the group maximum), nonfinite (NaN / Inf
# in two tokens).
CASES = [
    # <1,16,1,4> tall (N/32 <= SMs, K >= 4096), 5..7 tokens
    (5, 4096, 4096, "none", 0, 0, False, "adv"),
    (6, 4224, 4224, "res", 1, 0, True, "nonfinite"),     # G = 33: not a multiple of 16 warps
    (7, 4096, 4096, "swiglu", 1, 1, False, "rand"),
    (5, 4096, 4096, "qkv", 0, 2, False, "adv"),
    (7, 4096, 4096, "qkv", 1, 2, True, "rand"),
    (5, 2048, 5120, "none", 0, 1, False, "headroom"),
    # <1,16,1,4,PACK> tall, 1..4 tokens
    (1, 4096, 14336, "none", 1, 0, False, "adv"),
    (4, 4224, 4224, "res", 0, 0, True, "rand"),
    (2, 4096, 4096, "swiglu", 0, 1, False, "nonfinite"),
    (4, 4096, 4096, "qkv", 1, 2, False, "adv"),
    (1, 4096, 8192, "qkv", 0, 2, True, "rand"),
    (3, 4096, 6144, "none", 1, 1, False, "headroom"),
    # <1,8,2,5> wide, 5..8 tokens
    (8, 14336, 1536, "none", 0, 0, False, "rand"),       # 448 tiles over 264 sub-CTAs: both reduction buffers
    (5, 4256, 2432, "res", 1, 0, True, "adv"),           # N/32 = 133: one tile past the grid
    (8, 6144, 384, "swiglu", 1, 1, False, "rand"),       # G = 3 < 8 warps
    (6, 6144, 1024, "qkv", 0, 2, False, "adv"),
    (8, 4096, 128, "qkv", 1, 2, True, "rand"),           # G = 1
    (5, 4256, 1664, "none", 0, 1, False, "nonfinite"),
    # <1,8,2,5,PACK> wide, 1..4 tokens
    (1, 14336, 4096, "none", 0, 0, False, "adv"),
    (4, 4256, 384, "res", 1, 0, False, "headroom"),
    (2, 14336, 2048, "swiglu", 1, 1, True, "rand"),
    (3, 6144, 1024, "qkv", 0, 2, False, "rand"),
    (4, 6144, 128, "qkv", 1, 2, False, "adv"),
    (2, 4256, 1664, "none", 0, 1, True, "nonfinite"),
    # <1,8,2,4> wide, 5..8 tokens whose staged rows leave no room for 5 stages
    (8, 14336, 1664, "none", 0, 0, True, "rand"),        # G = 13
    (5, 4256, 5760, "res", 1, 0, False, "adv"),
    (8, 6144, 2048, "swiglu", 1, 1, False, "rand"),
    (6, 6144, 2560, "qkv", 0, 2, True, "rand"),
    (7, 6144, 3072, "qkv", 1, 2, False, "adv"),
    (5, 4256, 2560, "none", 0, 1, False, "headroom"),
    # <1,8,2,4,PACK>
    (4, 14336, 3200, "none", 0, 0, False, "adv"),        # G = 25
    (4, 4256, 4096, "res", 1, 0, True, "rand"),
    (3, 6144, 4352, "swiglu", 1, 1, False, "rand"),
    (4, 6144, 3584, "qkv", 0, 2, False, "rand"),
    (4, 6144, 4096, "qkv", 1, 2, True, "adv"),
    (4, 4256, 3200, "none", 0, 1, False, "nonfinite"),
    (1, 4256, 13312, "res", 0, 0, False, "rand"),        # one row leaves no room for 5 stages only at K > 12.5k
    # <2,8,2,4> 9..16 tokens
    (16, 14336, 1664, "none", 0, 0, False, "rand"),
    (9, 4256, 3072, "res", 1, 0, True, "adv"),
    (16, 6144, 384, "swiglu", 1, 1, False, "rand"),
    (12, 6144, 1024, "qkv", 0, 2, False, "adv"),
    (16, 4096, 1536, "qkv", 1, 2, True, "rand"),
    (9, 4256, 2048, "none", 0, 1, False, "nonfinite"),
    (16, 4256, 128, "none", 0, 0, False, "headroom"),
]

# exchange cases on a one-rank comm: (mc, N, K).  Each runs the push (NONE epilogue, N x K) and the reduce-in with the
# SWIGLU, QKV_ROPE and QKV_ROPE + int8-KV epilogues (N x K, N = (hq + 2 hkv) * 128), with and without the fused RMSNorm.
TP_CASES = [(5, 4096, 4096), (4, 4096, 4096), (8, 6144, 1024), (1, 6144, 1024), (16, 6144, 1024)]


def qkv_heads(n):
    """(q heads, kv heads, head size) of a qkv case of width n"""
    return n // 128 - 16, 8, 128


def weights(n, k, sym, headroom=False, seed=0):
    """q (N, K) nibbles, z (N, G) (8 when sym: the packer stores 8), s (N, G) fp16, in packed row order"""
    rng = np.random.default_rng(seed)
    q = rng.integers(0, 16, size=(n, k), dtype=np.uint8)
    z = np.full((n, k // 128), 8, np.uint8) if sym else rng.integers(0, 16, size=(n, k // 128), dtype=np.uint8)
    s = rng.uniform(0.005, 0.02, size=(n, k // 128)).astype(np.float16)
    if headroom:       # the int32 / (float)r headroom: q = 15, z = 0 against mantissas at the group maximum
        q[:, :128] = 15
        z[:, 0] = 0
    return q, z, s


def activations(kind, m, k, seed=0):
    """(M, K) fp16 activations of one of the kinds of CASES"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((m, k)) * np.logspace(-2, 1, k)[rng.permutation(k)]
    if kind == "adv":
        for t in range(m):
            for g in range(k // 128):
                sl = slice(g * 128, (g + 1) * 128)
                j = g % 7 - 3
                pat = (t + g) % 6
                v = rng.standard_normal(128) * 2.0 ** j
                i = rng.integers(128)
                if pat == 0:        # group maximum exactly a power of two
                    v = np.clip(v, -2.0 ** j * 0.99, 2.0 ** j * 0.99)
                    v[i] = -(2.0 ** j)
                elif pat == 1:      # group maximum at the top of its binade
                    v = np.clip(v, -2.0 ** j, 2.0 ** j)
                    v[i] = (2 - 2.0 ** -10) * 2.0 ** j
                elif pat == 2:      # all zero
                    v[:] = 0
                elif pat == 3:      # fp16 subnormals only
                    v = rng.integers(-1023, 1024, 128) * 2.0 ** -24
                elif pat == 4:      # one huge element: the tiny ones flush to zero mantissas
                    v = rng.standard_normal(128) * 1e-3
                    v[i] = 1536.0
                x[t, sl] = v
    elif kind == "headroom":
        x = rng.standard_normal((m, k)) * 0.1
        x[:, :128] = (2 - 2.0 ** -10) * 2.0 ** -4
    x = x.astype(np.float16)
    if kind == "nonfinite":
        x[0, 7] = np.inf
        x[1, k - 3] = np.nan
    return x
