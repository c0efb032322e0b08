"""GPU parity against the REFERENCE's own kernels (the reference's hot-path .cu files recompiled for sm_90a behind the
thin shim oracle/ref_shim.cu) on identical inputs -- north_star: "outputs match the reference's own kernels on
identical inputs (bit-exact for GPTQ unpack/index, within 1e-3 rel for fp16)".

The reference's outputs on this module's seeded inputs are stored in tests/golden/vs_reference.npz: a SHA-256 digest of
the whole output where the comparison is bit-exact; where it is a tolerance, float outputs of up to 16384 elements
whole and a fixed seeded sample of 4096 elements of larger ones; small tables whole.  With
ZL_RECORD_REFERENCE_GOLDEN=<file> and oracle/_ref/libzl_ref.so built (build() with ZHILIGHT_REFERENCE set), the tests run the reference kernels instead, check against them, and write that file."""
import hashlib
import os
import zlib

import numpy as np
import pytest
import torch

from oracle import gptq
from tests.helpers import rel_l2

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libzl_ref.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "vs_reference.npz")
RECORD = os.environ.get("ZL_RECORD_REFERENCE_GOLDEN")
SAMPLE = 4096         # elements kept of a larger float output compared within a tolerance
WHOLE = 16384         # float outputs up to this many elements are kept whole
FULL = 2048           # full(): small tables of any type


def _bytes(t):
    return t.detach().contiguous().cpu().reshape(-1).view(torch.uint8).numpy().tobytes()


def _sample_idx(key, size):
    if size <= WHOLE:
        return np.arange(size)
    return np.sort(np.random.default_rng(zlib.crc32(key.encode())).choice(size, size=SAMPLE, replace=False))


def _encode(t):
    """flat values in the fixture: fp16 as float16, bf16 as its 16-bit pattern, anything else as float32"""
    t = t.detach().contiguous().cpu().reshape(-1)
    if t.dtype == torch.float16:
        return t.numpy()
    if t.dtype == torch.bfloat16:
        return t.view(torch.int16).numpy().view(np.uint16)
    return t.float().numpy()


def _decode(a):
    if a.dtype == np.uint16:
        return (a.astype(np.uint32) << 16).view(np.float32)
    return a.astype(np.float32)


class RefOutputs:
    """The reference kernels' outputs: recorded live from oracle/_ref (record mode) or read from the stored fixture."""

    def __init__(self, ref):
        self.ref = ref
        self.rec = {}
        self.data = None if ref is not None else np.load(GOLDEN)

    def _get(self, key, fn, make):
        name = key.replace("/", ".")
        if self.ref is None:
            return self.data[name]
        v = make(fn(self.ref))
        assert name not in self.rec, key
        self.rec[name] = v
        return v

    def digest(self, key, fn):
        """sha256 of the reference tensor's bytes; compare with digest_of(ours)"""
        return bytes(self._get(key, fn, lambda t: np.frombuffer(hashlib.sha256(_bytes(t)).digest(), np.uint8)))

    def sample(self, key, fn):
        """(flat indices, float32 values) of the reference tensor: all of it up to WHOLE elements, else a fixed seeded
        sample; pick(ours, idx) gives ours"""
        name = key.replace("/", ".")
        if self.ref is None:
            size = int(self.data[name + ".size"])
            return _sample_idx(key, size), _decode(self.data[name])
        t = fn(self.ref)
        idx = _sample_idx(key, t.numel())
        assert name not in self.rec, key
        self.rec[name] = _encode(t)[idx]
        self.rec[name + ".size"] = np.int64(t.numel())
        return idx, _decode(self.rec[name])

    def full(self, key, fn):
        """the whole (small) reference output as numpy (bf16 as float32)"""
        def make(t):
            assert t.numel() <= FULL, key
            return t.detach().float().cpu().numpy() if t.dtype == torch.bfloat16 else t.detach().cpu().numpy()
        return self._get(key, fn, make)

    def save(self, path):
        np.savez_compressed(path, **self.rec)


def digest_of(t):
    return hashlib.sha256(_bytes(t)).digest()


def pick(t, idx):
    a = t.detach().float().cpu().reshape(-1).numpy() if isinstance(t, torch.Tensor) else np.asarray(t, np.float32).reshape(-1)
    return a[idx]


@pytest.fixture(scope="module")
def ref(cuda):
    if RECORD:
        assert os.path.exists(REF_LIB), "recording needs oracle/_ref/libzl_ref.so"
        from oracle.gen_ref_golden import Ref
        outs = RefOutputs(Ref())
        yield outs
        outs.save(RECORD)
    else:
        yield RefOutputs(None)


def _t(a, cuda):
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


def test_load_pipeline_bit_exact_vs_reference(lib, ref, cuda):
    from zhilight_b200 import ops
    k, n = 4096, 4096
    qw, qz, sc, gi = gptq.make_gptq_checkpoint(k, n, 128, False, seed=0)
    o_qw, o_qz, o_sc = ops.gptq_to_k_major(_t(qw, cuda), _t(qz, cuda), _t(sc, cuda))
    for i, o in enumerate((o_qw, o_qz, o_sc)):
        assert digest_of(o) == ref.digest("load/%d" % i, lambda r, i=i: r.gptq_to_k_major(qw, qz, sc)[i])
    assert digest_of(ops.gptq_dequant_k_major(o_qw, o_qz, o_sc)) == \
        ref.digest("load/dequant", lambda r: r.dequant_k_major(*r.gptq_to_k_major(qw, qz, sc)))


def test_awq_pipeline_bit_exact_vs_reference(lib, ref, cuda):
    from zhilight_b200 import ops
    k, n, g = 1024, 512, 128
    rng = np.random.default_rng(1)
    qw = rng.integers(0, 2 ** 32, size=(k, n // 8), dtype=np.uint64).astype(np.uint32).view(np.int32)
    qz = rng.integers(0, 2 ** 32, size=(k // g, n // 8), dtype=np.uint64).astype(np.uint32).view(np.int32)
    sc = (0.01 * rng.random((k // g, n))).astype(np.float16)
    o = ops.gptq_to_k_major(_t(qw, cuda), _t(qz, cuda), _t(sc, cuda), is_awq=True)
    for i, b in enumerate(o):
        assert digest_of(b) == ref.digest("awq_load/%d" % i, lambda r, i=i: r.gptq_to_k_major(qw, qz, sc, awq=True)[i])


@pytest.mark.parametrize("sym", [False, True])
@pytest.mark.parametrize("m", [1, 4, 16, 33])
def test_w4a16_vs_reference_gemv(lib, ref, cuda, sym, m):
    """BASELINE config 1 shape.  The reference accumulates 8 products in fp16, we accumulate in fp32: the two
    must agree to ~1e-3 (L2) and ours must be the closer one to the exact result."""
    from zhilight_b200 import ops
    k = n = 4096
    qw, qz, sc, gi = gptq.make_gptq_checkpoint(k, n, 128, sym, seed=0)
    d_qw, d_qz, d_sc = ops.gptq_to_k_major(_t(qw, cuda), _t(qz, cuda), _t(sc, cuda))   # == the reference's (test above)
    x = torch.randn(m, k, generator=torch.Generator().manual_seed(0)).half().to(cuda)
    idx, y_ref = ref.sample("gemv/%d/%d" % (m, sym), lambda r: r.gemv(x, *r.gptq_to_k_major(qw, qz, sc), None, sym))
    packed = ops.w4_pack(d_qw, d_qz, d_sc, 128, sym)
    y = ops.w4a16_gemm(x, packed, n, k).float().cpu().numpy()
    o_qw, o_qz, o_sc, _ = gptq.to_k_major(qw, qz, sc, gi, 128)
    exact = gptq.gemm_f32(x.cpu().numpy(), gptq.dequant_k_major_f32(o_qw, o_qz, o_sc, sym))
    assert rel_l2(pick(y, idx), y_ref) <= 2e-3
    assert rel_l2(y, exact) <= 1e-3
    assert rel_l2(pick(y, idx), pick(exact, idx)) <= rel_l2(y_ref, pick(exact, idx)) + 1e-4


def test_swiglu_vs_reference_fused_gate_in(lib, ref, cuda):
    from zhilight_b200 import ops
    k, f = 4096, 1024
    a = gptq.make_gptq_checkpoint(k, f, 128, False, seed=2)
    b = gptq.make_gptq_checkpoint(k, f, 128, False, seed=3)
    ga = ops.gptq_to_k_major(_t(a[0], cuda), _t(a[1], cuda), _t(a[2], cuda))
    ub = ops.gptq_to_k_major(_t(b[0], cuda), _t(b[1], cuda), _t(b[2], cuda))
    x = torch.randn(2, k, generator=torch.Generator().manual_seed(1)).half().to(cuda)
    idx, y_ref = ref.sample("gate_in", lambda r: r.gate_in(x, r.gptq_to_k_major(a[0], a[1], a[2]),
                                                         r.gptq_to_k_major(b[0], b[1], b[2])))
    fused = [torch.cat([p, q]).contiguous() for p, q in zip(ga, ub)]
    packed = ops.w4_pack(fused[0], fused[1], fused[2], 128, False, ops.swiglu_row_map(f, cuda))
    y = ops.w4a16_gemm(x, packed, 2 * f, k, epilogue=ops.EPI_SWIGLU).float().cpu().numpy()
    assert rel_l2(pick(y, idx), y_ref) <= 4e-3


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_norm_rope_vs_reference(lib, ref, cuda, dtype):
    from zhilight_b200 import ops
    g = torch.Generator().manual_seed(3)
    t, d = 7, 4096
    a = torch.randn(t, d, generator=g).to(dtype).to(cuda)
    b = torch.randn(t, d, generator=g).to(dtype).to(cuda)
    w = (1 + 0.1 * torch.randn(d, generator=g)).to(dtype).to(cuda)
    ulp = 2 ** -10 if dtype == torch.float16 else 2 ** -7
    tag = str(dtype).split(".")[-1]
    close = lambda ours, idx, theirs, atol: np.testing.assert_allclose(pick(ours, idx), theirs, rtol=ulp, atol=atol)
    close(ops.rmsnorm(a, w, 1e-5), *ref.sample("rmsnorm/" + tag, lambda r: r.rmsnorm(a, w, 1e-5)), 1e-6)
    s, y = ops.add_rmsnorm(a, b, w, 1e-5, mode=1)
    assert digest_of(s) == ref.digest("fuse_add/s/" + tag, lambda r: r.rmsnorm_fuse_add(a, b, w, 1e-5)[0])
    close(y, *ref.sample("fuse_add/y/" + tag, lambda r: r.rmsnorm_fuse_add(a, b, w, 1e-5)[1]), 1e-6)
    assert digest_of(ops.element_add_scale(a, b, 1.0)) == ref.digest("element_add/" + tag, lambda r: r.element_add(a, b))
    hq, hkv, dh = 32, 8, 128
    qkv = torch.randn(t, (hq + 2 * hkv) * dh, generator=g).to(dtype).to(cuda)
    pos = torch.tensor([0, 1, 2, 100, 1000, 5000, 8191], dtype=torch.int32, device=cuda)
    cos, sin = ops.rope_cos_sin(pos, dh, 500000.0, dict(factor=8.0, low=1.0, high=4.0, orig=8192.0))
    q, k, v = ops.rope_qk_cache(cos, sin, qkv, hq, hkv, dh)
    rope = lambda r: r.rope_qk_cache(cos, sin, qkv, hq, hkv, dh)
    close(q, *ref.sample("rope/q/" + tag, lambda r: rope(r)[0]), 1e-3)
    close(k, *ref.sample("rope/k/" + tag, lambda r: rope(r)[1]), 1e-3)
    assert digest_of(v) == ref.digest("rope/v/" + tag, lambda r: rope(r)[2])


@pytest.mark.parametrize("lens", [[4096, 123], [300, 1024, 77], [2048, 2048]])
def test_decode_attention_vs_reference(lib, ref, cuda, lens):
    """src/nn/tests/test_attention_rag_buffer.cpp shape: 4 kv-heads x m_query 4, lens {4096, 123}."""
    from zhilight_b200 import ops
    hq, hkv, d = 16, 4, 128
    g = torch.Generator().manual_seed(4)
    b = len(lens)
    q = torch.randn(b, 1, hq, d, generator=g).half().to(cuda)
    ks = [torch.randn(lb, hkv, d, generator=g).half().to(cuda) for lb in lens]
    vs = [torch.randn(lb, hkv, d, generator=g).half().to(cuda) for lb in lens]
    masks = []
    for lb in lens:
        m = torch.ones(lb, dtype=torch.int8)
        m[lb - 3:] = 0
        masks.append(m)
    mask = torch.cat(masks).to(cuda)
    lens_t = torch.tensor(lens, dtype=torch.int32, device=cuda)
    idx, out_ref = ref.sample("attention/%s" % "-".join(map(str, lens)),
                              lambda r: r.attention(q, lens_t, ks, vs, mask, d ** -0.5, hkv))
    out = ops.decode_attention(q, lens_t, ks, vs, mask, d ** -0.5, max(lens), hkv)
    assert rel_l2(pick(out, idx), out_ref) <= 1e-3


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_int8_linear_bit_exact_vs_reference_kernels(lib, ref, cuda, dt):
    """Int8Linear = quant_calc_scale -> s32 GEMM -> quant_scale_back (linear.cpp:560-636).  The s32 GEMM is exact
    integer arithmetic (torch int matmul stands in for cuBLASLt); both ends are the reference's own kernels."""
    from zhilight_b200 import ops
    m, n, k = 7, 1536, 4096
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(m, k, generator=g) * 1.3).to(dt).to(cuda)
    w_q = torch.randint(-127, 128, (n, k), generator=g, dtype=torch.int8).to(cuda)
    w_s = (0.0005 + 0.003 * torch.rand(n, generator=g)).to(dt).to(cuda)
    tag = str(dt).split(".")[-1]
    q, s = ops.int8_quant_per_token(x)
    assert digest_of(q) == ref.digest("int8/q/" + tag, lambda r: r.quant_calc_scale_dt(x)[0])
    assert digest_of(s) == ref.digest("int8/s/" + tag, lambda r: r.quant_calc_scale_dt(x)[1])
    acc = (q.cpu().int() @ w_q.cpu().int().T).to(cuda)
    y = ops.int8_linear(x, w_q, w_s)
    assert digest_of(y) == ref.digest("int8/y/" + tag, lambda r: r.quant_scale_back(acc, s, w_s, dt))


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_rmsnorm_quant_vs_reference(lib, ref, cuda, dt):
    from zhilight_b200 import ops
    t, d = 5, 4096
    g = torch.Generator().manual_seed(4)
    x = torch.randn(t, d, generator=g).to(dt).to(cuda)
    w = (1 + 0.2 * torch.randn(d, generator=g)).to(dt).to(cuda)
    tag = str(dt).split(".")[-1]
    y, q, s = ops.rmsnorm_quant(x, w, 1e-5)
    assert digest_of(q) == ref.digest("ln_quant/q/" + tag, lambda r: r.layernorm_quant(x, w, 1e-5)[1])
    np.testing.assert_allclose(s.cpu().numpy(), ref.full("ln_quant/s/" + tag, lambda r: r.layernorm_quant(x, w, 1e-5)[2]),
                               rtol=1e-6, atol=0)
    idx, ry = ref.sample("ln_quant/y/" + tag, lambda r: r.layernorm_quant(x, w, 1e-5)[0])
    assert rel_l2(pick(y, idx), ry) < 1e-3


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_fp8_linear_vs_reference(lib, ref, cuda, dt):
    """dynamic_scaled_quant codes must be identical; the GEMM is cuBLASLt fp8 in the reference (fp32 accumulate,
    different summation order): <= 1e-3 rel."""
    from zhilight_b200 import ops
    m, n, k = 8, 2048, 4096
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(m, k, generator=g) * 2).to(dt).to(cuda)
    w8 = (torch.randn(n, k, generator=g) * 0.5).to(torch.float8_e4m3fn).view(torch.uint8).to(cuda)
    sw = torch.tensor([0.01], dtype=torch.float32, device=cuda)
    tag = str(dt).split(".")[-1]
    q, s = ops.fp8_quant_per_tensor(x)
    assert digest_of(s) == ref.digest("fp8/s/" + tag, lambda r: r.fp8_quant(x)[1])
    assert digest_of(q) == ref.digest("fp8/q/" + tag, lambda r: r.fp8_quant(x)[0])
    idx, y_ref = ref.sample("fp8/y/" + tag, lambda r: r.fp8_gemm(*r.fp8_quant(x), w8, sw, None, dt))
    y = ops.w8a8_gemm(q, s, w8, sw, dt, kind=ops.W8_FP8).float().cpu().numpy()
    assert rel_l2(pick(y, idx), y_ref) < (1e-3 if dt == torch.float16 else 4e-3)


# ---- round 2: rope tables, Marlin, native AWQ against the reference's own kernels ----
LLAMA3_8 = dict(factor=8.0, low=1.0, high=4.0, orig=8192)
LLAMA3_32 = dict(factor=32.0, low=1.0, high=4.0, orig=8192)


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("theta,l3", [(10000.0, None), (500000.0, LLAMA3_8), (500000.0, LLAMA3_32)],
                         ids=["plain", "llama3-f8", "llama3-f32"])
def test_rope_cos_sin_vs_reference_rope_preparer(lib, ref, cuda, d, theta, l3):
    """zl_rope_cos_sin against RopePreparer / KERNEL_rope_cos_sin(_llama3) (src/nn/position/rope_preparer.cu:49-161).
    Both evaluate the same fp32 expression, so the tables agree to the last bits even at position 100000 where a
    1-ulp change of inv_freq already moves cos by 1e-2: every llama3-rope model depends on this table."""
    from zhilight_b200 import ops
    pos = torch.tensor([0, 1, 2, 63, 4095, 8191, 8192, 100000], dtype=torch.int32, device=cuda)
    key = "rope_table/%d/%g/%s" % (d, theta, l3["factor"] if l3 else "plain")
    c_ref = ref.full(key + "/cos", lambda r: r.rope_cos_sin(pos, d, theta, l3)[0])
    s_ref = ref.full(key + "/sin", lambda r: r.rope_cos_sin(pos, d, theta, l3)[1])
    c, s = (a.cpu().numpy() for a in ops.rope_cos_sin(pos, d, theta, l3))
    np.testing.assert_allclose(c, c_ref, rtol=0, atol=2e-6)
    np.testing.assert_allclose(s, s_ref, rtol=0, atol=2e-6)
    assert float((c == c_ref).mean()) > 0.99 and float((s == s_ref).mean()) > 0.99


def _sym_checkpoint(k, n, seed):
    rng = np.random.default_rng(seed)
    qw = rng.integers(0, 2 ** 32, size=(k // 8, n), dtype=np.uint64).astype(np.uint32).view(np.int32)
    sc = (0.002 + 0.004 * rng.random((k // 128, n))).astype(np.float16)
    qz = np.full((k // 128, n // 8), 0x77777777, dtype=np.uint32).view(np.int32)      # stored 7 -> zero 8 (u4b8)
    return qw, qz, sc


@pytest.mark.parametrize("m", [1, 16, 32, 64])
@pytest.mark.parametrize("k,n", [(4096, 4096), (4096, 14336)])
def test_quant_type_8_vs_reference_marlin_kernel(lib, ref, cuda, k, n, m):
    """QuantType 8 (GPTQ_Marlin): our kernels on a symmetric g128 checkpoint against the reference's gptq_marlin_gemm
    (src/nn/quant/marlin/gptq_marlin.cu:2034-2192) fed by gptq_marlin_repack + the scale permutation of
    GPTQMarlin::post_load (linear.cpp:1402-1428).  Marlin multiplies fp16 dequantised weights with fp32 accumulation;
    M <= 16 runs our exact-integer kernel, M > 16 the wgmma kernel: both within 1e-3 (L2) of it and of the fp32 oracle."""
    from zhilight_b200 import ops
    qw, qz, sc = _sym_checkpoint(k, n, 5)
    x = torch.randn(m, k, generator=torch.Generator().manual_seed(m)).half().to(cuda)
    idx, y_ref = ref.sample("marlin/%d/%d/%d" % (k, n, m), lambda r: r.marlin_gemm(x, r.t(qw), r.t(sc)))
    o_qw, o_qz, o_sc = ops.gptq_to_k_major(_t(qw, cuda), _t(qz, cuda), _t(sc, cuda))
    packed = ops.w4_pack(o_qw, o_qz, o_sc, 128, True, variant=1)
    y = ops.w4a16_gemm_fused(x, packed, n, k, variant=1).float().cpu().numpy()
    k_qw, k_qz, k_sc, _ = gptq.to_k_major(qw, qz, sc, np.arange(k) // 128, 128)
    exact = gptq.gemm_f32(x.cpu().numpy(), gptq.dequant_k_major_f32(k_qw, k_qz, k_sc, True))
    assert rel_l2(pick(y, idx), y_ref) <= 1e-3
    assert rel_l2(y, exact) <= 1e-3 and rel_l2(y_ref, pick(exact, idx)) <= 1e-3


def test_marlin_repack_is_a_permutation_of_the_checkpoint(lib, ref, cuda):
    """gptq_marlin_repack (gptq_marlin_repack.cu:258-318) only permutes nibbles: same multiset per 16 x 64 tile."""
    k, n = 256, 128
    qw, _, _ = _sym_checkpoint(k, n, 9)
    nib = lambda a: np.stack([(a >> (4 * i)) & 15 for i in range(8)]).reshape(-1)
    hist = ref.full("marlin_repack/hist", lambda r: torch.from_numpy(np.bincount(
        nib(r.marlin_repack(r.t(qw)).cpu().numpy().view(np.uint32)).astype(np.int64), minlength=16)))
    shape = ref.full("marlin_repack/shape", lambda r: torch.tensor(r.marlin_repack(r.t(qw)).shape))
    assert tuple(shape) == (k // 16, 2 * n)
    np.testing.assert_array_equal(hist, np.bincount(nib(qw.view(np.uint32)).astype(np.int64), minlength=16))


@pytest.mark.parametrize("m", [1, 8, 32])
def test_awq_native_gemm_vs_ours(lib, ref, cuda, m):
    """QuantType 6 through the reference's native awq_gemm (src/nn/quant/awq/gemm_kernels.cu:404-468, split-k 32) against
    our AWQ path (shuffle_awq / un_shuffle into the k-major layout, then the W4A16 kernels): same w = (q - z) * s."""
    from zhilight_b200 import ops
    k, n, g = 2048, 1024, 128
    rng = np.random.default_rng(3)
    qw = rng.integers(0, 2 ** 32, size=(k, n // 8), dtype=np.uint64).astype(np.uint32).view(np.int32)
    qz = rng.integers(0, 2 ** 32, size=(k // g, n // 8), dtype=np.uint64).astype(np.uint32).view(np.int32)
    sc = (0.002 + 0.004 * rng.random((k // g, n))).astype(np.float16)
    x = torch.randn(m, k, generator=torch.Generator().manual_seed(7)).half().to(cuda)
    idx, y_ref = ref.sample("awq_gemm/%d" % m, lambda r: r.awq_gemm(x, r.t(qw), r.t(sc), r.t(qz)))
    o_qw, o_qz, o_sc = ops.gptq_to_k_major(_t(qw, cuda), _t(qz, cuda), _t(sc, cuda), is_awq=True)
    packed = ops.w4_pack(o_qw, o_qz, o_sc, 128, False, variant=1)
    y = ops.w4a16_gemm_fused(x, packed, n, k, variant=1).float().cpu().numpy()
    # awq_gemm sums 32 fp16 partial tensors (KERNEL_sum_dim0): it is the noisier side
    assert rel_l2(pick(y, idx), y_ref) <= 3e-3


# ---- int8 KV cache: quantising append and the split-KV quant attention kernel ----
def _kv8_case(cuda, lens, hq, hkv, d, seed):
    g = torch.Generator().manual_seed(seed)
    b = len(lens)
    q = torch.randn(b, 1, hq, d, generator=g).half().to(cuda)
    ks = [torch.randn(lb, hkv, d, generator=g).half().to(cuda) for lb in lens]
    vs = [torch.randn(lb, hkv, d, generator=g).half().to(cuda) for lb in lens]
    masks = []
    for lb in lens:
        m = torch.ones(lb, dtype=torch.int8)
        m[lb - 3:] = 0
        m[torch.randperm(lb - 3, generator=g)[: lb // 11]] = 0
        masks.append(m)
    return q, ks, vs, torch.cat(masks).to(cuda), torch.tensor(lens, dtype=torch.int32, device=cuda)


def test_kv_int8_quant_append_bit_exact_vs_reference(lib, ref, cuda):
    """codes and scales of our cache-side quantisation == int8_op::quant_calc_scale(x, 127, 128) (quant_kernel.cu:15-47)"""
    from zhilight_b200 import ops
    hkv, d, t = 2, 128, 7
    g = torch.Generator().manual_seed(3)
    k = (torch.randn(t, hkv, d, generator=g) * 2).half().to(cuda)
    v = torch.randn(t, hkv, d, generator=g).half().to(cuda)
    kq_ref, ks_ref = (ref.full("kv_append/k/%d" % i, lambda r, i=i: r.quant_u8(k.view(t * hkv, d))[i]) for i in range(2))
    vq_ref, vs_ref = (ref.full("kv_append/v/%d" % i, lambda r, i=i: r.quant_u8(v.view(t * hkv, d))[i]) for i in range(2))
    kq_ref, ks_ref, vq_ref, vs_ref = (torch.from_numpy(a).to(cuda) for a in (kq_ref, ks_ref, vq_ref, vs_ref))
    tb = torch.tensor([0, 1, 0, 1, 0, 1, 0], dtype=torch.int32, device=cuda)
    pl = torch.tensor([0, 0, 1, 1, 2, 2, 3], dtype=torch.int32, device=cuda)
    kb = [torch.zeros(4, hkv, d, dtype=torch.uint8, device=cuda) for _ in range(2)]
    vb = [torch.zeros(4, hkv, d, dtype=torch.uint8, device=cuda) for _ in range(2)]
    sk = [torch.zeros(4, hkv, dtype=torch.float32, device=cuda) for _ in range(2)]
    sv = [torch.zeros(4, hkv, dtype=torch.float32, device=cuda) for _ in range(2)]
    ops.kv_int8_quant_append(k, v, tb, pl, kb, vb, sk, sv)
    for i in range(t):
        b_, p_ = int(tb[i]), int(pl[i])
        assert torch.equal(kb[b_][p_], kq_ref.view(t, hkv, d)[i]) and torch.equal(vb[b_][p_], vq_ref.view(t, hkv, d)[i])
        assert torch.equal(sk[b_][p_], ks_ref.view(t, hkv)[i]) and torch.equal(sv[b_][p_], vs_ref.view(t, hkv)[i])


@pytest.mark.parametrize("lens", [[1600, 600], [2000], [1100, 1300, 40]])
def test_decode_attention_kv8_vs_reference_quant_kernel(lib, ref, cuda, lens):
    """zl_decode_attention_kv8 against KERNEL_mqa_rag_buffer_split_kv_quant (attention_kernel.cu:804-880) on the same uint8
    caches and scales (the reference only takes its quant kernel above 1024 keys, with < 1024 keys per split).

    The reference kernel offsets the K / V pointers of split s by s * len_split rows but NOT the scale pointers
    (attention_kernel.cu:847-851: scale_key = scale_key_addrs[b] + head_kv), i.e. every split after the first multiplies
    its logits and probabilities with the scales of the FIRST split's tokens: 0.2-0.4 relative
    error against the fp32 evaluation of the same cache.  The comparison therefore uses caches whose rows all share one
    scale per head (every row carries one element of magnitude 4.0), where that indexing is harmless; with per-row scales
    our kernel is checked against the fp32 evaluation (next test and the assertions on `exact` here).
    The reference multiplies q.k in fp16 (quant_attention.cuh:60-70): both within 2e-3, ours within 1e-3 of exact."""
    from zhilight_b200 import ops
    hq, hkv, d = 8, 2, 128
    q, ks, vs, mask, lens_t = _kv8_case(cuda, lens, hq, hkv, d, 17)
    for t in ks + vs:                      # one common absmax per (row, head): identical scales along the buffer
        t.clamp_(-4.0, 4.0)
        t[:, :, 5] = 4.0
    key = "kv8_attention/%s" % "-".join(map(str, lens))
    kq, vq, sk, sv = [], [], [], []
    for i, (k, v) in enumerate(zip(ks, vs)):
        for src, codes, scales, name in ((k, kq, sk, "k"), (v, vq, sv, "v")):
            lb = src.shape[0]
            c = torch.zeros(lb, hkv, d, dtype=torch.uint8, device=cuda)
            sc = torch.zeros(lb, hkv, dtype=torch.float32, device=cuda)
            c2, sc2 = torch.zeros_like(c), torch.zeros_like(sc)
            ops.kv_int8_quant_append(src, src, torch.zeros(lb, dtype=torch.int32, device=cuda),
                                     torch.arange(lb, dtype=torch.int32, device=cuda), [c], [c2], [sc], [sc2])
            assert digest_of(c) == ref.digest("%s/%s%d/codes" % (key, name, i), lambda r: r.quant_u8(src.view(-1, d))[0])
            assert digest_of(sc) == ref.digest("%s/%s%d/scales" % (key, name, i), lambda r: r.quant_u8(src.view(-1, d))[1])
            codes.append(c)
            scales.append(sc)
    assert float(sk[0].max() - sk[0].min()) == 0.0
    scale = 1.0 / np.sqrt(d)
    idx, y_ref = ref.sample(key, lambda r: r.attention_kv8(q, lens_t, kq, vq, sk, sv, mask, scale, hkv))
    y = ops.decode_attention_kv8(q, lens_t, kq, vq, sk, sv, mask, scale, max(lens), hkv).float().cpu().numpy()
    # fp32 evaluation of the same quantised cache
    from oracle import ops as oops
    kd = [((a.float() - 128) * s[:, :, None]).cpu().numpy() for a, s in zip(kq, sk)]
    vd = [((a.float() - 128) * s[:, :, None]).cpu().numpy() for a, s in zip(vq, sv)]
    off = np.cumsum([0] + lens)
    masks = [mask[off[i]:off[i + 1]].cpu().numpy().reshape(1, -1) for i in range(len(lens))]
    exact = oops.decode_attention(q.cpu().numpy(), kd, vd, lens, masks, scale, hq // hkv, "f32")
    assert rel_l2(y, exact) <= 1e-3
    assert rel_l2(pick(y, idx), y_ref) <= 2e-3
    # at least as close to the exact result as the reference
    assert rel_l2(pick(y, idx), pick(exact, idx)) <= rel_l2(y_ref, pick(exact, idx)) + 2e-4


def test_decode_attention_kv8_per_row_scales_long_context(lib, cuda):
    """per-row scales (what a real cache holds) over split contexts: against the fp32 evaluation of the quantised cache"""
    from zhilight_b200 import ops
    from oracle import ops as oops
    hq, hkv, d = 8, 2, 128
    lens = [1600, 600, 2100]
    g = torch.Generator().manual_seed(23)
    q = torch.randn(3, 1, hq, d, generator=g).half().to(cuda)
    kq = [torch.randint(0, 256, (lb, hkv, d), generator=g, dtype=torch.uint8).to(cuda) for lb in lens]
    vq = [torch.randint(0, 256, (lb, hkv, d), generator=g, dtype=torch.uint8).to(cuda) for lb in lens]
    sk = [(0.002 + 0.004 * torch.rand(lb, hkv, generator=g)).to(cuda) for lb in lens]
    sv = [(0.005 + 0.02 * torch.rand(lb, hkv, generator=g)).to(cuda) for lb in lens]
    lens_t = torch.tensor(lens, dtype=torch.int32, device=cuda)
    mask = (torch.rand(sum(lens), generator=g) > 0.1).to(torch.int8).to(cuda)
    scale = 1.0 / np.sqrt(d)
    y = ops.decode_attention_kv8(q, lens_t, kq, vq, sk, sv, mask, scale, max(lens), hkv).float().cpu().numpy()
    kd = [((a.float() - 128) * s[:, :, None]).cpu().numpy() for a, s in zip(kq, sk)]
    vd = [((a.float() - 128) * s[:, :, None]).cpu().numpy() for a, s in zip(vq, sv)]
    off = np.cumsum([0] + lens)
    masks = [mask[off[i]:off[i + 1]].cpu().numpy().reshape(1, -1) for i in range(len(lens))]
    exact = oops.decode_attention(q.cpu().numpy(), kd, vd, lens, masks, scale, hq // hkv, "f32")
    assert rel_l2(y, exact) <= 1e-3


def test_decode_attention_kv8_short_context_and_gqa4(lib, cuda):
    """below the reference's split threshold (its quant kernel is never taken there) and with m_query = 4: against the fp32
    evaluation of the quantised cache"""
    from zhilight_b200 import ops
    from oracle import ops as oops
    hq, hkv, d = 8, 2, 128
    lens = [130, 17, 512]
    g = torch.Generator().manual_seed(5)
    q = torch.randn(3, 1, hq, d, generator=g).half().to(cuda)
    kq = [torch.randint(0, 256, (lb, hkv, d), generator=g, dtype=torch.uint8).to(cuda) for lb in lens]
    vq = [torch.randint(0, 256, (lb, hkv, d), generator=g, dtype=torch.uint8).to(cuda) for lb in lens]
    sk = [(0.01 + 0.01 * torch.rand(lb, hkv, generator=g)).to(cuda) for lb in lens]
    sv = [(0.01 + 0.01 * torch.rand(lb, hkv, generator=g)).to(cuda) for lb in lens]
    lens_t = torch.tensor(lens, dtype=torch.int32, device=cuda)
    mask = torch.ones(sum(lens), dtype=torch.int8, device=cuda)
    scale = 1.0 / np.sqrt(d)
    y = ops.decode_attention_kv8(q, lens_t, kq, vq, sk, sv, mask, scale, max(lens), hkv).float().cpu().numpy()
    kd = [((a.float() - 128) * s[:, :, None]).cpu().numpy() for a, s in zip(kq, sk)]
    vd = [((a.float() - 128) * s[:, :, None]).cpu().numpy() for a, s in zip(vq, sv)]
    masks = [np.ones((1, lb), np.int8) for lb in lens]
    exact = oops.decode_attention(q.cpu().numpy(), kd, vd, lens, masks, scale, hq // hkv, "f32")
    assert rel_l2(y, exact) <= 1e-3
