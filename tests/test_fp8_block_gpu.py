"""FP8 block-scaled Linear (QuantType 10) on the GPU against the CPU oracle (tests/fp8_block_oracle.py).

The activation quantisation is bit-exact (codes and scales).  The block GEMM is held to 2e-3 relative L2 against a
float64 sum of the same codes; its block scales span 1e-3 .. 1e2, so one scale per row or scaling after the k-sum
fails by orders of magnitude.  The decode driver is compared with the oracle model run through the same Linear.  Where
the driver's attention differs from the oracle's in the last bits (chunked prefill, joined steps, the int8 KV cache), an
fp16 ulp upstream moves an activation to the neighbouring e4m3 code (3 mantissa bits: a 6-12% step), and the logits
differ by a few 1e-2.  The per-tensor FP8 model (QuantType 7) shows the same spread on the same comparison, measured on
an H100: a 70-token chunked prefill of TINY128 against the token-by-token oracle, 4.7e-2 (type 7) and 5.2e-2 (type 10),
against 1.0e-3 for the fp16 model.  Those paths are held to 6e-2 (1e-1 for TINY128 in chunks of 64); decode steps of
the tiny models to 6e-3 / 2e-2.  A scale applied to the wrong 128x128 block is off by up to 16x (the synthetic scales
span 0.0075 .. 0.12) and fails all of these bounds."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import model as omodel, ops as oops
from tests import fp8_block_oracle as fb
from tests.helpers import rel_l2
from tests.kv8_oracle import Kv8OracleLlama
from tests.test_llama_gpu import LAYER8B, TINY, TINY128

pytestmark = pytest.mark.gpu
DT = {"f16": torch.float16, "bf16": torch.bfloat16}
F32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_FP8 = os.path.join(ROOT, "oracle", "_ref", "libzl_ref_fp8.so")
DROPIN_FP8 = os.path.join(ROOT, "oracle", "_ref", "libzl_dropin_fp8.so")


def _x(m, k, tag, seed, amp=1.5):
    r = np.random.default_rng(seed)
    return oops._t(r.standard_normal((m, k)) * amp, tag)


def _dev(a, tag):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=F32)).to(DT[tag]).cuda()


def _host(t):
    return t.float().cpu().numpy()


@pytest.mark.parametrize("tag", ["f16", "bf16"])
@pytest.mark.parametrize("m,k", [(1, 128), (5, 4096), (33, 14336), (300, 1024)])
def test_quant_codes_and_scales_bit_exact(lib, cuda, tag, m, k):
    from zhilight_b200 import ops
    x = _x(m, k, tag, seed=m + k)
    x[0, :128] = 0                                         # all-zero group: amax clamps to 1e-4
    if k >= 256:
        x[-1, 128:256] *= 1e-6                             # below the clamp
        x[-1, 130] = -3.0                                  # the group's extreme: -448
    x = oops._t(x, tag)
    q, s = ops.fp8_quant_per_token_group(_dev(x, tag))
    rq, rs = fb.quant_per_token_group(x)
    np.testing.assert_array_equal(q.cpu().numpy(), rq)
    np.testing.assert_array_equal(s.cpu().numpy()[:, :m], rs[:, :m])
    assert q.cpu().numpy()[0, :128].max() == 0


def test_quant_strided_input(lib, cuda):
    from zhilight_b200 import _lib, ops
    x = _x(6, 768, "f16", seed=3)
    xd = _dev(x, "f16")[:, 256:768]                        # row stride 768, K = 512
    ld = 8
    q = torch.empty((6, 512), dtype=torch.uint8, device="cuda")
    s = torch.empty((4, ld), dtype=torch.float32, device="cuda")
    _lib.call("zl_fp8_quant_per_token_group", ops.ctypes.c_void_p(xd.data_ptr()), 768, ops._p(q), ops._p(s), ld, 6, 512,
              0, 0, ops._stream())
    rq, rs = fb.quant_per_token_group(x[:, 256:768])
    np.testing.assert_array_equal(q.cpu().numpy(), rq)
    np.testing.assert_array_equal(s.cpu().numpy()[:, :6], rs[:, :6])


def _gen(out_dir, lib_path):
    r = subprocess.run([sys.executable, "-m", "tests.fp8_block_golden", out_dir, lib_path], cwd=ROOT, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return np.load(os.path.join(out_dir, "fp8_block_ref.npz"))


def test_quant_matches_reference_fixture(lib, cuda):
    """The committed outputs of the reference's own kernel (tests/golden/fp8_block_ref.npz), bit for bit."""
    from tests import fp8_block_golden as fg
    from zhilight_b200 import ops
    with np.load(fg.FIXTURE) as g:
        for name, tag, cm, key in fg.keys():
            if not cm:
                continue
            m = fg.SHAPES[name][0]
            q, s = ops.fp8_quant_per_token_group(_dev(fg.case_input(name, tag), tag))
            np.testing.assert_array_equal(q.cpu().numpy(), g[key + "_q"], err_msg=key)
            np.testing.assert_array_equal(s.cpu().numpy()[:, :m], g[key + "_s"][:, :m], err_msg=key)


def test_quant_matches_reference_kernel(lib, cuda, tmp_path):
    """The reference's KERNEL_per_token_cast_to_fp8 run here (oracle/_ref/libzl_ref_fp8.so) against the oracle."""
    if not os.path.exists(REF_FP8):
        pytest.skip("oracle/_ref/libzl_ref_fp8.so not built")
    from tests import fp8_block_golden as fg
    with _gen(str(tmp_path), REF_FP8) as g:
        assert fg.check(g) == len(fg.keys())


def test_dropin_matches_reference_and_c_abi(lib, cuda, tmp_path):
    """integration/zl_nn_dropin.cpp: per_token_cast_to_fp8 gives the reference kernel's codes and scales in both scale
    layouts, and deep_gemm_fp8_block_h20_group gives zl_fp8_block_gemm's output on the same operands (bit for bit: the
    same kernel); its grouped form returns -1 (checked inside the generator)."""
    if not (os.path.exists(REF_FP8) and os.path.exists(DROPIN_FP8)):
        pytest.skip("oracle/_ref/libzl_ref_fp8.so / libzl_dropin_fp8.so not built")
    from tests import fp8_block_golden as fg
    from zhilight_b200 import ops
    with _gen(str(tmp_path / "ref"), REF_FP8) as a, _gen(str(tmp_path / "dropin"), DROPIN_FP8) as b:
        for _, _, _, key in fg.keys():
            for sfx in ("_q", "_s"):
                np.testing.assert_array_equal(a[key + sfx], b[key + sfx], err_msg=key + sfx)
        for name in fg.GEMM_CASES:
            xq, sx, wq, sw = (torch.from_numpy(t).cuda() for t in fg.gemm_operands(name))
            y = _host(ops.fp8_block_gemm(xq, sx, wq, sw, torch.bfloat16))
            np.testing.assert_array_equal(b["y_" + name], y, err_msg=name)


# every M boundary (mma.sync up to 32, wgmma passes of 32/64/128 tokens, 256-row chunks) at one K/N, and every K x N
# (K = 128 is a single block; N = 4160 ends in a partial 64-row scale row) at M on each side of the route switch
GEMM_CASES = ([(m, 4096, 4160, "f16") for m in (1, 2, 16, 31, 32, 33, 64, 255, 256, 257, 600)]
              + [(m, 4096, 4160, "bf16") for m in (1, 32, 33, 257)]
              + [(m, k, n, t) for m in (1, 33, 257) for k in (128, 14336) for n in (128, 4160, 6144)
                 for t in ("f16", "bf16")]
              + [(2, 4096, 128, "bf16"), (600, 4096, 6144, "bf16"), (8, 4096, 6144, "f16")])


@pytest.mark.parametrize("m,k,n,tag", GEMM_CASES)
def test_block_gemm_matches_float64_oracle(lib, cuda, m, k, n, tag):
    from zhilight_b200 import ops
    rng = np.random.default_rng(m * 7 + k + n)
    x = _x(m, k, tag, seed=m + 2 * k + n)
    xq, sx = fb.quant_per_token_group(x)
    wq, sw = fb.random_weight(n, k, rng)
    y = ops.fp8_block_gemm(torch.from_numpy(xq).cuda(), torch.from_numpy(sx).cuda(), torch.from_numpy(wq).cuda(),
                           torch.from_numpy(sw).cuda(), DT[tag])
    ref = fb.block_gemm(xq, sx, wq, sw)
    out = _host(y)
    assert np.isfinite(out).all()
    assert rel_l2(out, ref) <= 2e-3, rel_l2(out, ref)


@pytest.mark.parametrize("tag", ["f16", "bf16"])
@pytest.mark.parametrize("m", [1, 40])
def test_layers_linear_matches_oracle(lib, cuda, tag, m):
    from zhilight_b200 import layers
    rng = np.random.default_rng(m)
    n, k = 4160, 1024
    wq, sw = fb.random_weight(n, k, rng)
    lin = layers.Linear(k, n, quant=10, dtype={"f16": "half", "bf16": "bfloat16"}[tag])
    lin.load_state_dict({"weight": torch.from_numpy(wq).view(torch.float8_e4m3fn),
                         "weight_scale_inv": torch.from_numpy(sw)})
    x = _x(m, k, tag, seed=m)
    y = lin(_dev(x, tag).reshape(1, m, k))
    assert y.shape == (1, m, n)
    assert rel_l2(_host(y.reshape(m, n)), fb.linear(x, wq, sw)) <= 2e-3


def test_layers_linear_rejects_bias_and_bad_scales(lib, cuda):
    from zhilight_b200 import _lib, layers
    rng = np.random.default_rng(0)
    wq, sw = fb.random_weight(256, 256, rng)
    w = torch.from_numpy(wq)
    with pytest.raises(_lib.ZLError):
        layers.Linear(256, 256, quant=10).load_state_dict({"weight": w, "weight_scale_inv": torch.from_numpy(sw),
                                                           "bias": torch.zeros(256)})
    with pytest.raises(_lib.ZLError):
        layers.Linear(256, 256, quant=10).load_state_dict({"weight": w, "weight_scale_inv": torch.from_numpy(sw[:1])})
    with pytest.raises(_lib.ZLError):
        layers.Linear(256, 256, quant=10).load_state_dict({"weight": w, "weight_scale_inv": torch.from_numpy(sw).half()})


# ------------------------------------------------------------------ decode driver
LINEARS = ("attn.project_q", "attn.project_k", "attn.project_v", "attn.attn_out", "ff.w_in", "ff.w_gated", "ff.w_out")


def make_state_dict(cfg, seed=0, dtype="f16"):
    """make_state_dict's dense checkpoint with every layer Linear replaced by e4m3 codes (exponent MSB cleared like the
    type-7 checkpoints: |w| < 2) and weight_scale_inv drawn log-uniformly over 0.0075 .. 0.12."""
    sd = omodel.make_state_dict(cfg, 0, seed=seed, dtype=dtype)
    rng = np.random.default_rng(seed + 17)
    for l in range(cfg["num_layers"]):
        for name in LINEARS:
            p = "layers.%d.%s" % (l, name)
            n, k = sd[p + ".weight"].shape
            wq, sw = fb.random_weight(n, k, rng, 0.0075, 0.12)
            sd[p + ".weight"] = wq & np.uint8(0xBF)
            sd[p + ".weight_scale_inv"] = sw
    return sd


class _BlockLinear:
    def _linear(self, x, prefix):
        cache = self.__dict__.setdefault("_wv", {})
        if prefix not in cache:
            cache[prefix] = oops.e4m3_decode(self.sd[prefix + ".weight"])
        y = fb.linear(np.asarray(x, F32), self.sd[prefix + ".weight"], self.sd[prefix + ".weight_scale_inv"],
                      cache[prefix])
        return oops._t(y.astype(F32), self.dtype)


class BlockOracle(_BlockLinear, omodel.OracleLlama):
    pass


class BlockKv8Oracle(_BlockLinear, Kv8OracleLlama):
    pass


def _decoder(cfg, dtype, sd, **kw):
    from zhilight_b200.llama import LlamaDecoder
    dec = LlamaDecoder(quant_type=10, dtype=dtype, **cfg, **kw)
    dec.load_state_dict(sd)
    return dec


@pytest.mark.parametrize("cfg,dtype,tol", [(TINY, "f16", 6e-3), (TINY, "bf16", 2e-2), (TINY128, "f16", 6e-3)],
                         ids=["tiny-f16", "tiny-bf16", "tiny128-f16"])
def test_decode_matches_oracle(lib, cuda, cfg, dtype, tol):
    sd = make_state_dict(cfg, seed=1, dtype=dtype)
    dec = _decoder(cfg, dtype, sd, max_batch=3, max_seq=64)
    orc = BlockOracle(cfg, sd, 0, 128, False, dtype)
    rng = np.random.default_rng(0)
    pos = np.zeros(3, np.int32)
    tok = rng.integers(0, cfg["vocab_size"], size=3).astype(np.int32)
    for s in range(4):
        b = 3 if s % 3 != 2 else 2
        nxt, logits = dec.decode(tok[:b], pos[:b], want_logits=True)
        ref = orc.decode(tok[:b], pos[:b], tasks=list(range(b)))
        assert np.isfinite(logits).all()
        assert rel_l2(logits, ref) <= tol, (s, rel_l2(logits, ref))
        tok[:b] = rng.integers(0, cfg["vocab_size"], size=b)
        pos[:b] += 1
    dec.close()


# TINY128 in chunks of 64: 5.2e-2 on the prefill logits, growing to 6.6e-2 over the decode steps that follow (H100).
# The per-tensor FP8 model (QuantType 7) runs the same comparison at the same bounds: its spread is of the same size.
@pytest.mark.parametrize("quant", [10, 7])
@pytest.mark.parametrize("cfg,chunk,tol", [(TINY, 32, 6e-2), (TINY128, 64, 1e-1)], ids=["tiny-32", "tiny128-64"])
def test_chunked_prefill_matches_oracle(lib, cuda, cfg, chunk, tol, quant):
    if quant == 10:
        sd = make_state_dict(cfg, seed=2)
        orc = BlockOracle(cfg, sd, 0, 128, False, "f16")
    else:
        sd = omodel.make_state_dict(cfg, 7, seed=2)
        orc = omodel.OracleLlama(cfg, sd, 7, 128, False, "f16")
    from zhilight_b200.llama import LlamaDecoder
    dec = LlamaDecoder(quant_type=quant, dtype="f16", max_batch=2, max_seq=128, prefill_chunk=chunk, **cfg)
    dec.load_state_dict(sd)
    rng = np.random.default_rng(4)
    prompt = rng.integers(0, cfg["vocab_size"], size=70).astype(np.int32)
    _, lg = dec.prefill(0, prompt, want_logits=True)
    for p, t in enumerate(prompt):
        r = orc.decode(np.array([t]), [p], tasks=[0])
    assert rel_l2(lg, r) <= tol
    tok = np.array([int(np.argmax(r[0]))], np.int32)
    pos = np.array([len(prompt)], np.int32)
    for _ in range(2):
        nxt, logits = dec.decode(tok, pos, want_logits=True)
        ref = orc.decode(tok, pos, tasks=[0])
        assert rel_l2(logits, ref) <= tol
        tok = np.argmax(ref, axis=1).astype(np.int32)
        pos += 1
    dec.close()


def test_joined_steps_match_oracle(lib, cuda):
    """Tasks 0-1 decode while task 2's prompt runs in the same joined steps."""
    cfg = TINY
    sd = make_state_dict(cfg, seed=3)
    dec = _decoder(cfg, "f16", sd, max_batch=4, max_seq=128, prefill_chunk=48)
    orc = BlockOracle(cfg, sd, 0, 128, False, "f16")
    rng = np.random.default_rng(5)
    V, tol = cfg["vocab_size"], 6e-2
    pos = np.zeros(3, np.int32)
    for t, n in enumerate((5, 9)):
        prompt = rng.integers(0, V, n).astype(np.int32)
        dec.prefill(t, prompt)
        for p, x in enumerate(prompt):
            orc.decode(prompt[p:p + 1], [p], tasks=[t])
        pos[t] = n
    prompt2 = rng.integers(0, V, 40).astype(np.int32)
    off = 0
    for i, cn in enumerate((32, 8)):
        last = i == 1
        tok = rng.integers(0, V, 2).astype(np.int32)
        segs = [(t, tok[t:t + 1], int(pos[t]), True) for t in range(2)] + [(2, prompt2[off:off + cn], off, last)]
        nxt, logits = dec.step_joined(segs, want_logits=True)
        ref = orc.decode(tok, pos[:2], tasks=[0, 1])
        for p in range(off, off + cn):
            r2 = orc.decode(prompt2[p:p + 1], [p], tasks=[2])
        assert rel_l2(logits[:2], ref) <= tol, i
        if last:
            assert rel_l2(logits[2], r2[0]) <= tol
        pos[:2] += 1
        off += cn
    dec.close()


def test_int8_kv_cache_decode_matches_oracle(lib, cuda):
    cfg = TINY
    sd = make_state_dict(cfg, seed=4)
    dec = _decoder(cfg, "f16", sd, max_batch=3, max_seq=64, kv_cache_dtype="int8")
    orc = BlockKv8Oracle(cfg, sd, 0, 128, False, "f16")
    rng = np.random.default_rng(1)
    pos = np.zeros(3, np.int32)
    tok = rng.integers(0, cfg["vocab_size"], size=3).astype(np.int32)
    for s in range(8):
        nxt, logits = dec.decode(tok, pos, want_logits=True)
        ref = orc.decode(tok, pos, tasks=[0, 1, 2])
        assert np.isfinite(logits).all()
        assert rel_l2(logits, ref) <= 6e-2, (s, rel_l2(logits, ref))
        tok = rng.integers(0, cfg["vocab_size"], size=3).astype(np.int32)
        pos += 1
    dec.close()


def test_llama8b_layers_decode_and_prefill(lib, cuda):
    """Three 8B-shaped layers (qkv 6144, o 4096, gate/up 2 x 14336, down K = 14336) at batch 1 and 8 and a 20-token
    prefill, against the oracle model."""
    cfg = LAYER8B
    sd = make_state_dict(cfg, seed=5)
    # 8B widths: smaller block scales keep fp16 activations finite through three layers
    for name in list(sd):
        if name.endswith(".weight_scale_inv"):
            sd[name] = (sd[name] * F32(0.25)).astype(F32)
    dec = _decoder(cfg, "f16", sd, max_batch=8, max_seq=64, prefill_chunk=48)
    orc = BlockOracle(cfg, sd, 0, 128, False, "f16")
    rng = np.random.default_rng(6)
    prompt = rng.integers(0, cfg["vocab_size"], size=20).astype(np.int32)
    _, lg = dec.prefill(0, prompt, want_logits=True)
    for p, t in enumerate(prompt):
        r = orc.decode(prompt[p:p + 1], [p], tasks=[0])
    assert np.isfinite(lg).all() and rel_l2(lg, r) <= 6e-2, rel_l2(lg, r)
    tok = rng.integers(0, cfg["vocab_size"], size=8).astype(np.int32)
    pos = np.array([20] + [0] * 7, np.int32)
    for b in (1, 8):
        nxt, logits = dec.decode(tok[:b], pos[:b], want_logits=True)
        ref = orc.decode(tok[:b], pos[:b], tasks=list(range(b)))
        assert np.isfinite(logits).all() and rel_l2(logits, ref) <= 6e-2, (b, rel_l2(logits, ref))
        pos[:b] += 1
    dec.close()


def test_synthetic_type10_model_runs(lib, cuda):
    from zhilight_b200.llama import LlamaDecoder
    dec = LlamaDecoder(quant_type=10, dtype="f16", max_batch=2, max_seq=32, **TINY128)
    dec.init_synthetic(3)
    nxt, logits = dec.decode(np.array([1, 2], np.int32), np.array([0, 0], np.int32), want_logits=True)
    assert np.isfinite(logits).all() and logits.std() > 0
    dec.close()


def test_driver_refuses_fp8_block_bias(lib, cuda):
    from zhilight_b200 import _lib
    sd = make_state_dict(TINY, seed=6)
    sd["layers.0.attn.project_q.bias"] = np.zeros(256, np.float16)
    from zhilight_b200.llama import LlamaDecoder
    dec = LlamaDecoder(quant_type=10, dtype="f16", max_batch=2, max_seq=32, **TINY)
    with pytest.raises(_lib.ZLError) as e:
        dec.load_state_dict(sd)
    assert e.value.code == -2
    dec.close()
