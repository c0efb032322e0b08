"""int8 KV cache in the decode driver (LlamaDecoder(kv_cache_dtype="int8")): the cache bytes, the logits against the int8
oracle, and the invariances of the step (graph, PDL, host / device stepping, chunking, the dual-stream prefill,
continuous batching)."""
import os

import numpy as np
import pytest

from oracle import model as omodel
from tests.helpers import rel_l2
from tests.kv8_oracle import Kv8OracleLlama, quant_rows

pytestmark = pytest.mark.gpu

TINY = dict(num_layers=2, dim_model=256, num_heads=4, num_kv_heads=2, dim_head=64, dim_ff=512, vocab_size=512,
            eps=1e-5, rope_theta=10000.0, rope_llama3=None)
TINY128 = dict(num_layers=2, dim_model=512, num_heads=4, num_kv_heads=1, dim_head=128, dim_ff=640, vocab_size=1000,
               eps=1e-5, rope_theta=500000.0, rope_llama3=dict(factor=8.0, low=1.0, high=4.0, orig=8192.0))


def _decoder(sd, cfg, quant, kv8, **kw):
    from zhilight_b200.llama import LlamaDecoder
    dec = LlamaDecoder(quant_type=quant, group_size=128, kv_cache_dtype="int8" if kv8 else None, **kw, **cfg)
    dec.load_state_dict(sd)
    return dec


def _quant_rows_u8(rows):
    """zl_int8_quant_rows_u8 of fp16 (n, H_kv, d) rows -> uint8 codes (n, H_kv, d), fp32 scales (n, H_kv)."""
    import torch
    from zhilight_b200 import _lib
    n, hkv, d = rows.shape
    x = torch.from_numpy(np.ascontiguousarray(rows, np.float16)).cuda().reshape(n * hkv, d)
    q = torch.empty((n * hkv, d), dtype=torch.uint8, device="cuda")
    s = torch.empty((n * hkv,), dtype=torch.float32, device="cuda")
    _lib.call("zl_int8_quant_rows_u8", x.data_ptr(), q.data_ptr(), s.data_ptr(), n * hkv, d, 0, None)
    torch.cuda.synchronize()
    return q.cpu().numpy().reshape(n, hkv, d), s.cpu().numpy().reshape(n, hkv)


def _assert_cache_is_twin_quantised(dec8, dec16, layer, task, row0, row1):
    """Rows row0 .. row1 (all written) of the int8 model's cache == the fp16 twin's rows quantised."""
    k8, v8, sk, sv = dec8.read_kv(layer, task, row0, row1 - row0)
    k16, v16 = dec16.read_kv(layer, task, row0, row1 - row0)
    for codes, scales, rows in ((k8, sk, k16), (v8, sv, v16)):
        qc, qs = _quant_rows_u8(rows)
        np.testing.assert_array_equal(codes, qc)
        np.testing.assert_array_equal(scales, qs)
        oc, os_ = quant_rows(rows)            # the oracle's quantisation (pinned against the reference) agrees
        np.testing.assert_array_equal(codes, oc)
        np.testing.assert_array_equal(scales, os_)


# Layer 0's K / V rows depend only on the token and its position, so the int8 model's layer-0 cache must be exactly its
# fp16 twin's layer-0 cache quantised: any batch, any step, any fuse level, any GEMM route
@pytest.mark.parametrize("fuse", [0, 1, 2])
@pytest.mark.parametrize("batch", [1, 3, 17])
def test_layer0_cache_is_the_fp16_twin_quantised_gptq(lib, cuda, fuse, batch):
    sd = omodel.make_state_dict(TINY, 5, 128, False, seed=21)
    kw = dict(max_batch=batch, max_seq=64, fuse=fuse, prefill_chunk=32)
    dec8, dec16 = _decoder(sd, TINY, 5, True, **kw), _decoder(sd, TINY, 5, False, **kw)
    rng = np.random.default_rng(batch)
    prompt = rng.integers(0, TINY["vocab_size"], size=40).astype(np.int32)        # chunks of 32 (wgmma) and 8
    for dec in (dec8, dec16):
        dec.prefill(0, prompt)
    pos = np.full(batch, len(prompt), np.int32)
    pos[1:] = np.arange(batch - 1) % 5
    start = pos.copy()
    start[0] = 0
    for _ in range(3):
        tok = rng.integers(0, TINY["vocab_size"], size=batch).astype(np.int32)
        for dec in (dec8, dec16):
            dec.decode(tok, pos)
        pos += 1
    for task in range(batch):
        _assert_cache_is_twin_quantised(dec8, dec16, 0, task, int(start[task]), int(pos[task]))
    dec8.close()
    dec16.close()


@pytest.mark.parametrize("quant,cfg", [(6, TINY), (0, TINY), (2, TINY), (5, TINY128)], ids=["awq", "dense", "w8a8", "gptq-d128"])
def test_layer0_cache_is_the_fp16_twin_quantised_other_models(lib, cuda, quant, cfg):
    sd = omodel.make_state_dict(cfg, quant, 128, False, seed=22)
    kw = dict(max_batch=3, max_seq=64, fuse=2, prefill_chunk=16)
    dec8, dec16 = _decoder(sd, cfg, quant, True, **kw), _decoder(sd, cfg, quant, False, **kw)
    rng = np.random.default_rng(3)
    prompt = rng.integers(0, cfg["vocab_size"], size=20).astype(np.int32)
    for dec in (dec8, dec16):
        dec.prefill(2, prompt)
    pos = np.array([0, 4, len(prompt)], np.int32)
    start = np.array([0, 4, 0], np.int32)
    for _ in range(2):
        tok = rng.integers(0, cfg["vocab_size"], size=3).astype(np.int32)
        for dec in (dec8, dec16):
            dec.decode(tok, pos)
        pos += 1
    for task in range(3):
        _assert_cache_is_twin_quantised(dec8, dec16, 0, task, int(start[task]), int(pos[task]))
    dec8.close()
    dec16.close()


def _run(cfg, quant, sym=False, steps=16, fuse=2, seed=0, **kw):
    sd = omodel.make_state_dict(cfg, quant, 128, sym, seed=seed)
    dec = _decoder(sd, cfg, quant, True, sym=sym, max_batch=3, max_seq=64, fuse=fuse, **kw)
    orc = Kv8OracleLlama(cfg, sd, quant, 128, sym, "f16", fuse_norm=fuse >= 1)
    rng = np.random.default_rng(seed)
    pos = np.zeros(3, np.int32)
    tok = rng.integers(0, cfg["vocab_size"], size=3).astype(np.int32)
    outs = []   # (next tokens, logits, int8 oracle logits, input tokens) per step
    for s in range(steps):
        b = 3 if s % 3 != 2 else 2
        nxt, logits = dec.decode(tok[:b], pos[:b], want_logits=True)
        outs.append((nxt.copy(), logits.copy(), orc.decode(tok[:b], pos[:b], tasks=list(range(b))), tok[:b].copy()))
        tok[:b] = rng.integers(0, cfg["vocab_size"], size=b)
        pos[:b] += 1
    dec.close()
    return outs


@pytest.mark.parametrize("quant,sym,cfg,fuse,tol", [
    (5, False, TINY, 2, 1.5e-2), (5, True, TINY128, 2, 1.5e-2), (5, False, TINY128, 0, 1.5e-2), (6, False, TINY, 2, 1.5e-2),
    (0, False, TINY, 2, 1.5e-2), (2, False, TINY, 2, 4e-2)], ids=["gptq", "gptq-sym-d128", "gptq-fuse0", "awq", "dense", "w8a8"])
def test_decode_matches_int8_oracle(lib, cuda, quant, sym, cfg, fuse, tol):
    """Looser than the fp16-cache decode tests (2e-3; W8A8 6e-3), and why: one code step is 1/127 of its row's absmax,
    about 16 fp16 ulps, so the last-bit fp16 differences upstream that those tests accept move some layer >= 1 K / V code
    by one step (layer 0's codes are bit-exact, test above).  Measured on an H100 over 16 steps: up to 9.6e-3 (W8A8, whose
    per-token int8 activations flip the same way: 2.6e-2).  That is of the order of the oracle's own fp16-vs-int8 spread
    (1.2e-2 .. 2.2e-2, tests/test_kv8_cpu.py), so the bound alone cannot tell the caches apart; the W4 / dense logits
    must also be closer to the int8 oracle than to the fp16 one, by 1.5x on average over the steps (measured: 2.3x
    .. 2.9x on the first steps)."""
    sd = omodel.make_state_dict(cfg, quant, 128, sym, seed=0)
    orc16 = omodel.OracleLlama(cfg, sd, quant, 128, sym, "f16", fuse_norm=fuse >= 1)
    pos = np.zeros(3, np.int32)
    to8, to16 = [], []
    for nxt, logits, ref, tok in _run(cfg, quant, sym=sym, fuse=fuse):
        assert np.isfinite(logits).all()
        assert rel_l2(logits, ref) <= tol
        b = len(nxt)
        to8.append(rel_l2(logits, ref))
        to16.append(rel_l2(logits, orc16.decode(tok, pos[:b], tasks=list(range(b)))))
        pos[:b] += 1
    if quant != 2:
        assert 1.5 * np.mean(to8) < np.mean(to16), (to8, to16)


def test_graph_pdl_and_stepping_do_not_change_tokens(lib, cuda):
    runs = [_run(TINY, 5, steps=8, use_pdl=p, use_graph=g) for p, g in ((False, False), (True, False), (True, True))]
    for a, b, c in zip(*runs):
        np.testing.assert_array_equal(a[1], b[1])
        np.testing.assert_array_equal(a[1], c[1])
        np.testing.assert_array_equal(a[0], c[0])
    sd = omodel.make_state_dict(TINY, 5, 128, False, seed=3)
    finals = []
    for mode in ("host", "device"):
        dec = _decoder(sd, TINY, 5, True, max_batch=2, max_seq=64)
        tok, pos = np.array([7, 400], np.int32), np.array([0, 3], np.int32)
        if mode == "host":
            for _ in range(10):
                tok = dec.decode(tok, pos)
                pos = pos + 1
        else:
            dec.set_state(tok, pos)
            for _ in range(10):
                dec.step_device(2)
            tok, pos = dec.get_state(2)
        finals.append((tok.copy(), pos.copy(), dec.read_kv(1, 1, 0, 13)))
        dec.close()
    np.testing.assert_array_equal(finals[0][0], finals[1][0])
    for a, b in zip(finals[0][2], finals[1][2]):
        np.testing.assert_array_equal(a, b)


def test_long_context_crosses_attention_buckets(lib, cuda):
    sd = omodel.make_state_dict(TINY, 5, 128, False, seed=5)
    dec = _decoder(sd, TINY, 5, True, max_batch=1, max_seq=1200)
    orc = Kv8OracleLlama(TINY, sd, 5, 128, False, "f16", fuse_norm=True)
    rng = np.random.default_rng(0)
    toks = rng.integers(0, TINY["vocab_size"], size=1030).astype(np.int32)
    for p in range(1030):       # buckets 256 -> 512 -> 1024 -> 1200, and more than 1024 keys (two kv8 key splits at least)
        _, logits = dec.decode(toks[p:p + 1], np.array([p], np.int32), want_logits=True)
        ref = orc.decode(toks[p:p + 1], [p])
        if p in (0, 255, 256, 511, 512, 1023, 1024, 1029):
            assert rel_l2(logits, ref) <= 1.5e-2, p      # the decode bound of test_decode_matches_int8_oracle
    dec.close()


def test_chunked_prefill_chunk_16_against_2048(lib, cuda):
    sd = omodel.make_state_dict(TINY128, 5, 128, False, seed=9)
    prompt = np.random.default_rng(4).integers(0, TINY128["vocab_size"], size=70).astype(np.int32)
    res = []
    for chunk in (16, 2048):
        dec = _decoder(sd, TINY128, 5, True, max_batch=1, max_seq=128, prefill_chunk=chunk)
        _, logits = dec.prefill(0, prompt, want_logits=True)
        res.append((logits, dec.read_kv(0, 0, 0, len(prompt))))
        dec.close()
    # 16-token chunks run the exact-integer GEMM, one 70-token chunk the wgmma GEMM (weights rounded to fp16): the fp16
    # K / V rows can differ in their last bit, so a code may move by one step
    for a, b in zip(res[0][1][:2], res[1][1][:2]):
        assert np.abs(a.astype(np.int32) - b.astype(np.int32)).max() <= 1
        assert (a == b).mean() > 0.97
    orc = Kv8OracleLlama(TINY128, sd, 5, 128, False, "f16", fuse_norm=True)
    for p, t in enumerate(prompt):
        ref = orc.decode(np.array([t]), [p])
    # the fp16-cache chunked-prefill test allows 5e-3.  The one-step code flips of test_decode_matches_int8_oracle grow
    # with the wgmma GEMM's fp16-rounded weights (measured on an H100: up to 1.6e-2), which is as large as the oracle's
    # fp16-vs-int8 spread: this bound only catches gross errors.  The codes of the two chunkings are checked above, and
    # the prefill's cache bytes in test_layer0_cache_is_the_fp16_twin_quantised_*.
    for logits, _ in res:
        assert rel_l2(logits, ref) <= 2.5e-2
    assert rel_l2(res[0][0], res[1][0]) <= 2.5e-2


@pytest.mark.parametrize("cfg", [TINY128, TINY], ids=["d128", "d64"])
def test_dual_stream_prefill_matches_single_stream(lib, cuda, monkeypatch, cfg):
    sd = omodel.make_state_dict(cfg, 5, 128, False, seed=13)
    prompt = np.random.default_rng(6).integers(0, cfg["vocab_size"], size=84).astype(np.int32)
    outs = []
    for dual in ("0", "1"):
        monkeypatch.setenv("ZL_PREFILL_DUAL", dual)
        dec = _decoder(sd, cfg, 5, True, max_batch=1, max_seq=128, prefill_chunk=32)
        nxt, logits = dec.prefill(0, prompt, want_logits=True)
        steps = [logits.copy()]
        tok, pos = np.array([nxt], np.int32), np.array([len(prompt)], np.int32)
        for _ in range(3):
            tok, lg = dec.decode(tok, pos, want_logits=True)
            steps.append(lg.copy())
            pos = pos + 1
        dec.close()
        outs.append(steps)
    # M = 32 chunks (wgmma GEMM) against two M = 16 halves (exact-integer GEMM): the bound of the chunked-prefill test
    for a, b in zip(*outs):
        assert np.isfinite(a).all() and np.isfinite(b).all()
        assert rel_l2(b, a) <= 2.5e-2
    orc = Kv8OracleLlama(cfg, sd, 5, 128, False, "f16", fuse_norm=True)
    for p, t in enumerate(prompt):
        ref = orc.decode(np.array([t]), [p])
    assert rel_l2(outs[1][0], ref) <= 2.5e-2


def test_prefill_between_device_steps_leaves_other_tasks_untouched(lib, cuda):
    sd = omodel.make_state_dict(TINY, 5, 128, False, seed=17)
    dec = _decoder(sd, TINY, 5, True, max_batch=3, max_seq=64, prefill_chunk=16)
    dec.set_state(np.array([5, 9], np.int32), np.array([0, 2], np.int32))
    for _ in range(4):
        dec.step_device(2)
    dec.sync()
    before = [dec.read_kv(l, t, 0, 64) for l in range(2) for t in (0, 1)]
    dec.prefill(2, np.arange(30, dtype=np.int32) * 7 % TINY["vocab_size"])
    after = [dec.read_kv(l, t, 0, 64) for l in range(2) for t in (0, 1)]
    for a, b in zip(before, after):
        for x, y in zip(a, b):
            np.testing.assert_array_equal(x, y)
    assert dec.read_kv(0, 2, 0, 30)[2].min() > 0      # the prompt's rows were written (non-zero scales)
    dec.step_device(2)
    tok, pos = dec.get_state(2)
    np.testing.assert_array_equal(pos, [5, 7])
    dec.close()


def test_kv_allocation_is_about_half(lib, cuda):
    """Capacity: an int8 cache takes (d + 4) / (2 d) of the fp16 cache's bytes (codes + one fp32 scale per kv head)."""
    import torch
    cfg = dict(TINY128, num_layers=2)
    max_batch, max_seq = 4, 16384
    used = {}
    for kv8 in (False, True):
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        dec = _decoder(omodel.make_state_dict(cfg, 5, 128, False, seed=1), cfg, 5, kv8, max_batch=max_batch,
                       max_seq=max_seq)
        dec.sync()
        used[kv8] = free0 - torch.cuda.mem_get_info()[0]
        dec.close()
    d, hkv = cfg["dim_head"], cfg["num_kv_heads"]
    kv16 = 2 * cfg["num_layers"] * max_batch * max_seq * hkv * d * 2
    kv8_bytes = 2 * cfg["num_layers"] * max_batch * max_seq * hkv * (d + 4)
    assert kv8_bytes / kv16 == pytest.approx(0.516, abs=1e-3)
    # everything else is the same allocation in both models (plus a few KB of staging rows)
    assert abs((used[False] - used[True]) - (kv16 - kv8_bytes)) <= 8 << 20, (used, kv16, kv8_bytes)


def test_read_kv_checks_its_arguments(lib, cuda):
    from zhilight_b200 import _lib
    sd = omodel.make_state_dict(TINY, 5, 128, False, seed=1)
    dec = _decoder(sd, TINY, 5, False, max_batch=1, max_seq=16)
    buf = np.empty(16 * 2 * 64 * 4, np.uint8)
    p = buf.ctypes.data
    for args in ((2, 0, 0, 1, p, p, None, None), (0, 1, 0, 1, p, p, None, None), (0, 0, 10, 7, p, p, None, None),
                 (0, 0, 0, 1, p, p, p, None)):      # scales of a plain cache
        assert dec.lib.zl_llama_read_kv(dec.h, *args) == -1, args
    with pytest.raises(_lib.ZLError):
        dec.read_kv(0, 0, 0, 17)
    dec.close()
