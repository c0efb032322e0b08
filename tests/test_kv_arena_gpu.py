"""GPU checks of the KV arena (kv_rows > 0): a serving scenario gives the same tokens, logits and KV rows bit for bit as
the fixed layout while tasks grow, move and compact; a full arena refuses with nothing enqueued and serves the same
call after a release; k_kv_relocate on its own matches numpy; and a model whose fixed layout would not fit on the card
allocates about kv_rows rows and runs."""
import ctypes

import numpy as np
import pytest

from oracle import model as omodel
from tests.test_llama_gpu import TINY, TINY128

pytestmark = pytest.mark.gpu


def _decoder(cfg, quant, dtype="f16", kv=None, kv_rows=None, max_batch=4, max_seq=256, chunk=32, **kw):
    from zhilight_b200.llama import LlamaDecoder
    dec = LlamaDecoder(quant_type=quant, dtype=dtype, max_batch=max_batch, max_seq=max_seq, prefill_chunk=chunk,
                       kv_cache_dtype=kv, kv_rows=kv_rows, **cfg, **kw)
    dec.load_state_dict(omodel.make_state_dict(cfg, quant, 128, False, seed=3, dtype=dtype))
    return dec


def _scenario(dec, vocab, joined):
    """prefill, decode, set_state + step_device, releases, a prompt that grows past its neighbours (a compaction with
    kv_rows = 384), re-prefills, a joined step, generate with stops, the step graph replayed after the moves, a prefix
    cache save and load, and a beam search.  -> every output and the KV rows every task wrote."""
    rng = np.random.default_rng(11)
    toks = lambda n: rng.integers(0, vocab, n).astype(np.int32)
    out, written = [], {}
    dec.enable_prefix_cache(16, 16)
    for t, n in ((0, 50), (1, 60), (2, 30)):
        out.append(dec.prefill(t, toks(n), want_logits=True))
        written[t] = n
    prompt3 = toks(40)
    out.append(dec.prefill_cached(3, prompt3, want_logits=True))
    written[3] = 40
    pos = np.array([50, 60, 30, 40], np.int32)
    nxt, lg = dec.decode(toks(4), pos, want_logits=True)
    out += [nxt, lg]
    dec.set_state(nxt, pos + 1)
    for _ in range(3):
        dec.step_device(4)
    t_, p_ = dec.get_state(4)
    out += [t_, p_, dec.get_logits(4)]
    written = {t: int(p_[t]) for t in range(4)}
    for t in (0, 2):
        dec.kv_release(t)
        written.pop(t)
    # task 1 grows from 64 to 192 rows: neither in place nor in a free extent, so the arena compacts
    out.append(dec.prefill(1, toks(100), pos0=int(p_[1]), want_logits=True))
    written[1] = int(p_[1]) + 100
    out.append(dec.prefill(0, toks(40), want_logits=True))
    written[0] = 40
    if joined:
        nj, lj = dec.step_joined([(2, toks(16), 0, True), (0, toks(1), 40, True)], want_logits=True)
        out += [nj, lj]
        t0 = int(nj[1])
    else:
        out.append(dec.prefill(2, toks(16), want_logits=True))
        out.append(dec.prefill(0, toks(1), pos0=40, want_logits=True))
        t0 = out[-1][0]
    written[0], written[2] = 41, 16
    tok = np.array([t0, 7, 9, 11], np.int32)
    dec.set_state(tok, np.array([41, written[1], 16, 40], np.int32))
    for t in range(4):
        dec.set_stop(t, stop_ids=[int(tok[t])], max_new_tokens=18)
    gen, fin, steps = dec.generate(4, 20)
    out += gen + [fin, np.array([steps])]
    t_, p_ = dec.get_state(4)
    dec.set_state(t_, np.minimum(p_, 255))
    for _ in range(2):
        dec.step_device(4)   # the B = 4 step graph, captured before the moves
    t_, p_ = dec.get_state(4)
    out += [t_, p_, dec.get_logits(4)]
    written = {t: int(p_[t]) for t in range(4)}
    res = dec.beam_search([toks(5)], beam_width=2, max_new_tokens=4, eos_id=int(tok[0]))
    out += [np.array(r[0]) for r in res[0]] + [np.array([r[1] for r in res[0]])]
    written[0] = written[1] = 5   # the beams' prompt rows are the same in both layouts; later rows depend on forks
    out.append(dec.prefill_cached(2, prompt3, want_logits=True))   # loads task 3's two cached blocks into task 2
    written[2] = 40
    rows = []
    for t, n in sorted(written.items()):
        for l in range(dec.cfg.num_layers):
            rows += list(dec.read_kv(l, t, 0, n))
    return out, rows


def _flatten(x):
    if isinstance(x, tuple):
        return [a for y in x for a in _flatten(y)]
    return [np.atleast_1d(np.ascontiguousarray(x))]


CASES = [
    ("gptq-d64", TINY, 5, "f16", None),
    ("gptq-d128", TINY128, 5, "f16", None),
    ("dense-bf16", TINY, 0, "bf16", None),
    ("w8a8", TINY, 2, "f16", None),
    ("kv8", TINY128, 5, "f16", "int8"),
]


@pytest.mark.parametrize("name,cfg,quant,dtype,kv", CASES, ids=[c[0] for c in CASES])
def test_arena_matches_fixed_layout(lib, cuda, name, cfg, quant, dtype, kv):
    runs = []
    for kv_rows in (None, 384):
        dec = _decoder(cfg, quant, dtype, kv, kv_rows)
        runs.append(_scenario(dec, cfg["vocab_size"], joined=kv is None))
        if kv_rows:
            assert dec.kv_free_rows() >= 0 and all(dec.kv_capacity(t) % 64 == 0 for t in range(4))
        dec.close()
    (o0, r0), (o1, r1) = runs
    f0 = [a for x in o0 for a in _flatten(x)]
    f1 = [a for x in o1 for a in _flatten(x)]
    assert len(f0) == len(f1)
    for i, (a, b) in enumerate(zip(f0, f1)):
        assert a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8)), ("output", i)
    assert len(r0) == len(r1)
    for i, (a, b) in enumerate(zip(r0, r1)):
        assert np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8)), i


def test_full_arena_refuses_then_serves_after_release(lib, cuda):
    from zhilight_b200 import _lib
    from zhilight_b200.llama import KV_FULL
    rng = np.random.default_rng(5)
    prompts = [rng.integers(0, TINY["vocab_size"], 60).astype(np.int32) for _ in range(3)]

    def run(dec, with_release):
        first = [dec.prefill(t, prompts[t]) for t in range(3)]
        dec.set_state(np.array(first[:2], np.int32), np.array([60, 60], np.int32))
        if with_release:
            free = dec.kv_free_rows()
            with pytest.raises(_lib.ZLError) as e:
                dec.generate(2, 40)   # both tasks need 128 rows: 64 more each, with 64 free
            assert e.value.code == KV_FULL
            assert dec.kv_free_rows() == free and dec.kv_capacity(0) == 64 and dec.kv_capacity(1) == 64
            t_, p_ = dec.get_state(2)
            np.testing.assert_array_equal(p_, [60, 60])
            dec.kv_release(2)
        return dec.generate(2, 40)

    outs = []
    for kv_rows, rel in ((None, False), (256, True)):
        dec = _decoder(TINY, 5, kv_rows=kv_rows, max_batch=3, max_seq=128)
        outs.append(run(dec, rel))
        dec.close()
    (g0, f0, s0), (g1, f1, s1) = outs
    assert s0 == s1 and np.array_equal(f0, f1) and all(np.array_equal(a, b) for a, b in zip(g0, g1))


def _relocate(bases, layers, moves, max_rows, row_bytes, srow_bytes):
    import torch
    from zhilight_b200 import _lib
    dev = torch.device("cuda:0")
    tab = torch.tensor([b.data_ptr() if b is not None else 0 for b in bases], dtype=torch.int64, device=dev)
    mv = torch.from_numpy(np.ascontiguousarray(moves, np.int32)).to(dev)
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(_lib.load().zl_kv_relocate(ctypes.c_void_p(tab.data_ptr()), layers, ctypes.c_void_p(mv.data_ptr()),
                                          len(moves), max_rows, row_bytes, srow_bytes, ctypes.c_void_p(st)))
    torch.cuda.synchronize()


def _random_moves(rng, rows, n):
    """n moves over disjoint segments of the row space: every source and destination apart from every other"""
    cuts = np.sort(rng.choice(np.arange(1, rows), 2 * n - 1, replace=False))
    seg = np.diff(np.concatenate([[0], cuts, [rows]]))
    start = np.concatenate([[0], cuts])
    order = rng.permutation(2 * n)
    moves = []
    for i in range(n):
        a, b = order[2 * i], order[2 * i + 1]
        length = int(min(seg[a], seg[b]))
        copy = int(rng.integers(0, length + 1))
        moves.append((int(start[a]), int(start[b]), copy, length - copy))
    return np.array(moves, np.int32)


@pytest.mark.parametrize("kind", ["f16", "bf16", "int8"])
@pytest.mark.parametrize("n", [1, 3, 17])
def test_relocate_matches_numpy(cuda, kind, n):
    import torch
    rng = np.random.default_rng(n * 7 + len(kind))
    layers, hkv, d, rows = 2, 3, 64, 12000
    vb = 1 if kind == "int8" else 2
    row_bytes, srow_bytes = hkv * d * vb, (hkv * 4 if kind == "int8" else 0)
    moves = _random_moves(rng, rows, n)
    if n == 1:
        moves = np.array([[0, 6000, 5999, 1]], np.int32)      # thousands of rows, a one-row tail
    if n == 3:
        moves[0] = (11998, 11999, 1, 0)                          # single rows
        moves[1] = (0, 5000, 1, 3999)
        moves[2] = (9000, 10000, 1000, 0)
    host = [rng.integers(0, 256, (rows, b), dtype=np.uint8) if b else None
            for b in (row_bytes, row_bytes, srow_bytes, srow_bytes)]
    bufs, want = [], []
    for l in range(layers):
        for t in range(4):
            h = host[t]
            if h is None:
                bufs.append(None)
                want.append(None)
                continue
            h = (h + l).astype(np.uint8)
            bufs.append(torch.from_numpy(h.copy()).cuda())
            w = h.copy()
            for s, dst, c, z in moves:
                w[dst:dst + c] = h[s:s + c]
                w[dst + c:dst + c + z] = 0
            want.append(w)
    max_rows = int((moves[:, 2] + moves[:, 3]).max())
    _relocate(bufs, layers, moves, max_rows, row_bytes, srow_bytes)
    for b, w in zip(bufs, want):
        if b is not None:
            assert np.array_equal(b.cpu().numpy(), w)


def test_capacity_beyond_the_fixed_layout(lib, cuda):
    """max_batch * max_seq rows of every layer would need ~137 GB; an arena of 4 x 64K rows allocates ~0.5 GB of KV and
    serves tasks of live rows that fit it."""
    import torch
    cfg = dict(TINY, num_layers=4)
    max_batch, max_seq, kv_rows = 1024, 65536, 4 * 65536
    row = cfg["num_layers"] * 2 * cfg["num_kv_heads"] * cfg["dim_head"] * 2   # bytes of one row over layers, K and V
    assert max_batch * max_seq * row > 100e9
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    dec = _decoder(cfg, 5, kv_rows=kv_rows, max_batch=max_batch, max_seq=max_seq, chunk=128)
    dec.sync()
    used = free0 - torch.cuda.mem_get_info()[0]
    assert kv_rows * row <= used <= kv_rows * row + (3 << 30), (used, kv_rows * row)
    rng = np.random.default_rng(2)
    first = [dec.prefill(t, rng.integers(0, cfg["vocab_size"], 128).astype(np.int32)) for t in range(8)]
    dec.set_state(np.array(first, np.int32), np.full(8, 128, np.int32))
    gen, fin, steps = dec.generate(8, 64)
    assert steps == 64 and all(len(g) == 64 for g in gen)
    assert all(dec.kv_capacity(t) >= 192 for t in range(8)) and dec.kv_capacity(8) == 0
    dec.close()
