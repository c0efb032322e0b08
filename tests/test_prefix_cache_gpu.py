"""GPU checks of the prompt prefix cache: KV blocks saved to the device pool and loaded into another task are the same
bits in every layer (codes and scales with an int8 cache); the prefill and decode steps that follow them give the same
logits bit for bit; prompts served from the cache stay within the prefill tolerance of the oracle model, the chained
keys included; and the pool's refusals, its LRU reuse, joined steps over loaded rows and the per-step launch count."""
import os
import socket

import numpy as np
import pytest

from oracle import model as omodel
from tests.helpers import rel_l2
from tests.test_llama_gpu import LAYER8B, TINY

pytestmark = pytest.mark.gpu

INVALID, STATE = -1, -4
BT = 16


def _decoder(quant=5, dtype="f16", fuse=2, kv=None, sym=False, max_seq=128, max_batch=2, chunk=32, seed=0, cfg=TINY,
             sd=None, **kw):
    from zhilight_b200.llama import LlamaDecoder
    dec = LlamaDecoder(quant_type=quant, dtype=dtype, fuse=fuse, sym=sym, max_batch=max_batch, max_seq=max_seq,
                       prefill_chunk=chunk, kv_cache_dtype=kv, **cfg, **kw)
    dec.load_state_dict(sd if sd is not None else omodel.make_state_dict(cfg, quant, 128, sym, seed=seed, dtype=dtype))
    return dec


def _oracle_prompt(orc, key, tokens):
    """the oracle's next-token logits after feeding `tokens` one at a time to a fresh task `key`"""
    for p, t in enumerate(tokens):
        r = orc.decode(np.array([t]), [p], tasks=[key])
    return r[0]


def _assert_same_rows(dec, layers, a, b, n):
    for l in range(layers):
        for x, y in zip(dec.read_kv(l, a, 0, n), dec.read_kv(l, b, 0, n)):
            assert np.array_equal(x, y), l


def _copy_then_compare(dec, layers, vocab, prefix_len, rest_len, seed, pool_blocks):
    """prefill task 0 with a prefix, save its blocks, load them into task 1: the rows, the prefill of the rest at
    pos0 = prefix_len and 8 decode steps after it are the same bits in both tasks"""
    rng = np.random.default_rng(seed)
    prefix = rng.integers(0, vocab, prefix_len).astype(np.int32)
    rest = rng.integers(0, vocab, rest_len).astype(np.int32)
    nb = prefix_len // dec.prefix_cache.block_tokens
    dec.prefill(0, prefix)
    dec.kv_save_blocks(0, range(nb), pool_blocks[:nb])
    dec.kv_load_blocks(1, range(nb), pool_blocks[:nb])
    _assert_same_rows(dec, layers, 0, 1, prefix_len)
    n0, l0 = dec.prefill(0, rest, pos0=prefix_len, want_logits=True)
    n1, l1 = dec.prefill(1, rest, pos0=prefix_len, want_logits=True)
    assert n0 == n1 and np.array_equal(l0, l1)
    tok = np.array([n0, n1], np.int32)
    pos = prefix_len + rest_len
    for _ in range(8):
        nxt, logits = dec.decode(tok, np.array([pos, pos], np.int32), want_logits=True)
        assert nxt[0] == nxt[1] and np.array_equal(logits[0], logits[1])
        tok = nxt
        pos += 1
    _assert_same_rows(dec, layers, 0, 1, pos)


KINDS = {
    "gptq-fuse2": dict(quant=5),
    "gptq-fuse0": dict(quant=5, fuse=0),
    "gptq-int8kv": dict(quant=5, kv="int8"),
    "bf16-dense": dict(quant=0, dtype="bf16"),
    "fp8": dict(quant=7),
}


@pytest.mark.parametrize("kind", list(KINDS))
def test_loaded_blocks_are_bit_exact(lib, cuda, kind):
    dec = _decoder(**KINDS[kind])
    dec.enable_prefix_cache(8, BT)
    # blocks land in scattered pool blocks; 48 + 21 rows: the rest starts on a block boundary mid-chunk
    _copy_then_compare(dec, TINY["num_layers"], TINY["vocab_size"], 3 * BT, 21, seed=1, pool_blocks=[5, 1, 3])
    dec.close()


def test_llama8b_layers_2048_token_prefix_bit_exact(lib, cuda):
    """three Llama-3.1-8B-shaped layers, 128-token blocks, a 2048-token prefix prefilled in chunks of 512"""
    from zhilight_b200.llama import LlamaDecoder
    dec = LlamaDecoder(quant_type=5, sym=True, max_batch=2, max_seq=2048 + 128, prefill_chunk=512, **LAYER8B)
    dec.init_synthetic(3)
    dec.enable_prefix_cache(20, 128)
    pool = list(range(19, 3, -1))
    _copy_then_compare(dec, LAYER8B["num_layers"], LAYER8B["vocab_size"], 2048, 40, seed=2, pool_blocks=pool)
    dec.close()


def test_cached_prompts_match_the_oracle(lib, cuda):
    """Prompts served through prefill_cached stay within the chunked-prefill tolerance of the oracle, and the chained
    keys never load B's rows computed after A into a prompt that has C before B."""
    sd = omodel.make_state_dict(TINY, 5, 128, False, seed=5)
    dec = _decoder(sd=sd)
    dec.enable_prefix_cache(16, BT)
    orc = omodel.OracleLlama(TINY, sd, 5, 128, False, "f16", fuse_norm=True)
    rng = np.random.default_rng(6)
    V = TINY["vocab_size"]
    blocks = {c: rng.integers(0, V, BT).astype(np.int32) for c in "ABC"}
    tail = lambda n: rng.integers(0, V, n).astype(np.int32)  # noqa: E731
    cat = lambda *xs: np.concatenate(xs)  # noqa: E731
    tol = 5e-3
    cases = [(0, cat(blocks["A"], blocks["B"], tail(7)), 0),         # cold: caches A and A/B
             (1, cat(blocks["A"], blocks["B"], tail(9)), 2 * BT),    # both blocks from the cache
             (0, cat(blocks["C"], tail(5)), 0),                      # caches C
             (1, cat(blocks["C"], blocks["B"], tail(6)), BT)]        # C only: B after A is not B after C
    for i, (task, prompt, want_cached) in enumerate(cases):
        nxt, cached, logits = dec.prefill_cached(task, prompt, want_logits=True)
        assert cached == want_cached, i
        ref = _oracle_prompt(orc, "p%d" % i, prompt)
        assert rel_l2(logits[0], ref) <= tol, i
        assert nxt == int(np.argmax(logits[0]))
        # decoding continues from the loaded + prefilled rows
        nxt2, l2 = dec.decode(np.array([nxt, nxt], np.int32)[:task + 1],
                              np.array([len(prompt)] * (task + 1), np.int32), want_logits=True)
        r2 = orc.decode(np.array([nxt]), [len(prompt)], tasks=["p%d" % i])
        assert rel_l2(l2[task], r2[0]) <= tol, i
    dec.close()


def test_small_pool_lru_reuse_stays_correct(lib, cuda):
    """A 3-block pool cycles through four two-block prefixes: blocks are evicted and rewritten, and every prompt served
    with a cached prefix gives the logits of a cold prefill on a model without a pool -- the same bits when both split
    the prompt alike (nothing or both stem blocks cached: the stem is exactly the first 32-row chunk)."""
    sd = omodel.make_state_dict(TINY, 5, 128, False, seed=7)
    dec = _decoder(sd=sd)
    dec.enable_prefix_cache(3, BT)
    ref = _decoder(sd=sd)
    rng = np.random.default_rng(8)
    V = TINY["vocab_size"]
    stems = [rng.integers(0, V, 2 * BT).astype(np.int32) for _ in range(4)]
    seen = []
    for i, s in enumerate([0, 0, 1, 1, 0, 2, 2, 3, 0, 3, 1, 1]):
        prompt = np.concatenate([stems[s], rng.integers(0, V, 3 + i % 5).astype(np.int32)])
        task = i % 2
        _, cached, logits = dec.prefill_cached(task, prompt, want_logits=True)
        _, cold = ref.prefill(task, prompt, want_logits=True)
        seen.append(cached)
        if cached in (0, 2 * BT):
            assert np.array_equal(logits, cold), i
        else:
            assert rel_l2(logits, cold) <= 5e-3, i
    # the policy's hits: full, partial (a stem's second block evicted) and none
    assert seen == [0, 32, 0, 32, 16, 0, 32, 0, 0, 16, 0, 32] and len(dec.prefix_cache) <= 3
    dec.close()
    ref.close()


def test_joined_step_over_loaded_rows(lib, cuda):
    """A joined step carries task 1's prompt from pos0 = its cached length beside task 0's decode row."""
    sd = omodel.make_state_dict(TINY, 5, 128, False, seed=9)
    dec = _decoder(sd=sd)
    dec.enable_prefix_cache(8, BT)
    orc = omodel.OracleLlama(TINY, sd, 5, 128, False, "f16", fuse_norm=True)
    rng = np.random.default_rng(10)
    V = TINY["vocab_size"]
    stem = rng.integers(0, V, 3 * BT).astype(np.int32)
    p0 = np.concatenate([stem, rng.integers(0, V, 4).astype(np.int32)])
    n0, cached = dec.prefill_cached(0, p0)
    assert cached == 0
    ref0 = _oracle_prompt(orc, 0, p0)
    p1 = np.concatenate([stem, rng.integers(0, V, 11).astype(np.int32)])
    hit = dec.prefix_cache.match(p1)
    m = len(hit) * BT
    assert m == 3 * BT
    dec.kv_load_blocks(1, range(len(hit)), hit)
    tok0 = int(np.argmax(ref0))
    nxt, logits = dec.step_joined([(0, np.array([tok0], np.int32), len(p0), True), (1, p1[m:], m, True)],
                                  want_logits=True)
    r0 = orc.decode(np.array([tok0]), [len(p0)], tasks=[0])
    r1 = _oracle_prompt(orc, 1, p1)
    assert rel_l2(logits[0], r0[0]) <= 5e-3 and rel_l2(logits[1], r1) <= 5e-3
    dec.close()


def test_pool_refusals(lib, cuda):
    from zhilight_b200 import _lib
    from zhilight_b200.llama import LlamaDecoder

    def code(fn, *a):
        with pytest.raises(_lib.ZLError) as e:
            fn(*a)
        return e.value.code

    raw = LlamaDecoder(quant_type=5, max_batch=2, max_seq=120, prefill_chunk=32, **TINY)   # not finalized
    assert code(raw.enable_prefix_cache, 4, BT) == STATE
    raw.close()
    dec = _decoder(max_seq=120)            # 120 rows: task blocks 0 .. 6 of 16
    assert code(dec.kv_save_blocks, 0, [0], [0]) == STATE          # no pool
    assert code(dec.kv_load_blocks, 0, [0], [0]) == STATE
    for bad_bt in (0, 8, 100, 512):
        assert code(dec.enable_prefix_cache, 4, bad_bt) == INVALID
    assert code(dec.enable_prefix_cache, 0, BT) == INVALID
    dec.enable_prefix_cache(4, BT)
    assert code(dec.enable_prefix_cache, 4, BT) == STATE            # created twice
    dec.prefill(0, np.arange(40, dtype=np.int32))
    for fn in (dec.kv_save_blocks, dec.kv_load_blocks):
        assert code(fn, -1, [0], [0]) == INVALID                    # task out of range
        assert code(fn, 2, [0], [0]) == INVALID
        assert code(fn, 0, [-1], [0]) == INVALID                    # task block out of range
        assert code(fn, 0, [7], [0]) == INVALID                     # (7 + 1) * 16 > max_seq
        assert code(fn, 0, [0], [4]) == INVALID                     # pool block out of range
        assert code(fn, 0, [0], [-1]) == INVALID
    assert code(dec.kv_save_blocks, 0, [0, 1], [2, 2]) == INVALID   # destination named twice
    assert code(dec.kv_load_blocks, 1, [3, 3], [0, 1]) == INVALID
    # a repeated source is fine, and nothing was enqueued by the refused calls
    dec.kv_save_blocks(0, [1, 1], [0, 3])
    dec.kv_load_blocks(1, [0, 6], [0, 0])
    k1 = dec.read_kv(0, 0, BT, BT)
    for blk in (0, 6):
        kb = dec.read_kv(0, 1, blk * BT, BT)
        assert all(np.array_equal(x, y) for x, y in zip(kb, k1))
    dec.close()


def test_pool_leaves_the_decode_step_unchanged(lib, cuda):
    """Kernels per decode step (graph nodes) and the decode logits are the same with a pool present and used."""
    sd = omodel.make_state_dict(TINY, 5, 128, False, seed=11)
    out = []
    for with_pool in (False, True):
        dec = _decoder(sd=sd)
        if with_pool:
            dec.enable_prefix_cache(4, BT)
        dec.prefill(0, np.arange(3, 40, dtype=np.int32))
        dec.prefill(1, np.arange(5, 30, dtype=np.int32))
        if with_pool:
            dec.kv_save_blocks(0, [0, 1], [2, 0])
            dec.kv_load_blocks(0, [0, 1], [2, 0])
        tok = np.array([7, 8], np.int32)
        for s in range(3):
            nxt, logits = dec.decode(tok, np.array([37 + s, 25 + s], np.int32), want_logits=True)
            tok = nxt
        out.append((dec.stats(2)[1], logits))
        dec.close()
    assert out[0][0] == out[1][0] > 0
    assert np.array_equal(out[0][1], out[1][1])


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _tp_worker(rank, ws, port, q):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=ws, device_id=torch.device("cuda", rank))
    res = {}
    try:
        from zhilight_b200 import dist as zdist
        from zhilight_b200.llama import LlamaDecoder
        sd = omodel.make_state_dict(TINY, 5, 128, False, seed=12)
        dec = LlamaDecoder(quant_type=5, max_batch=2, max_seq=96, tp_rank=rank, tp_size=ws, prefill_chunk=32, **TINY)
        comm = zdist.TPComm(32 * TINY["dim_model"], rank, ws)
        dec.set_comm(comm)
        dec.load_state_dict(zdist.shard_state_dict(sd, rank, ws))
        dec.enable_prefix_cache(6, BT)      # each rank: its own kv heads, the same decisions
        orc = omodel.OracleLlama(TINY, sd, 5, 128, False, "f16", fuse_norm=True)
        rng = np.random.default_rng(13)
        stem = rng.integers(0, TINY["vocab_size"], 2 * BT).astype(np.int32)
        vs = TINY["vocab_size"] // ws
        res["cached"], res["err"] = [], []
        for i, task in enumerate((0, 1)):
            prompt = np.concatenate([stem, rng.integers(0, TINY["vocab_size"], 6 + i).astype(np.int32)])
            _, cached, logits = dec.prefill_cached(task, prompt, want_logits=True)
            ref = _oracle_prompt(orc, i, prompt)
            res["cached"].append(cached)
            res["err"].append(float(rel_l2(logits[0], ref[rank * vs:(rank + 1) * vs])))
        dec.close()
        comm.close()
    except Exception:   # pragma: no cover
        import traceback
        res["error"] = traceback.format_exc()
    finally:
        q.put((rank, res))
        dist.destroy_process_group()


def test_tp2_ranks_cache_their_own_heads(lib, cuda):
    import torch
    ws = 2
    if torch.cuda.device_count() < ws:
        pytest.skip("needs %d GPUs" % ws)
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_tp_worker, args=(r, ws, port, q)) for r in range(ws)]
    for p in procs:
        p.start()
    results = dict(q.get(timeout=600) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    for r in range(ws):
        res = results[r]
        assert "error" not in res, res.get("error")
        assert res["cached"] == [0, 2 * BT], res
        assert max(res["err"]) <= 5e-3, res
