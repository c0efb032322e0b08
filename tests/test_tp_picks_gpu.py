"""Full-vocabulary picks under tensor parallelism: the vocabulary all-gather (zl_vocab_gather_*) on one GPU and, with
>= 2 GPUs on the box (skipped otherwise), between ranks, and a TP=2 decoder with enable_tp_picks whose sampled, processed,
beam and generate picks must equal the single-GPU operators over the concatenated logit shards, on every rank."""
import ctypes
import os
import socket

import numpy as np
import pytest

from oracle import model as omodel
from tests.test_llama_gpu import TINY

pytestmark = pytest.mark.gpu

INVALID, UNSUPPORTED, STATE = -1, -2, -4


def _rows(seed, T, V):
    """(T, V) fp32 rows with -inf entries, the same on every rank for a seed"""
    rng = np.random.default_rng(seed)
    full = (rng.standard_normal((T, V)) * 4).astype(np.float32)
    full[rng.random((T, V)) < 0.01] = -np.inf
    return full


def _bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.int32), np.ascontiguousarray(b).view(np.int32))


# ------------------------------------------------------------------------------------------------ one GPU
@pytest.mark.parametrize("V", [512, 128256])
def test_gather_one_rank_is_the_shard(lib, cuda, V):
    import torch
    from zhilight_b200.dist import VocabGather
    g = VocabGather(32, V, 0, 1)
    try:
        for T in (1, 3, 32):
            for epoch in range(4):
                full = _rows(1000 * T + epoch, T, V)
                if epoch == 1:   # a row stride past the shard's width
                    src = torch.zeros((T, V + 12), dtype=torch.float32, device=cuda)
                    src[:, :V] = torch.from_numpy(full).to(cuda)
                    shard = src[:, :V]
                else:
                    shard = torch.from_numpy(full).to(cuda)
                out = g.gather(shard)
                torch.cuda.synchronize()
                assert _bits_equal(out.cpu().numpy(), full), (T, epoch)
    finally:
        g.close()


def test_gather_refusals_enqueue_nothing(lib, cuda):
    import torch
    from zhilight_b200.dist import VocabGather
    h = ctypes.c_void_p()
    assert lib.zl_vocab_gather_create(0, 1, 4, 514, ctypes.byref(h)) == UNSUPPORTED        # vshard % 4
    assert lib.zl_vocab_gather_create(1, 2, 4, 516, ctypes.byref(h)) == UNSUPPORTED        # vshard 258
    assert lib.zl_vocab_gather_create(0, 3, 4, 512, ctypes.byref(h)) == INVALID            # V % ws
    assert lib.zl_vocab_gather_create(0, 1, 0, 512, ctypes.byref(h)) == INVALID            # rows
    assert lib.zl_vocab_gather_create(1, 1, 4, 512, ctypes.byref(h)) == INVALID            # rank
    g = VocabGather(4, 512, 0, 1)
    shard = torch.zeros((8, 520), dtype=torch.float32, device=cuda)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    lib.zl_launch_count(1)
    for rows, ld, ptr in [(0, 512, p(shard)), (5, 512, p(shard)), (-1, 512, p(shard)), (4, 508, p(shard)),
                          (4, 514, p(shard)), (4, 520, ctypes.c_void_p(shard.data_ptr() + 4)), (4, 520, None)]:
        assert lib.zl_vocab_allgather(g.handle, ptr, rows, ld, 0, s) == INVALID, (rows, ld)
    # a rank of two whose peers were never opened
    assert lib.zl_vocab_gather_create(0, 2, 4, 512, ctypes.byref(h)) == 0
    assert lib.zl_vocab_allgather(h, p(shard), 4, 256, 0, s) == STATE
    assert lib.zl_launch_count(0) == 0
    lib.zl_vocab_gather_destroy(h)
    g.close()


def test_set_vocab_gather_checks(lib, cuda):
    from zhilight_b200.dist import VocabGather
    from zhilight_b200.llama import LlamaDecoder
    sd = omodel.make_state_dict(TINY, 5, 128, False, seed=3)
    dec = LlamaDecoder(quant_type=5, max_batch=4, max_seq=32, **TINY)
    dec.load_state_dict(sd)
    want = dec.decode(np.array([1, 2, 3, 4], np.int32), np.zeros(4, np.int32))
    dec.enable_tp_picks()                                   # tp 1: nothing to gather
    assert getattr(dec, "_vgather", None) is None
    bad = [VocabGather(3, 512, 0, 1), VocabGather(4, 1024, 0, 1)]        # max_rows < max_batch, another vocabulary
    h = ctypes.c_void_p()
    assert lib.zl_vocab_gather_create(0, 2, 4, 512, ctypes.byref(h)) == 0   # world size 2 for a tp 1 model
    for g in bad:
        assert lib.zl_llama_set_vocab_gather(dec.h, g.handle) == INVALID
    assert lib.zl_llama_set_vocab_gather(dec.h, h) == INVALID
    ok = VocabGather(4, 512, 0, 1)
    assert lib.zl_llama_set_vocab_gather(dec.h, ok.handle) == 0
    np.testing.assert_array_equal(dec.decode(np.array([1, 2, 3, 4], np.int32), np.zeros(4, np.int32)), want)
    dec.close()
    for g in bad + [ok]:
        g.close()
    lib.zl_vocab_gather_destroy(h)


# ------------------------------------------------------------------------------------------------ two GPUs
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _device(rank):
    import torch
    return torch.device("cuda", rank)


SETTINGS = {
    "greedy": [{}] * 4,
    "t0.8": [dict(temperature=0.8, seed=11 + t) for t in range(4)],
    "top-k50": [dict(temperature=1.0, top_k=50, seed=21 + t) for t in range(4)],
    "top-p0.9": [dict(temperature=1.0, top_p=0.9, seed=31 + t) for t in range(4)],
    "penalties": [dict(temperature=0.8, repetition_penalty=1.3, seed=41), dict(temperature=0.8, presence_penalty=0.7, seed=42),
                  dict(repetition_penalty=1.5), dict(temperature=1.2, repetition_penalty=0.8, seed=44)],
    "ngram-bias": [dict(temperature=0.8, seed=51, ngram_penalty=1.3, logit_bias={7: 3.0, 11: -np.inf}),
                   dict(ngram_penalty=1.3), dict(temperature=1.0, seed=53, logit_bias={100: 5.0, 300: -2.5}),
                   dict(temperature=0.7, seed=54, ngram_penalty=1.3, repetition_penalty=1.1, logit_bias={1: 1.0})],
    "mixed": [{}, dict(temperature=0.8, top_p=0.95, top_k=50, seed=61), {}, dict(temperature=0.8, seed=63)],
}


def _allgather(obj):
    import torch.distributed as dist
    out = [None] * dist.get_world_size()
    dist.all_gather_object(out, obj)
    return out


def _set(dec, s):
    for t, p in enumerate(s):
        dec.set_sampling(t, **p)


def _oracle_state(dev, s, V, max_seq):
    """the driver's per-task pick state of zl_sample_processed, cleared as set_sampling clears it"""
    import torch
    from zhilight_b200.llama import logit_bias_arrays
    n = len(s)
    bt = np.zeros((n, 1024), np.int32)
    bv = np.zeros((n, 1024), np.float32)
    bc = np.zeros(n, np.int32)
    ng = np.zeros(n, np.float32)
    for t, p in enumerate(s):
        toks, vals = logit_bias_arrays(p.get("logit_bias"), V)
        bt[t, :toks.size], bv[t, :toks.size], bc[t] = toks, vals, toks.size
        ng[t] = 1.0 if p.get("presence_penalty") else p.get("ngram_penalty", 1.0)
    f = lambda a: torch.from_numpy(a).to(dev)
    params = [{k: v for k, v in p.items() if k not in ("ngram_penalty", "logit_bias")} for p in s]
    return dict(params=params, seq=torch.zeros((n, max_seq), dtype=torch.int32, device=dev),
                seq_len=torch.zeros(n, dtype=torch.int32, device=dev), ngram=f(ng), bt=f(bt), bv=f(bv), bc=f(bc),
                history=torch.zeros((n, (V + 31) // 32), dtype=torch.int32, device=dev))


def _oracle_pick(dev, st, full, pos):
    import torch
    from zhilight_b200 import ops
    out = ops.sample_processed(torch.from_numpy(full).to(dev), st["params"], st["seq"], st["seq_len"], st["ngram"], st["bt"],
                               st["bv"], st["bc"], None, torch.from_numpy(np.asarray(pos, np.int32)).to(dev),
                               st["history"])
    return out.cpu().numpy()


def _host_loop(dec, tok, pos, rules, n_steps, dummy):
    b = len(tok)
    tok, pos = np.array(tok, np.int32), np.array(pos, np.int32)
    out, fin = [[] for _ in range(b)], np.zeros(b, np.int32)
    steps = 0
    for _ in range(n_steps):
        if fin.all():
            break
        live = fin == 0
        nxt = dec.decode(np.where(live, tok, 0), np.where(live, pos, dummy))
        steps += 1
        for t in np.nonzero(live)[0]:
            x = int(nxt[t])
            out[t].append(x)
            ids, budget = rules[t] if rules[t] else ((), 0)
            if x in ids:
                fin[t] = 1
            elif budget and len(out[t]) >= budget:
                fin[t] = 2
            tok[t], pos[t] = x, pos[t] + 1
    return out, fin, steps


def _worker(rank, ws, port, q):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = _device(rank)
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=ws)
    res = {}
    try:
        from zhilight_b200 import dist as zdist, ops
        from zhilight_b200.llama import LlamaDecoder

        # ---- the bare gather: every rank's buffer is the concatenation of the shards, epoch after epoch ----
        gather_ok = []
        for V in (512, 128256):
            g = zdist.VocabGather(32, V, rank, ws)
            vs = V // ws
            for T in (1, 7, 32):
                for epoch in range(4):
                    full = _rows(7919 * T + epoch, T, V)
                    out = g.gather(torch.from_numpy(full[:, rank * vs:(rank + 1) * vs].copy()).to(dev))
                    torch.cuda.synchronize()
                    gather_ok.append(_bits_equal(out.cpu().numpy(), full))
                    dist.barrier()   # every rank has read its buffer before any rank gathers again
            g.close()
        res["gather"] = all(gather_ok)

        # ---- TP=2 decoder with full-vocabulary picks ----
        V, MS = TINY["vocab_size"], 64
        sd = omodel.make_state_dict(TINY, 5, 128, False, seed=6)
        comm = zdist.TPComm(16 * TINY["dim_model"], rank, ws)
        dec = LlamaDecoder(quant_type=5, max_batch=4, max_seq=MS, tp_rank=rank, tp_size=ws, prefill_chunk=16, **TINY)
        dec.set_comm(comm)
        dec.load_state_dict(zdist.shard_state_dict(sd, rank, ws))
        ref = LlamaDecoder(quant_type=5, max_batch=4, max_seq=MS, tp_rank=rank, tp_size=ws, prefill_chunk=16,
                           **TINY)   # no picks enabled
        ref_comm = zdist.TPComm(16 * TINY["dim_model"], rank, ws)
        ref.set_comm(ref_comm)
        ref.load_state_dict(zdist.shard_state_dict(sd, rank, ws))
        dec.enable_tp_picks()

        # greedy with picks enabled: the same picks and launches as without
        tok, pos = np.array([5, 99, 7, 300], np.int32), np.zeros(4, np.int32)
        same = True
        for _ in range(6):
            a, b = dec.decode(tok, pos), ref.decode(tok, pos)
            same = same and np.array_equal(a, b)
            tok, pos = a, pos + 1
        res["greedy_same"] = bool(same)
        res["greedy_kernels"] = (dec.stats(4)[1], ref.stats(4)[1])

        # sampled and processed decode: the picks of the single-GPU operator over the concatenated shards
        picks_ok = {}
        for name, s in SETTINGS.items():
            _set(dec, s)
            st = _oracle_state(dev, s, V, MS)
            tok, pos = np.array([5, 9, 5, 9], np.int32), np.zeros(4, np.int32)
            ok = True
            for _ in range(12):
                nxt, shard = dec.decode(tok, pos, want_logits=True)
                full = np.concatenate(_allgather(shard), axis=1)
                want = _oracle_pick(dev, st, full, pos)
                ranks = _allgather(nxt)
                ok = ok and all(np.array_equal(r, nxt) for r in ranks) and np.array_equal(nxt, want)
                tok, pos = nxt.astype(np.int32), pos + 1
            picks_ok[name] = bool(ok)
        res["picks"] = picks_ok
        _set(dec, [{}] * 4)

        # beam steps: zl_beam_topk over the concatenated shards, bit for bit
        groups = np.array([[0, 2], [2, 2]], np.int32)
        cum = np.array([0.0, -1.5, -0.25, -np.inf], np.float32)
        parent, token, score, shard = dec.beam_step(np.array([5, 8, 9, 2], np.int32), np.full(4, 3, np.int32), groups, cum,
                                                    4, want_logits=True)
        full = np.concatenate(_allgather(shard), axis=1)
        wp, wt, wsc = ops.beam_topk(torch.from_numpy(full).to(dev), torch.from_numpy(cum).to(dev), groups, 4)
        res["beam_step"] = bool(np.array_equal(parent, wp.cpu().numpy()) and np.array_equal(token, wt.cpu().numpy())
                                and _bits_equal(score, wsc.cpu().numpy()))
        res["beam_step_ranks"] = bool(all(np.array_equal(x, (parent, token, score)[i]) for i in range(3)
                                          for x in [o[i] for o in _allgather((parent, token, score))]))
        bs = dec.beam_search([[5, 9, 11, 4], [3, 4]], 2, 6, eos_id=2, num_results=2)
        res["beam_search_ranks"] = bool(all(repr(o) == repr(bs) for o in _allgather(bs)))

        # generate: the tokens, finish reasons and steps of a decode() host loop with the stop rules in Python
        gen_ok = {}
        for name in ("greedy", "t0.8", "ngram-bias"):
            s = SETTINGS[name]
            tok, pos = np.array([5, 9, 3, 12], np.int32), np.array([1, 2, 3, 4], np.int32)
            _set(dec, s)
            free, _, _ = _host_loop(dec, tok, pos, [None] * 4, 10, MS - 1)
            stop = next((x for i, x in enumerate(free[0]) if i >= 2 and x not in free[0][:i]), free[0][-1])
            rules = [([stop], 0), ((), 4), None, ((), 0)]
            _set(dec, s)
            want, wfin, wsteps = _host_loop(dec, tok, pos, rules, 10, MS - 1)
            _set(dec, s)
            dec.set_state(tok, pos)
            for t, r in enumerate(rules):
                dec.set_stop(t, *(r if r else ((), 0)))
            got, fin, steps = dec.generate(4, 10)
            mine = ([list(map(int, x)) for x in got], list(map(int, fin)), int(steps))
            gen_ok[name] = bool(mine == ([list(map(int, x)) for x in want], list(map(int, wfin)), wsteps)
                                and all(o == mine for o in _allgather(mine)))
        res["generate"] = gen_ok
        dec.close()
        ref.close()
        comm.close()
        ref_comm.close()
    except Exception:   # pragma: no cover
        import traceback
        res["error"] = traceback.format_exc()
    finally:
        q.put((rank, res))
        dist.destroy_process_group()


def _spawn(ws, target=_worker):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=target, args=(r, ws, port, q)) for r in range(ws)]
    for p in procs:
        p.start()
    results = dict(q.get(timeout=900) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    return results


@pytest.mark.parametrize("ws", [2])
def test_tp_picks(lib, cuda, ws):
    import torch
    if torch.cuda.device_count() < ws:
        pytest.skip("needs %d GPUs" % ws)
    results = _spawn(ws)
    for r in range(ws):
        res = results[r]
        assert "error" not in res, res.get("error")
        assert res["gather"], res
        assert res["greedy_same"] and res["greedy_kernels"][0] == res["greedy_kernels"][1], res
        assert all(res["picks"].values()), res["picks"]
        assert res["beam_step"] and res["beam_step_ranks"] and res["beam_search_ranks"], res
        assert all(res["generate"].values()), res["generate"]
