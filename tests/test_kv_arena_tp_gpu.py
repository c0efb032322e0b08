"""KV arena under tensor parallelism (needs >= 2 GPUs on the box; skipped otherwise): every rank makes the same calls, so
every rank's arena makes the same grants, moves and compactions for its own kv heads.  A TP decode whose tasks grow,
relocate and compact inside a 256-row arena gives the same logits and cache bytes, bit for bit, as with kv_rows = 0."""
import os

import numpy as np
import pytest

from oracle import model as omodel
from tests.test_tp_gpu import TINY, _free_port

pytestmark = pytest.mark.gpu

STEPS = 100   # tasks 0 and 1 cross 64 rows at step 64: task 0 moves to the free extent, task 1 is compacted down


def _worker(rank, ws, port, q):
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
        sd = omodel.make_state_dict(TINY, 5, 128, False, seed=4)
        runs = {}
        for kv_rows in (None, 256):
            dec = LlamaDecoder(quant_type=5, max_batch=2, max_seq=256, tp_rank=rank, tp_size=ws, kv_rows=kv_rows, **TINY)
            comm = zdist.TPComm(2 * TINY["dim_model"], rank, ws)
            dec.set_comm(comm)
            dec.load_state_dict(zdist.shard_state_dict(sd, rank, ws))
            tok = np.array([5, 99], dtype=np.int32)
            logits_all = []
            for step in range(STEPS):
                nxt, logits = dec.decode(tok, np.full(2, step, dtype=np.int32), want_logits=True)
                logits_all.append(logits.copy())
                tok = nxt
            caps = [dec.kv_capacity(t) for t in (0, 1)]
            runs[kv_rows] = (logits_all, [dec.read_kv(l, t, 0, STEPS) for l in range(TINY["num_layers"]) for t in (0, 1)],
                             caps)
            dec.close()
            comm.close()
        res["logits_equal"] = all(np.array_equal(a, b) for a, b in zip(runs[None][0], runs[256][0]))
        res["cache_equal"] = all(np.array_equal(x, y) for a, b in zip(runs[None][1], runs[256][1]) for x, y in zip(a, b))
        res["caps"] = runs[256][2]
    except Exception:   # pragma: no cover
        import traceback
        res["error"] = traceback.format_exc()
    finally:
        q.put((rank, res))
        dist.destroy_process_group()


def test_tp2_arena_decode_equals_fixed_layout(lib, cuda):
    import torch
    ws = 2
    if torch.cuda.device_count() < ws:
        pytest.skip("needs %d GPUs" % ws)
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, ws, port, q)) for r in range(ws)]
    for p in procs:
        p.start()
    results = dict(q.get(timeout=600) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    for r in range(ws):
        res = results[r]
        assert "error" not in res, res.get("error")
        assert res["logits_equal"] and res["cache_equal"], res
        assert res["caps"] == [128, 128], res
