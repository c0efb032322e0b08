"""int8 KV cache under tensor parallelism (needs >= 2 GPUs on the box; skipped otherwise): each rank caches its own kv
heads; the qkv GEMM's int8-cache epilogue runs together with the exchange reduced in while it stages its activations.
The fused exchange against ZL_TP_UNFUSED=1 (stand-alone exchange kernels, same arithmetic in the same order) must agree
bit for bit, logits and cache bytes, and the logits must match the int8 oracle."""
import os

import numpy as np
import pytest

from oracle import model as omodel
from tests.helpers import rel_l2
from tests.kv8_oracle import Kv8OracleLlama
from tests.test_tp_gpu import TINY, _free_port

pytestmark = pytest.mark.gpu


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
        sd = omodel.make_state_dict(TINY, 5, 128, False, seed=2)
        vs = TINY["vocab_size"] // ws
        runs = {}
        for unfused in (False, True):
            if unfused:
                os.environ["ZL_TP_UNFUSED"] = "1"
            else:
                os.environ.pop("ZL_TP_UNFUSED", None)
            dec = LlamaDecoder(quant_type=5, max_batch=2, max_seq=32, tp_rank=rank, tp_size=ws, kv_cache_dtype="int8",
                               **TINY)
            comm = zdist.TPComm(2 * TINY["dim_model"], rank, ws)
            dec.set_comm(comm)
            dec.load_state_dict(zdist.shard_state_dict(sd, rank, ws))
            orc = Kv8OracleLlama(TINY, sd, 5, 128, False, "f16", fuse_norm=True)
            tok = np.array([5, 99], dtype=np.int32)
            logits_all, worst = [], 0.0
            for step in range(8):
                pos = np.full(2, step, dtype=np.int32)
                nxt, logits = dec.decode(tok, pos, want_logits=True)
                ref = orc.decode(tok, pos)
                worst = max(worst, rel_l2(logits, ref[:, rank * vs:(rank + 1) * vs]))
                logits_all.append(logits.copy())
                tok = nxt
            runs[unfused] = (logits_all, [dec.read_kv(l, t, 0, 8) for l in range(TINY["num_layers"]) for t in (0, 1)],
                             worst, dec.kv_row)
            dec.close()
            comm.close()
        os.environ.pop("ZL_TP_UNFUSED", None)
        res["logits_equal"] = all(np.array_equal(a, b) for a, b in zip(runs[False][0], runs[True][0]))
        res["cache_equal"] = all(np.array_equal(x, y) for a, b in zip(runs[False][1], runs[True][1]) for x, y in zip(a, b))
        res["worst"] = (runs[False][2], runs[True][2])
        res["kv_row"] = runs[False][3]
    except Exception:   # pragma: no cover
        import traceback
        res["error"] = traceback.format_exc()
    finally:
        q.put((rank, res))
        dist.destroy_process_group()


def test_tp2_int8_cache_fused_exchange_equals_unfused_and_matches_oracle(lib, cuda):
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
        assert res["kv_row"] == (TINY["num_kv_heads"] // ws, TINY["dim_head"]), res
        assert max(res["worst"]) <= 1.5e-2, res      # the decode bound of test_kv8_gpu.test_decode_matches_int8_oracle
