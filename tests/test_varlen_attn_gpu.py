"""GPU parity: causal variable-length attention (zl_varlen_attention) -- prompt chunks and decode rows of different tasks
in one launch -- against the fp32 oracle (oracle/ops.py::decode_attention with per-row causal masks), against the decode
kernel for decode rows, and its batch-invariance and never-read-past-the-end guarantees, bit for bit."""
import numpy as np
import pytest
import torch

from oracle import ops as oops
from tests.helpers import rel_l2

pytestmark = pytest.mark.gpu

TOL = {torch.float16: ("f16", 1e-3), torch.bfloat16: ("bf16", 6e-3)}


def _caches(cuda, dtype, n_tasks, length, hkv, d, seed):
    g = torch.Generator().manual_seed(seed)
    ks = [torch.randn(length, hkv, d, generator=g).to(dtype).to(cuda) for _ in range(n_tasks)]
    vs = [torch.randn(length, hkv, d, generator=g).to(dtype).to(cuda) for _ in range(n_tasks)]
    return ks, vs


def _queries(cuda, dtype, rows, hq, d, seed):
    g = torch.Generator().manual_seed(seed + 1000)
    return torch.randn(rows, hq, d, generator=g).to(dtype).to(cuda)


def _seg_table(segs):
    """[(task, pos0, n)] -> (nseg, 4) {task, row0, pos0, n} with rows in list order."""
    out, row0 = [], 0
    for task, pos0, n in segs:
        out.append((task, row0, pos0, n))
        row0 += n
    return np.array(out, dtype=np.int32), row0


def _run(q, segs, ks, vs, hkv, scale):
    from zhilight_b200 import ops
    table, rows = _seg_table(segs)
    assert q.shape[0] == rows
    return ops.varlen_attention(q, table, ks, vs, scale, hkv)


def _oracle(q, segs, ks, vs, hkv, scale, name):
    hq = q.shape[1]
    qn = q.float().cpu().numpy()
    out = np.zeros_like(qn)
    row0 = 0
    for task, pos0, n in segs:
        lb = pos0 + n
        k = ks[task][:lb].float().cpu().numpy()
        v = vs[task][:lb].float().cpu().numpy()
        mask = (np.arange(lb)[None, :] <= pos0 + np.arange(n)[:, None]).astype(np.int8)
        out[row0:row0 + n] = oops.decode_attention(qn[None, row0:row0 + n], [k], [v], [lb], [mask], scale, hq // hkv,
                                                   name)[0]
        row0 += n
    return out


def _check(cuda, dtype, hq, hkv, d, segs, length, seed=0):
    name, tol = TOL[dtype]
    n_tasks = max(t for t, _, _ in segs) + 1
    ks, vs = _caches(cuda, dtype, n_tasks, length, hkv, d, seed)
    rows = sum(n for _, _, n in segs)
    q = _queries(cuda, dtype, rows, hq, d, seed)
    scale = 1.0 / np.sqrt(d)
    out = _run(q, segs, ks, vs, hkv, scale).float().cpu().numpy()
    ref = _oracle(q, segs, ks, vs, hkv, scale, name)
    assert np.isfinite(out).all()
    assert rel_l2(out, ref) <= tol
    row0 = 0
    for task, pos0, n in segs:     # per segment too: a wrong task / row mapping cannot hide in the global norm
        assert rel_l2(out[row0:row0 + n], ref[row0:row0 + n]) <= 2 * tol, (task, pos0, n)
        row0 += n


MIXED = [(0, 40, 1), (1, 700, 1), (2, 0, 37), (3, 515, 1), (4, 300, 20)]    # decode rows and two chunks of other tasks


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("hq,hkv", [(32, 8), (64, 8), (8, 8)])
def test_shapes_mixed_segments(lib, cuda, dtype, d, hq, hkv):
    _check(cuda, dtype, hq, hkv, d, MIXED, 800)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("hq,hkv", [(32, 8), (8, 8)])
def test_decode_only(lib, cuda, dtype, hq, hkv):
    segs = [(0, 0, 1), (1, 17, 1), (2, 511, 1), (3, 512, 1), (4, 1500, 1), (5, 2047, 1)]
    _check(cuda, dtype, hq, hkv, 128, segs, 2048, seed=1)


@pytest.mark.parametrize("n", [1, 15, 16, 17, 300])
@pytest.mark.parametrize("pos0", [0, 1000, 4100])
def test_one_chunk_crosses_split_boundaries(lib, cuda, n, pos0):
    _check(cuda, torch.float16, 32, 8, 128, [(0, pos0, n)], pos0 + n, seed=2)


def test_one_chunk_bf16_d64(lib, cuda):
    _check(cuda, torch.bfloat16, 64, 8, 64, [(1, 1000, 300)], 1300, seed=3)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_decode_rows_agree_with_decode_kernel(lib, cuda, dtype):
    from zhilight_b200 import ops
    _, tol = TOL[dtype]
    hq, hkv, d = 32, 8, 128
    lens = [1, 64, 300, 1024, 2000]
    ks, vs = _caches(cuda, dtype, len(lens), max(lens), hkv, d, 4)
    q = _queries(cuda, dtype, len(lens), hq, d, 4)
    scale = 1.0 / np.sqrt(d)
    out = _run(q, [(b, lb - 1, 1) for b, lb in enumerate(lens)], ks, vs, hkv, scale)
    ref = ops.decode_attention(q[:, None].contiguous(), torch.tensor(lens, dtype=torch.int32, device=cuda),
                               ks, vs, None, scale, max(lens), hkv)[:, 0]
    assert rel_l2(out.float().cpu().numpy(), ref.float().cpu().numpy()) <= tol


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_rows_are_batch_invariant_and_deterministic(lib, cuda, dtype):
    """A segment's rows are bit-identical whether launched alone or beside other segments (their split count depends
    only on their own positions), and two launches give identical output."""
    hq, hkv, d = 32, 8, 128
    ks, vs = _caches(cuda, dtype, 6, 5000, hkv, d, 5)
    scale = 1.0 / np.sqrt(d)
    chunk = [(2, 1000, 70)]
    others = [(0, 4500, 1), (1, 30, 1), (3, 4000, 200), (5, 10, 3)]
    q_chunk = _queries(cuda, dtype, 70, hq, d, 6)
    q_other = _queries(cuda, dtype, 205, hq, d, 7)
    alone = _run(q_chunk, chunk, ks, vs, hkv, scale)
    again = _run(q_chunk, chunk, ks, vs, hkv, scale)
    assert torch.equal(alone, again)
    # the chunk in the middle of a launch whose other segments need more key splits
    mixed_segs = others[:2] + chunk + others[2:]
    q_mixed = torch.cat([q_other[:2], q_chunk, q_other[2:]]).contiguous()
    mixed = _run(q_mixed, mixed_segs, ks, vs, hkv, scale)
    assert torch.equal(mixed[2:72], alone)
    # and the decode rows / other chunk alone match their rows of the mixed launch
    assert torch.equal(_run(q_other[:1].contiguous(), others[:1], ks, vs, hkv, scale), mixed[:1])
    assert torch.equal(_run(q_other[2:202].contiguous(), others[2:3], ks, vs, hkv, scale), mixed[72:272])


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_rows_past_a_task_end_are_never_read(lib, cuda, dtype):
    """NaN in every cache row at or past each task's pos0 + n, and in every row of tasks outside the launch: the output
    stays finite and bit-identical (the kernel zero-fills keys past a tile's last position instead of relying on
    unwritten rows being finite)."""
    hq, hkv, d = 32, 8, 128
    length = 1200
    ks, vs = _caches(cuda, dtype, 5, length, hkv, d, 8)
    segs = [(0, 0, 33), (1, 100, 1), (3, 511, 2), (4, 600, 300)]
    q = _queries(cuda, dtype, 336, hq, d, 8)
    scale = 1.0 / np.sqrt(d)
    clean = _run(q, segs, ks, vs, hkv, scale)
    pk = [k.clone() for k in ks]
    pv = [v.clone() for v in vs]
    for task, pos0, n in segs:
        pk[task][pos0 + n:] = float("nan")
        pv[task][pos0 + n:] = float("nan")
    for task in (2,):                          # not in the launch
        pk[task][:] = float("nan")
        pv[task][:] = float("nan")
    poisoned = _run(q, segs, pk, pv, hkv, scale)
    assert torch.isfinite(poisoned.float()).all()
    assert torch.equal(poisoned, clean)
