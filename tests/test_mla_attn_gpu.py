"""MLA decode attention (zl_mla_decode_attention / ops.mla_decode_attention) on the GPU against the fp32 oracle
(tests/mla_golden.mla_oracle: the latent rows as K and their first 512 columns as V), the reference's own kernels
(tests/golden/mla_ref.npz, and the same reference-signature call through the drop-in library), NaN-poisoned cache
tails, fully masked rows and launch-to-launch determinism."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import ops as oops
from tests import mla_golden
from tests.helpers import rel_l2
from zhilight_b200 import _lib, ops

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_MLA = os.path.join(ROOT, "oracle", "_ref", "libzl_ref_mla.so")
DROPIN_MLA = os.path.join(ROOT, "oracle", "_ref", "libzl_dropin_mla.so")
TOL = mla_golden.TOL
TORCH_DT = {"f16": torch.float16, "bf16": torch.bfloat16}
SCALE = float(1.0 / np.sqrt(192.0))


def _masks(kind, len_q, lens, r):
    out = []
    for lb in lens:
        m = np.ones((len_q, lb), np.int8)
        if kind == "causal":
            for i in range(len_q):
                m[i, lb - len_q + i + 1:] = 0
        elif kind == "random":
            m = (r.random((len_q, lb)) > 0.25).astype(np.int8)
        out.append(m)
    return out


def _inputs(seed, b, len_q, h, lens, kind, tag, pad=64, pad_value=0.0):
    """q (B, len_q, H, 576) and per-task caches holding `pad` extra rows of pad_value past each task's length."""
    r = np.random.default_rng(seed)
    q = oops._t(r.standard_normal((b, len_q, h, 576)), tag)
    kvs = [oops._t(r.standard_normal((lb, 1, 576)), tag) for lb in lens]
    masks = _masks(kind, len_q, lens, r)
    return q, kvs, masks, pad, pad_value


def _run(cuda, q, kvs, masks, lens, tag, pad=64, pad_value=0.0, use_mask=True, layout3=False):
    dt = TORCH_DT[tag]
    bufs = []
    for kv in kvs:
        full = torch.full((kv.shape[0] + pad, 576), pad_value, dtype=torch.float32)
        full[: kv.shape[0]] = torch.from_numpy(kv.reshape(-1, 576))
        t = full.to(dt).to(cuda)
        bufs.append(t.view(-1, 1, 576) if layout3 else t)
    mask = torch.from_numpy(np.concatenate([m.reshape(-1) for m in masks])).to(cuda) if use_mask else None
    lens_t = torch.tensor(lens, dtype=torch.int32, device=cuda)
    out = ops.mla_decode_attention(torch.from_numpy(q).to(dt).to(cuda), lens_t, bufs, mask, SCALE, max(lens))
    assert out.shape == (q.shape[0], q.shape[1], q.shape[2], 512) and out.dtype == dt
    return out.float().cpu().numpy()


def _oracle(q, kvs, masks, lens, h, tag):
    return mla_golden.mla_oracle(q, kvs, lens, masks, SCALE, tag)


# (H, len_q, lens, mask kind): every H at B = 3 with short ragged lengths, B = 33 over the ragged edge lengths, and long
# tasks at small B and H (the numpy oracle pays B len_q H ctx 1088 FLOP).  B = 33 at H = 128, len_q = 2 fills the 132 SMs
# with row tiles, so it runs unsplit even with a 16384-key task; the others split their keys.
EDGE = [1, 63, 64, 65, 511, 513, 1025]
CASES = [(h, lq, [1, 63, 513], kind) for h in (1, 16, 32, 64, 128) for lq, kind in ((1, "none"), (2, "causal"))]
CASES += [(16, 1, [EDGE[i % 7] for i in range(33)], "random"), (64, 2, [65, 511, 1025], "random"),
          (16, 1, [16500], "none"), (1, 2, [16384, 1025], "causal"),
          (128, 2, [16384] + [EDGE[i % 7] for i in range(32)], "causal")]


@pytest.mark.parametrize("tag", ["f16", "bf16"])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_mla_against_oracle(lib, cuda, case, tag):
    h, len_q, lens, kind = CASES[case]
    q, kvs, masks, _, _ = _inputs(100 + case, len(lens), len_q, h, lens, kind, tag)
    got = _run(cuda, q, kvs, masks, lens, tag, use_mask=kind != "none", layout3=case % 2 == 1)
    ref = _oracle(q, kvs, masks, lens, h, tag)
    err = rel_l2(got, ref)
    assert err <= TOL[tag], (CASES[case][:2], kind, err)


@pytest.mark.parametrize("tag", ["f16", "bf16"])
def test_mla_nan_tail_and_determinism(lib, cuda, tag):
    """Cache rows past every task's length are never read, and two launches give the same bits (split and unsplit)."""
    for h, len_q, lens in ((16, 1, [700, 1, 3000]), (128, 2, [300] * 40)):
        q, kvs, masks, _, _ = _inputs(7, len(lens), len_q, h, lens, "random", tag)
        a = _run(cuda, q, kvs, masks, lens, tag, pad=200, pad_value=0.0)
        b = _run(cuda, q, kvs, masks, lens, tag, pad=200, pad_value=float("nan"))
        c = _run(cuda, q, kvs, masks, lens, tag, pad=200, pad_value=float("nan"))
        assert np.isfinite(a).all()
        np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32))
        np.testing.assert_array_equal(b.view(np.uint32), c.view(np.uint32))


@pytest.mark.parametrize("lens", [[90], [3000, 40]])
def test_mla_fully_masked_row_is_zero(lib, cuda, lens):
    q, kvs, masks, _, _ = _inputs(11, len(lens), 2, 16, lens, "none", "f16")
    masks[0][1] = 0                     # query row 1 of task 0 attends no key
    got = _run(cuda, q, kvs, masks, lens, "f16")
    assert (got[0, 1] == 0).all()
    assert rel_l2(got, _oracle(q, kvs, masks, lens, 16, "f16")) <= TOL["f16"]


def test_mla_against_reference_goldens(lib, cuda):
    """Our kernel on the case_mla inputs against the reference's own kernels' outputs."""
    c = mla_golden.case_mla()
    assert c["scale"] == SCALE
    with np.load(mla_golden.FIXTURE) as g:
        for name, tag, key in mla_golden.keys():
            sc = c["cases"][name]
            kvs = [oops._t(kv, tag) for kv in sc["kvs"]]
            got = _run(cuda, oops._t(sc["q"], tag), kvs, sc["masks"], [int(x) for x in sc["lens"]], tag)
            err = rel_l2(got, g[key].astype(np.float32))
            assert err <= TOL[tag], (key, err)


def test_mla_dropin_call_agrees_with_reference(lib, cuda, tmp_path):
    """The reference-signature MLA call (multi_query_attention_rag_buffer, dim_head 576) through the reference's kernels
    and through integration/zl_nn_dropin.cpp, each in its own process."""
    if not (os.path.exists(REF_MLA) and os.path.exists(DROPIN_MLA)):
        pytest.skip("oracle/_ref/libzl_ref_mla.so / libzl_dropin_mla.so not built")
    outs = []
    for name, so in (("ref", REF_MLA), ("dropin", DROPIN_MLA)):
        d = str(tmp_path / name)
        r = subprocess.run([sys.executable, "-m", "tests.mla_golden", d, so], cwd=ROOT, capture_output=True, text=True,
                           timeout=600)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        outs.append(np.load(os.path.join(d, "mla_ref.npz")))
    for _, tag, key in mla_golden.keys():
        err = rel_l2(outs[1][key].astype(np.float32), outs[0][key].astype(np.float32))
        assert err <= TOL[tag], (key, err)
    mla_golden.check(outs[1])


def test_mla_ops_reject_malformed_cuda_shapes(lib, cuda):
    q = torch.zeros(1, 1, 16, 576, dtype=torch.float16, device=cuda)
    lens = torch.tensor([8], dtype=torch.int32, device=cuda)
    for qq, kv in ((q[..., :512].contiguous(), [torch.zeros(8, 576, dtype=torch.float16, device=cuda)]),
                   (q, [torch.zeros(8, 2, 576, dtype=torch.float16, device=cuda)])):
        with pytest.raises(_lib.ZLError) as e:
            ops.mla_decode_attention(qq, lens, kv, None, 0.1, 8)
        assert e.value.code == -1
