"""GPU parity: batch decode attention over per-task ragged KV buffers vs the oracle
(reference semantics attention_kernel.cu:434-489, 674-725, 730-923)."""
import numpy as np
import pytest
import torch

from oracle import ops as oops
from tests.attn_check import assert_close as _assert_close
from tests.attn_check import launched as _launched
from tests.helpers import rel_l2

pytestmark = pytest.mark.gpu


def _case(cuda, dtype, name, hq, hkv, d, lens, len_q=1, masked=True, seed=0, bshd=True):
    from zhilight_b200 import ops
    g = torch.Generator().manual_seed(seed)
    b = len(lens)
    q = torch.randn(b, len_q, hq, d, generator=g).to(dtype)
    ks, vs, masks = [], [], []
    for lb in lens:
        shape = (lb, hkv, d) if bshd else (hkv, lb, d)
        ks.append(torch.randn(*shape, generator=g).to(dtype))
        vs.append(torch.randn(*shape, generator=g).to(dtype))
        m = torch.ones(len_q, lb, dtype=torch.int8)
        if masked:
            for qi in range(len_q):
                valid = max(1, lb - 2 - 3 * qi)           # the reference's len_buf is padded past the tokens
                m[qi, valid:] = 0
                m[qi, torch.randperm(valid, generator=g)[: valid // 7]] = 0   # beam-tree style holes
        masks.append(m)
    scale = 1.0 / np.sqrt(d)
    mask_flat = torch.cat([m.reshape(-1) for m in masks]).to(cuda)
    out = ops.decode_attention(q.to(cuda), torch.tensor(lens, dtype=torch.int32, device=cuda),
                               [k.to(cuda) for k in ks], [v.to(cuda) for v in vs], mask_flat if masked else None,
                               scale, max(lens), hkv, bshd=bshd)
    kn = [k.float().numpy() if bshd else k.float().permute(1, 0, 2).contiguous().numpy() for k in ks]
    vn = [v.float().numpy() if bshd else v.float().permute(1, 0, 2).contiguous().numpy() for v in vs]
    ref = oops.decode_attention(q.float().numpy(), kn, vn, lens, [m.numpy() for m in masks], scale, hq // hkv, name)
    return out.float().cpu().numpy(), ref


@pytest.mark.parametrize("dtype,name,tol", [(torch.float16, "f16", 1e-3), (torch.bfloat16, "bf16", 6e-3)])
@pytest.mark.parametrize("hq,hkv,d", [(32, 8, 128), (32, 8, 64), (8, 1, 128), (16, 16, 64), (64, 8, 128), (32, 2, 128)])
def test_gqa_shapes(lib, cuda, dtype, name, tol, hq, hkv, d):
    out, ref = _case(cuda, dtype, name, hq, hkv, d, [130, 64, 17, 1])
    assert rel_l2(out, ref) <= tol
    # per (task, head) as well: a wrong head/task mapping cannot hide in the global norm
    for b in range(out.shape[0]):
        for h in range(hq):
            assert rel_l2(out[b, 0, h], ref[b, 0, h]) <= 4 * tol, (b, h)


@pytest.mark.parametrize("lens", [[4096, 123], [2048] * 3, [1500, 700, 3000, 64, 65], [1], [16], [15, 33]])
def test_split_kv_and_ragged_lengths(lib, cuda, lens):
    """src/nn/tests/test_attention_rag_buffer.cpp uses lens {4096, 123}, 4 kv-heads x m_query 4."""
    out, ref = _case(cuda, torch.float16, "f16", 16, 4, 128, lens, seed=1)
    assert rel_l2(out, ref) <= 1e-3


def test_no_mask_and_beam_queries(lib, cuda):
    out, ref = _case(cuda, torch.float16, "f16", 8, 2, 128, [300, 90], len_q=3, masked=True, seed=2)
    assert rel_l2(out, ref) <= 1e-3
    out, ref = _case(cuda, torch.float16, "f16", 8, 2, 128, [300, 90], len_q=1, masked=False, seed=3)
    assert rel_l2(out, ref) <= 1e-3


def test_hsd_layout(lib, cuda):
    out, ref = _case(cuda, torch.float16, "f16", 8, 2, 64, [200, 40], seed=4, bshd=False)
    assert rel_l2(out, ref) <= 1e-3


def test_fully_masked_row_is_zero_not_nan(lib, cuda):
    from zhilight_b200 import ops
    q = torch.randn(1, 1, 4, 64, device=cuda).half()
    k = [torch.randn(32, 1, 64, device=cuda).half()]
    v = [torch.randn(32, 1, 64, device=cuda).half()]
    mask = torch.zeros(32, dtype=torch.int8, device=cuda)
    out = ops.decode_attention(q, torch.tensor([32], dtype=torch.int32, device=cuda), k, v, mask, 0.125, 32, 1)
    assert torch.isfinite(out).all() and out.abs().max() < 1e-6     # sum seeded with 1e-20 (attention_kernel.cu:466)


# ---------------------------------------------------------------------------------------------------------------------
# Every route of zl_decode_attention (warp kernel, split-KV kernel) and of zl_decode_attention_kv8 against a float64
# reference, with the launched kernels checked by the profiler.  The host picks the route from the shapes and the SM
# count (decode_attn.cu zl_decode_attention, decode_attn_kv8.cu zl_decode_attention_kv8); _plan restates that rule so
# that the shapes below reach their kernel on any H100, and a change of the dispatch fails the route assertion instead
# of quietly testing another kernel.
# ---------------------------------------------------------------------------------------------------------------------
SHORT_RANGE, MAX_RANGE, MAX_SPLITS = 256, 1024, 64
KERNEL = {"warp": "k_decode_attn_warp<", "split": "k_decode_attn<", "kv8": "k_decode_attn_kv8<"}
HOT = 15.0          # logit of a planted key, +-1; the others are ~N(0, 1)
TOL = {torch.float16: 1e-3, torch.bfloat16: 6e-3}
KV8_TOL = {torch.float16: 1e-3, torch.bfloat16: 6e-3}   # by output dtype: bf16's own rounding (2^-9) is above 1e-3
DEVICE = "cuda:0"


def _cdiv(a, b):
    return -(-a // b)


def _round16(v):
    return (v + 15) & ~15


def _plan(b, len_q, hkv, mq, max_len_buf, kv8=False):
    """(kernel, key splits) the host launches for these shapes."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    base = b * len_q * hkv * _cdiv(mq, 8)
    if not kv8:
        short = _cdiv(max_len_buf, SHORT_RANGE)
        if short <= MAX_SPLITS and base * short <= 4 * sm:
            return "warp", short
    s = min(_cdiv(2 * sm, base), max(1, _cdiv(max_len_buf, 256)), MAX_SPLITS)
    return ("kv8" if kv8 else "split"), max(s, _cdiv(max_len_buf, MAX_RANGE), 1)


def _bucket(max_len):
    """The decode driver's power-of-two length bucket (llama_runner.cu len_bucket_of, without the max_seq cap)."""
    b = 256
    while b < max_len:
        b <<= 1
    return b


def _split_bounds(len_buf, splits):
    chunk = _round16(_cdiv(len_buf, splits))
    return [(k0, min(len_buf, k0 + chunk)) for k0 in range(0, len_buf, chunk)]


def _hot_keys(len_buf, split_counts):
    """Key 0, len_buf - 1, and per split its first and last key, the keys either side of its first 16-key tile
    boundary and of its 32-key warp boundaries: a kernel that drops or repeats one of them moves the output by O(1)."""
    hot = {0, len_buf - 1}
    for s in split_counts:
        for k0, k1 in _split_bounds(len_buf, s):
            edges = [k0, k0 + 15, k0 + 16, k1 - 1] + [k0 + 32 * j + e for j in range(1, 8) for e in (-1, 0)]
            hot.update(k for k in edges if k < k1)
    return sorted(hot)


def _assert_route(names, route, splits):
    for r, k in KERNEL.items():
        assert any(k in n for n in names) == (r == route), (route, splits, names)
    assert any("k_attn_combine" in n for n in names) == (splits > 1), (route, splits, names)


class _Inputs:
    """q (B, len_q, H_q, d) and per-task K / V whose keys are orthogonal to a per-kv-head direction u that every q
    head of the group shares: a key planted as (HOT + x) * u has logit HOT + x, x uniform in [-1, 1) (so that the
    splits' maxima differ and their merge weights matter), the rest ~N(0, 1).  Masks are bool (len_q,
    len_buf) per task, or None.  The float64 copies k64 / v64 ((len_buf, H_kv, d)) are what the kernels see."""

    def __init__(self, lens, len_q, hkv, mq, d, dtype, split_counts=(), mask="holes", pos0=0, seed=0):
        dev = torch.device(DEVICE)
        g = torch.Generator(device=dev).manual_seed(seed)
        f64 = torch.float64
        self.lens, self.len_q, self.hkv, self.mq, self.d, self.dtype = list(lens), len_q, hkv, mq, d, dtype
        self.scale = 1.0 / np.sqrt(d)
        b = len(lens)
        u = torch.randn(hkv, d, generator=g, device=dev, dtype=f64)
        u /= u.norm(dim=-1, keepdim=True)

        def perp(x):     # x (..., hkv, d) minus its component along u
            return x - (x * u).sum(-1, keepdim=True) * u

        noise = perp(torch.randn(b, len_q, mq, hkv, d, generator=g, device=dev, dtype=f64)).transpose(2, 3)
        self.q = (np.sqrt(d) * u[:, None, :] + noise).reshape(b, len_q, hkv * mq, d).to(dtype)
        self.k, self.v, self.masks = [], [], []
        for lb in self.lens:
            k = perp(torch.randn(lb, hkv, d, generator=g, device=dev, dtype=f64))
            hot = _hot_keys(lb, split_counts)
            k[hot] = (HOT + 2 * torch.rand(len(hot), 1, 1, generator=g, device=dev, dtype=f64) - 1) * u
            self.k.append(k.to(dtype))
            self.v.append(torch.randn(lb, hkv, d, generator=g, device=dev, dtype=f64).to(dtype))
            if mask == "causal":           # the driver's prompt-chunk mask: row i sees keys 0 ..= pos0 + i
                m = torch.arange(lb, device=dev)[None, :] <= pos0 + torch.arange(len_q, device=dev)[:, None]
            elif mask == "holes":          # beam-tree style holes, different per query; planted keys stay visible
                m = torch.rand(len_q, lb, generator=g, device=dev) >= 0.125
                m[:, hot] = True
            else:
                m = None
            self.masks.append(m)
        self.k64 = [k.to(f64) for k in self.k]
        self.v64 = [v.to(f64) for v in self.v]

    def mask_flat(self):
        if self.masks[0] is None:
            return None
        return torch.cat([m.reshape(-1) for m in self.masks]).to(torch.int8)

    def buf_lens(self):
        return torch.tensor(self.lens, dtype=torch.int32, device=self.q.device)

    def reference(self):
        """float64 decode attention (oracle/ops.py decode_attention): masked logits -inf, max seeded -1e20, sum + 1e-20."""
        b, len_q, hq, d = self.q.shape
        out = torch.zeros(b, len_q, hq, d, dtype=torch.float64, device=self.q.device)
        for i in range(b):
            qb = self.q[i].double().view(len_q, self.hkv, self.mq, d)
            s = torch.einsum("qgmd,lgd->qgml", qb, self.k64[i]) * self.scale
            if self.masks[i] is not None:
                s = s.masked_fill(~self.masks[i][:, None, None, :], float("-inf"))
            e = torch.exp(s - s.amax(-1, keepdim=True).clamp_min(-1e20))
            p = e / (e.sum(-1, keepdim=True) + 1e-20)
            out[i] = torch.einsum("qgml,lgd->qgmd", p, self.v64[i]).reshape(len_q, hq, d)
        return out


def _kv_buffers(x, bshd, tail, fill):
    """One task's K or V (len_buf, H_kv, d) in the kernel's layout, with `tail` more elements of `fill` after it."""
    body = (x if bshd else x.transpose(0, 1)).contiguous().reshape(-1)
    return torch.cat([body, torch.full((tail,), fill, dtype=x.dtype, device=x.device)])


def _run_fp(inp, max_len_buf, bshd=True, tail=0, fill=0.0):
    from zhilight_b200 import ops
    row = inp.hkv * inp.d
    ks = [_kv_buffers(k, bshd, tail * row, fill) for k in inp.k]
    vs = [_kv_buffers(v, bshd, tail * row, fill) for v in inp.v]
    mask = inp.mask_flat()
    return _launched(lambda: ops.decode_attention(inp.q, inp.buf_lens(), ks, vs, mask, inp.scale, max_len_buf, inp.hkv,
                                                  bshd=bshd))


class _Kv8Cache:
    """The int8 cache of an _Inputs' K / V, written by kv_int8_quant_append, with `tail` more rows of capacity per
    task (codes random, scales `fill`); the dequantised (code - 128) * scale rows replace the inputs' float64 K / V."""

    def __init__(self, inp, tail=0, fill=0.0, seed=1):
        from zhilight_b200 import ops
        dev = inp.q.device
        g = torch.Generator(device=dev).manual_seed(seed)
        hkv, d = inp.hkv, inp.d
        self.k, self.v, self.sk, self.sv = [], [], [], []
        for lb in inp.lens:
            for codes in (self.k, self.v):
                codes.append(torch.randint(0, 256, (lb + tail, hkv, d), generator=g, device=dev, dtype=torch.uint8))
            for sc in (self.sk, self.sv):
                sc.append(torch.full((lb + tail, hkv), fill, dtype=torch.float32, device=dev))
        batch = torch.cat([torch.full((lb,), i, dtype=torch.int32, device=dev) for i, lb in enumerate(inp.lens)])
        place = torch.cat([torch.arange(lb, dtype=torch.int32, device=dev) for lb in inp.lens])
        ops.kv_int8_quant_append(torch.cat(inp.k), torch.cat(inp.v), batch, place, self.k, self.v, self.sk, self.sv)
        inp.k64 = [(c[:lb].double() - 128) * s[:lb, :, None].double() for c, s, lb in zip(self.k, self.sk, inp.lens)]
        inp.v64 = [(c[:lb].double() - 128) * s[:lb, :, None].double() for c, s, lb in zip(self.v, self.sv, inp.lens)]

    def launch(self, inp, max_len_buf, out_dtype):
        from zhilight_b200 import ops
        return ops.decode_attention_kv8(inp.q, inp.buf_lens(), self.k, self.v, self.sk, self.sv, inp.mask_flat(), inp.scale,
                                        max_len_buf, inp.hkv, out_dtype=out_dtype)

    def run(self, inp, max_len_buf, out_dtype):
        return _launched(lambda: self.launch(inp, max_len_buf, out_dtype))


def _tasks(route, lens, len_q, hkv, mq, splits=None, kv8=False):
    """Tasks cycled from `lens` until _plan gives `route` with `splits` key splits (an int, "many" for >= 3, or None for
    any count): the split-KV kernel needs more work than the warp kernel takes."""
    for b in range(len(lens), 512):
        tasks = [lens[i % len(lens)] for i in range(b)]
        r, s = _plan(b, len_q, hkv, mq, max(tasks), kv8)
        if r == route and (splits is None or s == splits or (splits == "many" and s >= 3)):
            return tasks, s
        if route == "warp":
            break
    raise AssertionError("no batch of %s reaches %s with %s splits" % (lens, route, splits))


# (kernel, dtype (kv8: output dtype), d, m_query, kv heads, BSHD, len_q, lens, splits); len_q 256 is a causal prompt
# chunk whose last row sees the last key.  Each kernel covers f16 / bf16, d 64 / 128, m_query 1 5 7 8 12 16, len_q 1 / 3
# / 256 and 1, 2, many and exactly 64 key splits; the split-KV kernel also more than 64.  A single long task has at most
# two (kv head x head group) units, so that the host asks for 64 splits on any H100.
F16, BF16 = torch.float16, torch.bfloat16
MATRIX = [
    ("warp", F16, 128, 1, 8, True, 1, [256, 130, 17, 1], 1),
    ("warp", BF16, 64, 5, 4, False, 1, [300, 64, 17, 1], 2),
    ("warp", F16, 64, 7, 4, True, 3, [400, 90], 2),
    ("warp", BF16, 128, 8, 2, True, 1, [3000, 1200, 5], "many"),
    ("warp", F16, 128, 12, 2, False, 1, [2500, 33], "many"),
    ("warp", BF16, 128, 16, 1, True, 1, [16384], 64),
    ("warp", F16, 64, 5, 4, True, 1, [16300], 64),
    ("warp", F16, 128, 8, 1, True, 256, [256], 1),
    ("warp", BF16, 64, 12, 2, True, 3, [200, 100, 1], 1),
    ("warp", F16, 128, 16, 1, False, 3, [700], "many"),
    ("warp", BF16, 128, 7, 4, False, 1, [256, 255, 16, 15], 1),
    ("warp", F16, 64, 8, 2, True, 1, [1024, 1025], "many"),
    ("split", F16, 128, 1, 8, True, 1, [1000, 513, 1, 300], 1),
    ("split", BF16, 64, 5, 4, False, 1, [1500, 700, 64], 2),
    ("split", F16, 64, 7, 4, True, 3, [4000, 1000], "many"),
    ("split", BF16, 128, 8, 2, True, 256, [1256], 2),
    ("split", F16, 64, 16, 1, True, 256, [1256], 2),
    ("split", BF16, 128, 12, 2, False, 1, [4000, 3000, 2000], "many"),
    ("split", F16, 128, 16, 1, True, 1, [20000], 64),
    ("split", BF16, 64, 5, 2, True, 1, [20000], 64),
    ("split", F16, 128, 8, 2, True, 1, [70000], 69),
    ("split", BF16, 64, 7, 1, False, 1, [70000], 69),
    ("split", F16, 64, 12, 2, True, 3, [900, 1], 1),
    ("split", BF16, 128, 5, 4, True, 1, [2000, 100], 2),
    ("kv8", F16, 128, 1, 8, True, 1, [256, 130, 17, 1], 1),
    ("kv8", BF16, 64, 5, 4, True, 1, [300, 64], 2),
    ("kv8", F16, 64, 7, 4, True, 3, [3000, 90], "many"),
    ("kv8", BF16, 128, 8, 2, True, 256, [1256], 2),
    ("kv8", F16, 128, 12, 1, True, 1, [20000], 64),
    ("kv8", BF16, 128, 16, 1, True, 1, [16384], 64),
    ("kv8", F16, 64, 8, 2, True, 3, [1000, 1], 1),
    ("kv8", BF16, 64, 1, 8, True, 1, [1025, 1024, 15, 16], "many"),
    ("kv8", F16, 128, 5, 1, True, 1, [60000], 64),
    ("kv8", BF16, 128, 7, 4, True, 3, [5000], "many"),
    ("kv8", F16, 64, 16, 1, True, 256, [256], 1),
    ("kv8", F16, 128, 8, 2, True, 1, [2000, 300], 2),
]


def _matrix_id(c):
    route, dt, d, mq, hkv, bshd, len_q, lens, splits = c
    return "%s-%s-d%d-mq%d-hkv%d-%s-q%d-s%s" % (route, "f16" if dt == F16 else "bf16", d, mq, hkv,
                                               "bshd" if bshd else "hsd", len_q, splits)


@pytest.mark.parametrize("case", MATRIX, ids=[_matrix_id(c) for c in MATRIX])
def test_route_matrix_against_float64(lib, cuda, case):
    route, dtype, d, mq, hkv, bshd, len_q, lens, splits = case
    kv8 = route == "kv8"
    tasks, s = _tasks(route, lens, len_q, hkv, mq, splits, kv8)
    chunk = len_q == 256
    mask = "causal" if chunk else (None if mq in (5, 12) and len_q == 1 else "holes")
    inp = _Inputs(tasks, len_q, hkv, mq, d, F16 if kv8 else dtype, split_counts=[s], mask=mask,
                  pos0=tasks[0] - len_q if chunk else 0, seed=d + mq + len(tasks))
    if kv8:
        out, names = _Kv8Cache(inp).run(inp, max(tasks), dtype)
        tol = KV8_TOL[dtype]
    else:
        out, names = _run_fp(inp, max(tasks), bshd)
        tol = TOL[dtype]
    _assert_route(names, route, s)
    _assert_close(out, inp.reference(), tol, (route, s))


@pytest.mark.parametrize("dtype", [F16, BF16, "kv8"])
@pytest.mark.parametrize("shape", ["bucket-flips-route", "ragged"])
def test_max_len_buf_bucket_and_8192_agree(lib, cuda, dtype, shape):
    """The decode driver passes its power-of-two length bucket as max_len_buf, not the longest task: the split count,
    and with it possibly the kernel, changes, and short tasks get empty splits.  The result must not."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    kv8 = dtype == "kv8"
    hkv, mq, d = 8, 4, 128
    if shape == "bucket-flips-route":
        b = 4 * sm // (hkv * 8) + 1                # warp kernel at 5 splits (1025 keys), split-KV at 8 (the 2048 bucket)
        lens = [[1025, 700, 1, 300, 1024, 17][i % 6] for i in range(b)]
    else:
        lens = [3000, 40, 1, 2999]
    sizes = [max(lens), _bucket(max(lens)), 8192]
    plans = [_plan(len(lens), 1, hkv, mq, m, kv8) for m in sizes]
    if shape == "bucket-flips-route" and not kv8:
        assert plans[0][0] == "warp" and plans[1][0] == "split", plans
    inp = _Inputs(lens, 1, hkv, mq, d, F16 if kv8 else dtype, split_counts=[s for _, s in plans], seed=7)
    cache = _Kv8Cache(inp) if kv8 else None
    ref = inp.reference()
    for m, (route, s) in zip(sizes, plans):
        out, names = cache.run(inp, m, F16) if kv8 else _run_fp(inp, m)
        _assert_route(names, route, s)
        _assert_close(out, ref, KV8_TOL[F16] if kv8 else TOL[dtype], (m, route, s))


def _edge_tasks(route, max_len, hkv, mq):
    """Lengths 1, 15, 16, the split chunk of the longest task and one more, and four tasks of max_len: one fully
    masked, one whose second split is fully masked, two live; cycled to the batch that reaches `route`."""
    for b in range(9, 512):
        r, s = _plan(b, 1, hkv, mq, max_len, route == "kv8")
        if r == route:
            break
    assert r == route and s >= 2, (route, r, s)
    c = _round16(_cdiv(max_len, s))
    base = [1, 15, 16, c, c + 1, max_len, max_len, max_len, max_len]
    return [base[i % len(base)] for i in range(b)], s, c


@pytest.mark.parametrize("route,dtype,max_len", [("warp", F16, 257), ("warp", BF16, 1100), ("split", F16, 1025),
                                                 ("split", BF16, 3000), ("kv8", F16, 1025), ("kv8", BF16, 3000)])
def test_edge_lengths_and_fully_masked_task_and_split(lib, cuda, route, dtype, max_len):
    hkv, mq = 4, 8
    kv8 = route == "kv8"
    lens, s, c = _edge_tasks(route, max_len, hkv, mq)
    inp = _Inputs(lens, 1, hkv, mq, 128, F16 if kv8 else dtype, split_counts=[s], seed=11)
    for i in range(len(lens)):
        if i % 9 == 6:
            inp.masks[i][:] = False                  # a fully masked task beside live ones
        elif i % 9 == 7:
            inp.masks[i][:, c:2 * c] = False         # its second split fully masked
    out, names = _Kv8Cache(inp).run(inp, max_len, dtype) if kv8 else _run_fp(inp, max_len)
    _assert_route(names, route, s)
    ref = inp.reference()
    assert (ref[6::9] == 0).all()
    _assert_close(out, ref, (KV8_TOL if kv8 else TOL)[dtype], (route, s, c))


@pytest.mark.parametrize("route,bshd", [("warp", True), ("warp", False), ("split", True), ("split", False),
                                        ("kv8", True)])
def test_nothing_past_len_buf_is_read(lib, cuda, route, bshd):
    """Buffers with capacity past each task's length: a NaN tail (kv8: NaN scales, random codes) changes no bit."""
    hkv, mq = 2, 8
    lens, s = _tasks(route, [3000, 17, 64, 1, 255, 33], 1, hkv, mq, None, route == "kv8")
    inp = _Inputs(lens, 1, hkv, mq, 128, F16, split_counts=[s], seed=13)
    outs = []
    for fill in (0.0, float("nan")):
        if route == "kv8":
            out, names = _Kv8Cache(inp, tail=64, fill=fill).run(inp, max(lens), F16)
        else:
            out, names = _run_fp(inp, max(lens), bshd, tail=64, fill=fill)
        _assert_route(names, route, s)
        outs.append(out)
    assert torch.isfinite(outs[1]).all()
    assert torch.equal(outs[0], outs[1])
    _assert_close(outs[1], inp.reference(), (KV8_TOL if route == "kv8" else TOL)[F16])


def _scale_v_rows(inp, keys_of_task, absmax):
    """Rescale the V rows at the given keys of each task (all kv heads) to the given absolute maximum."""
    for i, keys in enumerate(keys_of_task):
        v = inp.v[i].double()
        v[keys] *= absmax / v[keys].abs().amax(-1, keepdim=True)
        inp.v[i] = v.to(inp.v[i].dtype)


@pytest.mark.parametrize("out_dtype", [F16, BF16])
@pytest.mark.parametrize("lens", [[256], [3000, 40], [16384]])
def test_kv8_large_v_rows_stay_finite(lib, cuda, out_dtype, lens):
    """V rows with |v|max = 10000 at the planted keys: the weight e * scale_v of such a row times 2^10 is past the fp16
    range, so the P.V operand has to be normalised by the split's largest weight."""
    hkv, mq = 2, 8
    _, s = _plan(len(lens), 1, hkv, mq, max(lens), kv8=True)
    inp = _Inputs(lens, 1, hkv, mq, 128, F16, split_counts=[s], mask=None, seed=17)
    _scale_v_rows(inp, [_hot_keys(lb, [s]) for lb in lens], 10000.0)
    out, names = _Kv8Cache(inp).run(inp, max(lens), out_dtype)
    _assert_route(names, "kv8", s)
    _assert_close(out, inp.reference(), KV8_TOL[out_dtype])


def test_kv8_tiny_v_rows_beside_unit_rows(lib, cuda):
    """|v|max = 1e-3 at the planted keys, 1.0 elsewhere, in the same splits: neither scale may be flushed."""
    hkv, mq, lens = 2, 8, [2000, 700]
    _, s = _plan(len(lens), 1, hkv, mq, max(lens), kv8=True)
    inp = _Inputs(lens, 1, hkv, mq, 128, F16, split_counts=[s], seed=19)
    hot = [_hot_keys(lb, [s]) for lb in lens]
    _scale_v_rows(inp, [[k for k in range(lb) if k not in set(h)] for lb, h in zip(lens, hot)], 1.0)
    _scale_v_rows(inp, hot, 1e-3)
    out, names = _Kv8Cache(inp).run(inp, max(lens), F16)
    _assert_route(names, "kv8", s)
    _assert_close(out, inp.reference(), KV8_TOL[F16])


def test_kv8_more_than_64_splits_is_unsupported(lib, cuda):
    """70 000 keys need 69 splits of <= 1024 keys: the fp16 cache runs them (test_route_matrix_against_float64), the int8
    cache kernel has at most 64 and must refuse rather than launch."""
    from zhilight_b200 import _lib
    inp = _Inputs([70000], 1, 1, 8, 128, F16, mask=None, seed=23)
    cache = _Kv8Cache(inp)
    assert _cdiv(70000, MAX_RANGE) > MAX_SPLITS

    def call():
        with pytest.raises(_lib.ZLError) as err:
            cache.launch(inp, 70000, F16)
        return err.value.code

    code, names = _launched(call)
    assert code == -2
    assert not any(k in n for n in names for k in KERNEL.values()), names
