"""The variable-length attention kernel (k_varlen_attn, behind ops.varlen_attention: every joined step of the decode
driver) and the MLA decode kernel (k_mla_decode_attn, behind ops.mla_decode_attention) against a float64 reference, at
every tile, key-split and head-group boundary, with the launched kernels checked by the profiler.

Random N(0, 1) keys spread the softmax over hundreds of keys, so one key more or less moves a row by a few per cent and
the whole output by far less.  Here each q head belongs to one of at least three classes, and each class has its own
direction and its own planted keys, whose logit is HOT +- 0.5 against ~N(0, 1) for the rest: the planted keys carry the
softmax, so a kernel that drops or adds one of them, or that mixes up heads of different classes, moves a row by O(1).
Keys are planted where off-by-one errors live (tile and split edges, the causal diagonal), and every case checks on the
float64 reference that removing any one planted key moves some row that sees it by more than the per-row tolerance."""
import numpy as np
import pytest
import torch

from tests import mla_golden
from tests.attn_check import assert_close, launched

pytestmark = pytest.mark.gpu

DEVICE = "cuda:0"
F16, BF16 = torch.float16, torch.bfloat16
F64 = torch.float64
HOT = 15.0          # logit of a planted key, +- SPREAD; the others are ~N(0, 1)
SPREAD = 0.5        # up to ~500 planted keys per head keep each one's removal above 4 x the bf16 per-row bound
CLASSES = 3         # planted-key classes of the q heads that share one kv head (fewer if there are fewer heads)


def _cdiv(a, b):
    return -(-a // b)


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _basis(groups, dim, k, g):
    """(groups, k, dim): k orthonormal directions per group."""
    q, _ = torch.linalg.qr(torch.randn(groups, dim, k, generator=g, device=DEVICE, dtype=F64))
    return q.transpose(1, 2).contiguous()


def _perp(x, u):
    """x (..., groups, dim) minus its components along the orthonormal rows of u (groups, k, dim)."""
    return x - torch.einsum("...gk,gkd->...gd", torch.einsum("...gd,gkd->...gk", x, u), u)


def _hot_logits(n, g):
    return HOT + SPREAD * (2 * torch.rand(n, generator=g, device=DEVICE, dtype=F64) - 1)


def _change(p, ov, oo, vv):
    """Relative change of each row when one key is removed: the softmax without key j gives o' = (o - w_j v_j) / (1 - w_j),
    so |o' - o| / |o| = w_j |o - v_j| / ((1 - w_j) |o|).  p (..., J) the keys' weights in each row, ov (..., J) the dot
    products o . v_j, oo (..., 1) |o|^2, vv (..., J) |v_j|^2.  A key that carries a row almost alone counts as changing it
    (the rest of the row is independent random V); a row that does not see the key does not change."""
    dist = (oo - 2 * ov + vv).clamp_min(0).sqrt()
    ch = p / (1 - p).clamp_min(1e-300) * dist / oo.sqrt().clamp_min(1e-300)
    ch = torch.where(p > 1 - 1e-6, torch.full_like(ch, float("inf")), ch)
    return torch.where(p > 0, ch, torch.zeros_like(ch))


def _assert_sensitive(change, tol, what):
    """change (J,): the largest relative change of any row when planted key j is removed."""
    worst = int(change.argmin())
    assert change[worst].item() > 4 * tol, (what, "planted key", worst, change[worst].item())


def _assert_route(names, kernel, splits, what):
    assert any(kernel in n for n in names), (what, names)
    assert any("k_attn_combine" in n for n in names) == (splits > 1), (what, splits, names)


# ---------------------------------------------------------------------------------------------------------------------
# Variable-length attention (zhilight_b200/csrc/varlen_attn.cu).  Rows come in segments (task, pos0, n): rows at
# positions pos0 .. pos0 + n - 1 of `task`, each attending keys 0 ..= its position.  A CTA holds a tile of `tile_rows`
# query rows of one segment x the `group_heads` q heads of one head group of a kv head (at most 64 MMA rows), and one
# split of 512 keys; splits are merged by k_attn_combine when max_keys needs more than one.
# ---------------------------------------------------------------------------------------------------------------------
VA_MMA_ROWS, VA_MAX_TILE_ROWS, VA_SPLIT_KEYS, VA_KEY_TILE = 64, 16, 512, 64
VA_TOL = {F16: 1e-3, BF16: 6e-3}


def _plan_varlen(m_query):
    """(q heads per group, query rows per tile, head groups per kv head): va_group_heads and va_tile_rows."""
    gh = min(m_query, VA_MMA_ROWS)
    tr = max(1, min(VA_MAX_TILE_ROWS, VA_MMA_ROWS // gh))
    return gh, tr, _cdiv(m_query, gh)


def _va_planted(length, segs, tile_rows):
    """Key 0, the last and first key of every 64-key tile (every 512-key split edge among them), and for every query tile
    of the task's segments the diagonal key of its first and last row (the row at position p plants key p)."""
    hot = {0}
    for e in range(VA_KEY_TILE, length, VA_KEY_TILE):
        hot.update((e - 1, e))
    for pos0, n in segs:
        for r0 in range(0, n, tile_rows):
            hot.update((pos0 + r0, pos0 + min(n, r0 + tile_rows) - 1))
    return sorted(k for k in hot if k < length)


class _Varlen:
    """q (rows, H_kv m_query, d), per-task K / V (len, H_kv, d) and the segment table.  q head m of kv head g is in
    class c = m % CLASSES of g, with direction u[g, c]: q = sqrt(d) u[g, c] + noise orthogonal to every u[g, .].  The
    planted keys of a task go round-robin to the (kv head, class) pairs; a key planted for (g, c) is (HOT + x) u[g, c] in
    kv head g, so that exactly the class-c heads of g see it with logit HOT + x; every other key is noise orthogonal to
    u[g, .]."""

    def __init__(self, segs, hkv, mq, d, dtype, seed):
        g = torch.Generator(device=DEVICE).manual_seed(seed)
        self.segs, self.hkv, self.mq, self.d, self.dtype = segs, hkv, mq, d, dtype
        self.scale = 1.0 / np.sqrt(d)
        _, self.tile_rows, _ = _plan_varlen(mq)
        ntask = max(t for t, _, _ in segs) + 1
        self.lens = [max(p + n for t, p, n in segs if t == task) for task in range(ntask)]
        self.rows = sum(n for _, _, n in segs)
        ncls = min(CLASSES, mq)
        u = _basis(hkv, d, ncls, g)                                           # (hkv, ncls, d)
        cls = torch.arange(mq, device=DEVICE) % ncls
        noise = _perp(torch.randn(self.rows, mq, hkv, d, generator=g, device=DEVICE, dtype=F64), u).transpose(1, 2)
        self.q = (np.sqrt(d) * u[:, cls] + noise).reshape(self.rows, hkv * mq, d).to(dtype)
        pair_kh = torch.arange(hkv * ncls, device=DEVICE) % hkv               # (kv head, class) pairs, round-robin
        pair_c = torch.arange(hkv * ncls, device=DEVICE) // hkv
        self.k, self.v, self.hot = [], [], []
        for task, lb in enumerate(self.lens):
            k = _perp(torch.randn(lb, hkv, d, generator=g, device=DEVICE, dtype=F64), u)
            hot = torch.tensor(_va_planted(lb, [(p, n) for t, p, n in segs if t == task], self.tile_rows),
                               device=DEVICE)
            pair = torch.arange(len(hot), device=DEVICE) % (hkv * ncls)
            k[hot, pair_kh[pair]] = _hot_logits(len(hot), g)[:, None] * u[pair_kh[pair], pair_c[pair]]
            self.k.append(k.to(dtype))
            self.v.append(torch.randn(lb, hkv, d, generator=g, device=DEVICE, dtype=F64).to(dtype))
            self.hot.append(hot)

    def table(self, segs=None):
        out, row0 = [], 0
        for task, pos0, n in segs or self.segs:
            out.append((task, row0, pos0, n))
            row0 += n
        return np.array(out, dtype=np.int32)

    def rows_of(self, seg_ids):
        starts = np.cumsum([0] + [n for _, _, n in self.segs])
        return torch.cat([torch.arange(starts[i], starts[i + 1], device=DEVICE) for i in seg_ids])

    def launch(self, max_keys=None, seg_ids=None):
        from zhilight_b200 import ops
        segs = self.segs if seg_ids is None else [self.segs[i] for i in seg_ids]
        q = self.q if seg_ids is None else self.q[self.rows_of(seg_ids)].contiguous()
        return launched(lambda: ops.varlen_attention(q, self.table(segs), self.k, self.v, self.scale, self.hkv,
                                                     max_keys=max_keys))

    def reference(self):
        """float64 causal attention per segment (oracle/ops.py decode_attention with the causal mask: max seeded -1e20,
        sum + 1e-20), and per task and planted key the largest relative change of a row when that key is removed."""
        hkv, mq, d = self.hkv, self.mq, self.d
        out = torch.zeros(self.rows, hkv * mq, d, dtype=F64, device=DEVICE)
        change = [torch.zeros(len(h), dtype=F64, device=DEVICE) for h in self.hot]
        row0 = 0
        for task, pos0, n in self.segs:
            lb = pos0 + n
            k, v = self.k[task][:lb].to(F64), self.v[task][:lb].to(F64)
            q = self.q[row0:row0 + n].to(F64).view(n, hkv, mq, d)
            s = torch.einsum("qgmd,lgd->qgml", q, k) * self.scale
            late = torch.arange(lb, device=DEVICE)[None, :] > pos0 + torch.arange(n, device=DEVICE)[:, None]
            s = s.masked_fill(late[:, None, None, :], float("-inf"))
            e = torch.exp(s - s.amax(-1, keepdim=True).clamp_min(-1e20))
            p = e / (e.sum(-1, keepdim=True) + 1e-20)
            o = torch.einsum("qgml,lgd->qgmd", p, v)
            out[row0:row0 + n] = o.reshape(n, hkv * mq, d)
            hot = self.hot[task]
            vh = v[hot]                                                      # (J, hkv, d)
            ch = _change(p[..., hot], torch.einsum("qgmd,jgd->qgmj", o, vh), (o * o).sum(-1, keepdim=True),
                         (vh * vh).sum(-1).t()[None, :, None, :])
            change[task] = torch.maximum(change[task], ch.amax((0, 1, 2)))
            row0 += n
        return out, torch.cat(change)


# Segment sets (task, pos0, n).  n is no multiple of any tile height above 1 (37, 23, 151 and 12 leave a part tile).
VA_SETS = {
    "decode": [(0, 0, 1), (1, 63, 1), (2, 64, 1), (3, 511, 1), (4, 512, 1), (5, 1023, 1)],
    "chunk0": [(0, 0, 151)],
    "span": [(0, 507, 37), (1, 1021, 23)],                     # start 5 and 3 rows before a split edge and cross it
    "mixed": [(0, 40, 1), (1, 700, 1), (2, 0, 37), (3, 515, 1), (4, 300, 20)],
    "long": [(0, 20470, 12), (1, 0, 1)],                       # 41 splits; the chunk crosses the 40th split edge
}
VA_OTHERS = ["decode", "chunk0", "mixed", "long"]
# m_query and kv heads: tile rows 16 16 16 12 9 8 5 4 2 1 1 1 1, and two head groups at 96 (64 + 32) and 128 (64 + 64)
VA_HEADS = [(1, 4), (2, 4), (3, 4), (5, 2), (7, 2), (8, 2), (12, 2), (16, 2), (24, 2), (40, 2), (64, 1), (96, 1),
            (128, 1)]
VA_TYPES = [(F16, 64), (BF16, 64), (F16, 128), (BF16, 128)]
# every m_query: "span" and two other sets, with both dtypes; every set: all four (dtype, d)
VA_MATRIX = []
for _i, (_mq, _hkv) in enumerate(VA_HEADS):
    for _j, _set in enumerate(["span", VA_OTHERS[(2 * _i) % 4], VA_OTHERS[(2 * _i + 1) % 4]]):
        VA_MATRIX.append((_mq, _hkv) + VA_TYPES[(3 * _i + _j + _i // 2) % 4] + (_set,))


def _va_id(c):
    mq, hkv, dt, d, name = c
    gh, tr, hg = _plan_varlen(mq)
    return "%s-d%d-mq%d-hkv%d-rows%d-hg%d-%s" % ("f16" if dt == F16 else "bf16", d, mq, hkv, tr, hg, name)


@pytest.mark.parametrize("case", VA_MATRIX, ids=[_va_id(c) for c in VA_MATRIX])
def test_varlen_boundaries_against_float64(lib, cuda, case):
    mq, hkv, dtype, d, name = case
    tol = VA_TOL[dtype]
    inp = _Varlen(VA_SETS[name], hkv, mq, d, dtype, seed=mq + d + len(name))
    ref, change = inp.reference()
    _assert_sensitive(change, tol, name)

    exact = max(inp.lens)
    out, names = inp.launch()
    _assert_route(names, "k_varlen_attn<", _cdiv(exact, VA_SPLIT_KEYS), exact)
    assert_close(out, ref, tol, exact)

    # more, empty, splits: split s always covers keys [512 s, 512 s + 512), so no row's bits may change
    for mk in sorted({2 * exact, 4 * exact, max(8192, 4 * exact)}):
        wide, names = inp.launch(max_keys=mk)
        _assert_route(names, "k_varlen_attn<", _cdiv(mk, VA_SPLIT_KEYS), mk)
        assert torch.equal(wide, out), mk

    # the segments that need one split, launched alone (direct write), against their rows in the launch above
    short = [i for i, (_, p, n) in enumerate(inp.segs) if p + n <= VA_SPLIT_KEYS]
    if short:
        alone, names = inp.launch(seg_ids=short)
        _assert_route(names, "k_varlen_attn<", 1, "alone")
        rows = inp.rows_of(short)
        assert torch.equal(alone, out[rows]), short
        assert_close(alone, ref[rows], tol, "alone")


# ---------------------------------------------------------------------------------------------------------------------
# MLA decode attention (zhilight_b200/csrc/mla_attn.cu).  One CTA = (key split, tile of 64 (query, head) rows, task);
# row r of a task is query r / H, head r % H, so a tile starts mid-query whenever 64 is no multiple of H.  Task b's
# split s covers keys [s chunk, s chunk + chunk), chunk = round64(cdiv(len_b, splits)); the split count comes from the
# SM count (mla_num_splits), which _plan_mla restates.
# ---------------------------------------------------------------------------------------------------------------------
MLA_D, MLA_DV, MLA_ROPE = 576, 512, 64
MLA_ROWS, MLA_MIN_SPLIT_KEYS, MLA_MAX_SPLITS, MLA_KEY_TILE = 64, 256, 64, 64
MLA_TOL = {F16: mla_golden.TOL["f16"], BF16: mla_golden.TOL["bf16"]}
MLA_SCALE = 1.0 / np.sqrt(192.0)
MLA_LATENT_Q = 0.2     # q's random part in columns 0..511: those columns add ~N(0, 0.33^2) to every logit


def _plan_mla(b, len_q, h, max_len_buf):
    """Key splits of zl_mla_decode_attention: one CTA per SM, splits only while b x row tiles leaves SMs idle."""
    fit = _sm_count() // (b * _cdiv(len_q * h, MLA_ROWS))
    return 1 if fit < 1 else min(fit, _cdiv(max_len_buf, MLA_MIN_SPLIT_KEYS), MLA_MAX_SPLITS)


def _mla_chunks(len_buf, splits):
    chunk = _cdiv(_cdiv(len_buf, splits), MLA_KEY_TILE) * MLA_KEY_TILE
    return [(k0, min(len_buf, k0 + chunk)) for k0 in range(0, len_buf, chunk)]


def _mla_planted(len_buf, split_counts):
    """Key 0, len_buf - 1, and for each split count every chunk's first and last key and the last and first key of
    each of its 64-key tiles."""
    hot = {0, len_buf - 1}
    for s in split_counts:
        for k0, k1 in _mla_chunks(len_buf, s):
            hot.update((k0, k1 - 1))
            for e in range(k0 + MLA_KEY_TILE, k1, MLA_KEY_TILE):
                hot.update((e - 1, e))
    return sorted(hot)


def _bucket(max_len):
    """Power-of-two length bucket, at least 256."""
    b = 256
    while b < max_len:
        b <<= 1
    return b


class _Mla:
    """q (B, len_q, H, 576) and per-task latent caches (len, 576), K = the whole row, V = its first 512 columns.
    Head h is in class c = h % CLASSES with direction u[c] in the rope columns 512..575 (K only): q's rope part is
    u[c] / scale plus small orthogonal noise, its latent part small noise; a planted key's rope part is (HOT + x) u[c],
    every other key's rope part noise orthogonal to u[.], and every key's latent (V) part independent N(0, 1).  Masks
    (len_q, len_b) bool per task: "none", "causal" (query i sees keys < len - len_q + i + 1) or "holes" (1/8 of the
    keys per query; each planted key stays visible to at least one query, and which ones differ per query)."""

    def __init__(self, lens, len_q, h, dtype, mask, split_counts, seed):
        g = torch.Generator(device=DEVICE).manual_seed(seed)
        self.lens, self.len_q, self.h, self.dtype, self.mask = list(lens), len_q, h, dtype, mask
        b = len(lens)
        ncls = min(CLASSES, h)
        u = _basis(1, MLA_ROPE, ncls, g)                                       # (1, ncls, 64)
        cls = torch.arange(h, device=DEVICE) % ncls
        q = torch.empty(b, len_q, h, MLA_D, dtype=F64, device=DEVICE)
        q[..., :MLA_DV] = MLA_LATENT_Q * torch.randn(b, len_q, h, MLA_DV, generator=g, device=DEVICE, dtype=F64)
        q[..., MLA_DV:] = u[0, cls] / MLA_SCALE + MLA_LATENT_Q * _perp(
            torch.randn(b, len_q, h, 1, MLA_ROPE, generator=g, device=DEVICE, dtype=F64), u)[..., 0, :]
        self.q = q.to(dtype)
        self.kv, self.masks, self.hot = [], [], []
        for lb in self.lens:
            kv = torch.randn(lb, MLA_D, generator=g, device=DEVICE, dtype=F64)
            kv[:, MLA_DV:] = _perp(kv[:, None, MLA_DV:], u)[:, 0]
            hot = torch.tensor(_mla_planted(lb, split_counts), device=DEVICE)
            rank = torch.arange(len(hot), device=DEVICE)
            kv[hot, MLA_DV:] = _hot_logits(len(hot), g)[:, None] * u[0, rank % ncls]
            self.kv.append(kv.to(dtype))
            self.hot.append(hot)
            keys = torch.arange(lb, device=DEVICE)
            if mask == "causal":
                m = keys[None, :] < lb - len_q + 1 + torch.arange(len_q, device=DEVICE)[:, None]
            elif mask == "holes":
                m = torch.rand(len_q, lb, generator=g, device=DEVICE) >= 0.125
                m[rank % len_q, hot] = True
            else:
                m = None
            self.masks.append(m)

    def launch(self, max_len_buf):
        from zhilight_b200 import ops
        mask = None if self.mask == "none" else torch.cat([m.reshape(-1) for m in self.masks]).to(torch.int8)
        lens = torch.tensor(self.lens, dtype=torch.int32, device=DEVICE)
        return launched(lambda: ops.mla_decode_attention(self.q, lens, self.kv, mask, MLA_SCALE, max_len_buf))

    def reference(self):
        """float64 (B, len_q, H, 512) and per task and planted key the largest relative change of a row when that key
        is removed."""
        out = torch.zeros(len(self.lens), self.len_q, self.h, MLA_DV, dtype=F64, device=DEVICE)
        change = []
        for i, lb in enumerate(self.lens):
            kv = self.kv[i].to(F64)
            s = torch.einsum("qhd,ld->qhl", self.q[i].to(F64), kv) * MLA_SCALE
            if self.masks[i] is not None:
                s = s.masked_fill(~self.masks[i][:, None, :], float("-inf"))
            e = torch.exp(s - s.amax(-1, keepdim=True).clamp_min(-1e20))
            p = e / (e.sum(-1, keepdim=True) + 1e-20)
            v = kv[:, :MLA_DV]
            o = p @ v
            out[i] = o
            vh = v[self.hot[i]]
            ch = _change(p[..., self.hot[i]], o @ vh.t(), (o * o).sum(-1, keepdim=True), (vh * vh).sum(-1))
            change.append(ch.amax((0, 1)))
        return out, torch.cat(change)


def _mla_batch(base, len_q, h, splits):
    """Tasks cycled from `base` until _plan_mla gives `splits` (an int, or "many" for >= 3) at max_len_buf = max(lens).
    "c" and "c+1" in `base` stand for the longest task's split chunk and one more key."""
    top = max(x for x in base if isinstance(x, int))
    for b in range(len(base), 512):
        s = _plan_mla(b, len_q, h, top)
        if s == splits or (splits == "many" and s >= 3):
            chunk = _mla_chunks(top, s)[0][1]
            named = {"c": chunk, "c+1": min(top, chunk + 1)}
            return [named.get(x, x) for x in (base[i % len(base)] for i in range(b))], s
    raise AssertionError("no batch of %s reaches %s splits" % (base, splits))


EDGE = [1, 63, 64, 65, 511, 513, 1025]
RAGGED = [1, 63, 64, 65, "c", "c+1"]
# (H, len_q, mask, tasks, splits at max_len_buf = max(lens), dtype).  H 20 x len_q 4, 48 x 3, 100 x 1 and 128 x 4 have
# row tiles that start in the middle of a query's heads; B = 33 at H = 128, len_q = 2 fills every SM with row tiles and
# runs unsplit even with a 16384-key task.
MLA_MATRIX = [
    (1, 1, "none", [16384], 64, F16),
    (1, 3, "holes", [5000] + RAGGED, "many", BF16),
    (3, 2, "causal", [3000] + RAGGED, "many", F16),
    (3, 4, "holes", [200, 64, 1, 65], 1, BF16),
    (16, 4, "holes", [4000] + RAGGED, 2, F16),
    (20, 4, "holes", [2000, 63, "c", "c+1", 1], "many", BF16),
    (48, 3, "causal", [6000, 65, "c", "c+1", 1, 64], "many", F16),
    (100, 1, "none", [16384], "many", BF16),     # 64 splits on 132 SMs
    (100, 1, "holes", [700, 1, 63, 64, 65], "many", F16),
    (128, 4, "holes", [9000, 1, "c", "c+1"], "many", BF16),
    (128, 2, "causal", [16384] + [EDGE[i % 7] for i in range(32)], 1, F16),
    (128, 1, "none", [3000, 64, 1], 2, BF16),
]


def _mla_id(c):
    h, len_q, mask, base, splits, dt = c
    return "%s-h%d-q%d-%s-L%d-s%s" % ("f16" if dt == F16 else "bf16", h, len_q, mask,
                                       max(x for x in base if isinstance(x, int)), splits)


@pytest.mark.parametrize("case", MLA_MATRIX, ids=[_mla_id(c) for c in MLA_MATRIX])
def test_mla_boundaries_against_float64(lib, cuda, case):
    h, len_q, mask, base, splits, dtype = case
    tol = MLA_TOL[dtype]
    lens, s = _mla_batch(base, len_q, h, splits)
    top = max(lens)
    sizes = [top, _bucket(top), max(16384, 2 * top)]
    plans = [_plan_mla(len(lens), len_q, h, m) for m in sizes]
    assert plans[0] == s
    inp = _Mla(lens, len_q, h, dtype, mask, plans, seed=h + len_q + len(lens))
    ref, change = inp.reference()
    _assert_sensitive(change, tol, (h, len_q, mask))
    for m, sp in zip(sizes, plans):
        out, names = inp.launch(m)
        _assert_route(names, "k_mla_decode_attn<", sp, (m, sp))
        assert_close(out, ref, tol, (m, sp))
