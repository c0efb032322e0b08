"""Every exact-integer W4A16 kernel (tests/w4_int_cases.py) against the float64 restatement of its arithmetic
(tests/w4_int_oracle.py): each output element within one fp16 ulp (plus the fp32 rounding bound) of the emulation and
within the quantisation bound of the exact GEMM; the int8-KV epilogue bit for bit equal to its fp16 rows quantised; and the
tensor-parallel exchange kernels on a one-rank comm, whose push and reduce-in run the same tags, slots and rounding points
as at two ranks (only the peer mapping differs)."""
import ctypes

import numpy as np
import pytest
import torch

from tests import w4_int_cases as C
from tests import w4_int_oracle as O

pytestmark = pytest.mark.gpu

LEN = 12            # cache rows per task
SENT16 = -7.0       # fp16 cache sentinel


def _dev(a, cuda):
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


def _pack(q, z, s, sym, cuda):
    from zhilight_b200 import ops
    qw = _dev(O.pack_k_major(q).view(np.int32), cuda)
    return ops.w4_pack(qw, _dev(z, cuda), _dev(s, cuda), 128, sym, None, variant=1)


def _pack_flag(mc, n, k, tp):
    from zhilight_b200 import _lib
    out = (ctypes.c_int * 9)()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert _lib.load().zl_w4_v3_plan(mc, n, k, tp, sms, out) == 0, (mc, n, k, tp)
    return bool(out[5])


def _launch(x, packed, n, k, epi=0, bias=None, residual=None, y=None, ln_w=None, rope=None, kv8=None, k_perm=None,
            tp=None):
    """zl_w4a16_gemm_fused on the ZLW4I layout; tp = dict(comm, mode, index, h_out)"""
    from zhilight_b200 import _lib, ops
    a = _lib.W4FusedArgs()
    m = x.shape[0]
    a.x, a.ldx, a.packed = x.data_ptr(), x.stride(0), packed.data_ptr()
    a.bias, a.residual = ops._dp(bias), ops._dp(residual)
    a.M, a.N, a.K, a.group_size, a.epilogue, a.variant = m, n, k, 128, epi, 1
    a.ln_weight, a.eps = ops._dp(ln_w), 1e-5
    a.k_perm = ops._dp(k_perm)
    keep, q = [], None
    if epi == ops.EPI_QKV_ROPE:
        q = torch.empty((m, rope["hq"] * rope["d"]), dtype=torch.float16, device=x.device)
        tabs = [ops._ptr_table(rope[b], x.device) for b in ("k_bufs", "v_bufs")]
        keep += tabs
        a.cos, a.sin, a.q_out = rope["cos"].data_ptr(), rope["sin"].data_ptr(), q.data_ptr()
        a.token_batch, a.placement = rope["tb"].data_ptr(), rope["pl"].data_ptr()
        a.k_addrs, a.v_addrs = tabs[0].data_ptr(), tabs[1].data_ptr()
        a.num_heads, a.num_kv_heads, a.dim_head = rope["hq"], rope["hkv"], rope["d"]
        if kv8 is not None:
            st = [ops._ptr_table(kv8[b], x.device) for b in ("sk", "sv")]
            keep += st
            a.kv_int8, a.scale_k_addrs, a.scale_v_addrs = 1, st[0].data_ptr(), st[1].data_ptr()
            a.kv8_stage, a.kv8_counters = kv8["stage"].data_ptr(), kv8["cnt"].data_ptr()
    a.y = ops._dp(y)
    if tp is not None:
        a.tp_comm, a.tp_mode, a.tp_index = tp["comm"].handle, tp["mode"], tp["index"]
        a.tp_h_out = ops._dp(tp.get("h_out"))
    rc = _lib.load().zl_w4a16_gemm_fused(ctypes.byref(a), ops._stream())
    torch.cuda.synchronize()
    return rc, q


def _close(got, want, tol, ok, what):
    """every element of the tokens `ok` within tol of want; the others (poisoned tokens) NaN"""
    got = np.asarray(got, dtype=np.float64)
    err = np.abs(got - want)
    bad = ~(err <= tol) & ok.reshape((-1,) + (1,) * (got.ndim - 1))
    assert not bad.any(), (what, np.argwhere(bad)[:5].tolist(), got[bad][:5], np.asarray(want)[bad][:5], tol[bad][:5])
    assert np.isnan(got[~ok]).all(), what


class _Qkv:
    """the QKV_ROPE epilogue's inputs and the caches it writes: tokens interleave 3 tasks, every 4th token is not placed"""

    def __init__(self, cuda, m, n, kv8):
        from zhilight_b200 import ops
        self.hq, self.hkv, self.d = C.qkv_heads(n)
        pos = torch.tensor([(5 * i) % 11 for i in range(m)], dtype=torch.int32, device=cuda)
        self.cos, self.sin = ops.rope_cos_sin(pos, self.d, 10000.0)
        self.tb_h = [i % 3 for i in range(m)]
        self.pl_h = [-1 if i % 4 == 3 else i // 3 for i in range(m)]
        shape = (LEN, self.hkv, self.d)
        if kv8:
            self.k = [torch.full(shape, 77, dtype=torch.uint8, device=cuda) for _ in range(3)]
            self.v = [torch.full(shape, 77, dtype=torch.uint8, device=cuda) for _ in range(3)]
            self.kv8 = dict(sk=[torch.full(shape[:2], -1.0, device=cuda) for _ in range(3)],
                            sv=[torch.full(shape[:2], -1.0, device=cuda) for _ in range(3)],
                            stage=torch.empty(m, 2, self.hkv, self.d, dtype=torch.float16, device=cuda),
                            cnt=torch.zeros(m, 2, self.hkv, dtype=torch.int32, device=cuda))
        else:
            self.k = [torch.full(shape, SENT16, dtype=torch.float16, device=cuda) for _ in range(3)]
            self.v = [torch.full(shape, SENT16, dtype=torch.float16, device=cuda) for _ in range(3)]
            self.kv8 = None
        self.rope = dict(cos=self.cos, sin=self.sin, tb=torch.tensor(self.tb_h, dtype=torch.int32, device=cuda),
                         pl=torch.tensor(self.pl_h, dtype=torch.int32, device=cuda), k_bufs=self.k, v_bufs=self.v,
                         hq=self.hq, hkv=self.hkv, d=self.d)

    def written(self):
        return {(t, p) for t, p in zip(self.tb_h, self.pl_h) if p >= 0}

    def check_fp16(self, q, r, ok):
        """q and the cached K / V rows against the emulation (and the exact GEMM) through the epilogue"""
        cs, sn = self.cos.cpu().numpy(), self.sin.cpu().numpy()
        qn = q.float().cpu().numpy().reshape(q.shape[0], self.hq, self.d)
        for v, dv, what in ((r["v"], r["f32"], "emulation"), (r["exact"], r["f32"] + r["qb"], "exact")):
            out, tol = O.epi_qkv(v, dv, cs, sn, self.hq, self.hkv, self.d)
            _close(qn, out[:, :self.hq], tol[:, :self.hq], ok, "q vs " + what)
            for i, (b, p) in enumerate(zip(self.tb_h, self.pl_h)):
                if p < 0:
                    continue
                for bufs, h0 in ((self.k, self.hq), (self.v, self.hq + self.hkv)):
                    row = bufs[b][p].float().cpu().numpy()[None]
                    _close(row, out[i:i + 1, h0:h0 + self.hkv], tol[i:i + 1, h0:h0 + self.hkv], ok[i:i + 1],
                           "cache row vs " + what)
        for b in range(3):
            for p in range(LEN):
                if (b, p) not in self.written():
                    assert bool((self.k[b][p] == SENT16).all()) and bool((self.v[b][p] == SENT16).all()), (b, p)

    def check_int8(self, fp16):
        """codes and scales = zl_int8_quant_rows_u8 of the fp16 epilogue's rows, bit for bit; other rows untouched"""
        from zhilight_b200 import _lib
        assert int(self.kv8["cnt"].abs().sum()) == 0, "counters must be back at zero"
        for b in range(3):
            for bufs16, bufs8, scales in ((fp16.k, self.k, self.kv8["sk"]), (fp16.v, self.v, self.kv8["sv"])):
                r16 = bufs16[b].reshape(-1, self.d).contiguous()
                codes = torch.empty(r16.shape, dtype=torch.uint8, device=r16.device)
                sc = torch.empty(r16.shape[0], dtype=torch.float32, device=r16.device)
                _lib.call("zl_int8_quant_rows_u8", r16.data_ptr(), codes.data_ptr(), sc.data_ptr(), r16.shape[0], self.d,
                          0, None)
                torch.cuda.synchronize()
                codes, sc = codes.reshape(bufs8[b].shape), sc.reshape(scales[b].shape)
                for p in range(LEN):
                    if (b, p) in self.written():
                        assert torch.equal(bufs8[b][p], codes[p]) and torch.equal(scales[b][p], sc[p]), (b, p)
                    else:
                        assert bool((bufs8[b][p] == 77).all()) and bool((scales[b][p] == -1.0).all()), (b, p)


def _check_dense(y, epi, r, ok, residual=None):
    kw = dict(residual=residual)
    for v, dv, what in ((r["v"], r["f32"], "emulation"), (r["exact"], r["f32"] + r["qb"], "exact")):
        out, tol = O.epilogue(epi, v, dv, **kw)
        _close(y.float().cpu().numpy(), out, tol, ok, what)


@pytest.mark.parametrize("case", C.CASES, ids=["-".join(map(str, c)) for c in C.CASES])
def test_kernel_against_float64(lib, cuda, case):
    from zhilight_b200 import ops
    mc, n, k, epi, norm, fu, sym, kind = case
    seed = C.CASES.index(case)
    rng = np.random.default_rng(1000 + seed)
    q, z, s = C.weights(n, k, sym, headroom=kind == "headroom", seed=seed)
    x = C.activations(kind, mc, k, seed=seed)
    ln_w = (1 + 0.1 * rng.standard_normal(k)).astype(np.float16) if norm else None
    k_perm = rng.permutation(k).astype(np.int32) if fu == 1 else None
    bias = (0.1 * rng.standard_normal(n)).astype(np.float16) if epi in ("res", "qkv") else None
    packed = _pack(q, z, s, sym, cuda)
    r = O.gemm(x, q, z, s, pack=_pack_flag(mc, n, k, 0), ln_w=ln_w, k_perm=k_perm, bias=bias)
    ok = ~r["poison"]
    assert list(np.flatnonzero(r["poison"])) == ([0, 1] if kind == "nonfinite" else [])
    d = lambda a: None if a is None else _dev(a, cuda)
    xd = _dev(x, cuda)
    if epi == "qkv":
        qk16 = _Qkv(cuda, mc, n, False)
        rc, q16 = _launch(xd, packed, n, k, ops.EPI_QKV_ROPE, bias=d(bias), ln_w=d(ln_w), rope=qk16.rope, k_perm=d(k_perm))
        assert rc == 0
        qk16.check_fp16(q16, r, ok)
        if fu == 2:
            qk8 = _Qkv(cuda, mc, n, True)
            for _ in range(2):     # back to back: the counters are left at zero
                rc, q8 = _launch(xd, packed, n, k, ops.EPI_QKV_ROPE, bias=d(bias), ln_w=d(ln_w), rope=qk8.rope, kv8=qk8.kv8)
                assert rc == 0 and torch.equal(q8, q16)
                qk8.check_int8(qk16)
        return
    code = dict(none=ops.EPI_NONE, res=ops.EPI_RESIDUAL, swiglu=ops.EPI_SWIGLU)[epi]
    res = rng.standard_normal((mc, n)).astype(np.float16) if epi == "res" else None
    y = torch.full((mc, n // 2 if epi == "swiglu" else n), SENT16, dtype=torch.float16, device=cuda)
    rc, _ = _launch(xd, packed, n, k, code, bias=d(bias), residual=d(res), y=y, ln_w=d(ln_w), k_perm=d(k_perm))
    assert rc == 0
    _check_dense(y, epi, r, ok, residual=res)


# ---------------------------------------------------------------- the exchange kernels on a one-rank comm
class _Comm:
    """a one-rank TPComm and a view of its symmetric buffer (comm_dev.cuh restated): [2 parities][ws sources][slot] payload,
    [ws][64] uint64 flags, then the tagged region [2 parities][ws sources][2 * slot] of {2 x fp16, tag} words"""

    def __init__(self, cuda, max_elems):
        from zhilight_b200 import _lib, dist as zdist
        self.c = zdist.TPComm(max_elems, 0, 1)
        self.handle = self.c.handle
        base, nbytes = ctypes.c_void_p(), ctypes.c_size_t()
        _lib.call("zl_comm_local_buffer", self.handle, ctypes.byref(base), ctypes.byref(nbytes))
        self.slot = ((max_elems + 31) // 32 * 32 * 2 + 127) // 128 * 128
        self.ll = 2 * self.slot + 64 * 8
        assert nbytes.value == self.ll + 2 * 2 * self.slot
        self.words = torch.as_tensor(zdist._DeviceArray(base.value, (nbytes.value // 4,), "<i4"), device=cuda)
        self.step = 0

    def begin_step(self):
        from zhilight_b200 import _lib, ops
        _lib.call("zl_comm_ll_begin_step", self.handle, ops._stream())
        self.step += 1

    @staticmethod
    def tag(step, index):
        return ((step << 9) + index + 1) & 0xFFFFFFFF

    def parity(self, index):
        return ((index & 511) + ((index >> 9) & 1) * (self.step & 1)) & 1

    def region(self, parity):
        """word range [a, b) of the tagged slot of `parity` (source 0)"""
        a = (self.ll + parity * 2 * self.slot) // 4
        return a, a + 2 * self.slot // 4

    def fill(self, value=-1):
        torch.cuda.synchronize()
        self.words[self.ll // 4:] = value
        torch.cuda.synchronize()

    def read(self, parity):
        a, b = self.region(parity)
        return self.words[a:b].cpu().numpy().view(np.uint32).reshape(-1, 2)

    def write(self, parity, halves, tag):
        """tagged words carrying the fp16 values `halves` (flattened, even count) into the slot of `parity`"""
        a, _ = self.region(parity)
        w = np.empty((halves.size // 2, 2), np.uint32)
        w[:, 0] = np.ascontiguousarray(halves, dtype=np.float16).reshape(-1).view(np.uint32)
        w[:, 1] = tag
        torch.cuda.synchronize()
        self.words[a:a + w.size] = torch.from_numpy(w.reshape(-1).view(np.int32)).to(self.words.device)
        torch.cuda.synchronize()

    def close(self):
        torch.cuda.synchronize()
        self.c.close()


def _bits(t):
    return t.cpu().numpy().view(np.uint16)


@pytest.mark.parametrize("case", C.TP_CASES, ids=["-".join(map(str, c)) for c in C.TP_CASES])
def test_exchange_kernels_on_one_rank(lib, cuda, case):
    from zhilight_b200 import ops
    mc, n, k = case
    seed = 100 + C.TP_CASES.index(case)
    rng = np.random.default_rng(seed)
    q, z, s = C.weights(n, k, False, seed=seed)
    packed = _pack(q, z, s, False, cuda)
    ln_w = (1 + 0.1 * rng.standard_normal(k)).astype(np.float16)
    comm = _Comm(cuda, 16 * 8192)
    try:
        # push (fusion 5) first: it confirms the slot, the tag and the parity this restatement writes for the consumers
        for norm, index in ((0, 2), (1, 3 | 512), (0, 4 | 512), (1, 7)):
            comm.fill()
            comm.begin_step()
            x = C.activations("rand", mc, k, seed=seed + index)
            lw = _dev(ln_w, cuda) if norm else None
            y0 = torch.empty(mc, n, dtype=torch.float16, device=cuda)
            assert _launch(_dev(x, cuda), packed, n, k, y=y0, ln_w=lw)[0] == 0
            r = O.gemm(x, q, z, s, pack=_pack_flag(mc, n, k, 2), ln_w=ln_w if norm else None)
            _check_dense(y0, "none", r, ~r["poison"])
            assert _launch(_dev(x, cuda), packed, n, k, ln_w=lw, tp=dict(comm=comm, mode=2, index=index))[0] == 0
            torch.cuda.synchronize()
            par = comm.parity(index)
            got = comm.read(par)
            nw = mc * n // 2
            assert (got[:nw, 1] == comm.tag(comm.step, index & 511)).all(), (norm, index)
            assert np.array_equal(got[:nw, 0], _bits(y0).reshape(-1).view(np.uint32)), (norm, index)
            assert (got[nw:] == 0xFFFFFFFF).all() and (comm.read(1 - par) == 0xFFFFFFFF).all(), (norm, index)
        # reduce-in (fusions 3 and 4): the host plays the producer; the other parity holds the same tag and other values
        for norm, index, epi in ((0, 1, "swiglu"), (1, 2 | 512, "swiglu"), (0, 5, "qkv"), (1, 6 | 512, "qkv")):
            fp16 = None
            for kv8 in (False, True) if epi == "qkv" else (False,):
                comm.fill()
                comm.begin_step()
                x = C.activations("rand", mc, k, seed=seed + 7 * index)
                part = C.activations("rand", mc, k, seed=seed + 7 * index + 1)
                decoy = C.activations("rand", mc, k, seed=seed + 7 * index + 2)
                tag, par = comm.tag(comm.step, index & 511), comm.parity(index)
                comm.write(par, part, tag)
                comm.write(1 - par, decoy, tag)
                h = (part.astype(np.float32) + x.astype(np.float32)).astype(np.float16)
                h_out = torch.full((mc, k), SENT16, dtype=torch.float16, device=cuda)
                tp = dict(comm=comm, mode=1, index=index, h_out=h_out)
                lw = _dev(ln_w, cuda) if norm else None
                r = O.gemm(h, q, z, s, pack=_pack_flag(mc, n, k, 1), ln_w=ln_w if norm else None)
                ok = ~r["poison"]
                if epi == "swiglu":
                    y = torch.empty(mc, n // 2, dtype=torch.float16, device=cuda)
                    assert _launch(_dev(x, cuda), packed, n, k, ops.EPI_SWIGLU, y=y, ln_w=lw, tp=tp)[0] == 0
                    _check_dense(y, "swiglu", r, ok)
                else:
                    qk = _Qkv(cuda, mc, n, kv8)
                    rc, qo = _launch(_dev(x, cuda), packed, n, k, ops.EPI_QKV_ROPE, ln_w=lw, rope=qk.rope, kv8=qk.kv8, tp=tp)
                    assert rc == 0
                    if kv8:
                        assert torch.equal(qo, fp16[0])
                        qk.check_int8(fp16[1])
                    else:
                        qk.check_fp16(qo, r, ok)
                        fp16 = (qo, qk)
                assert np.array_equal(_bits(h_out), h.view(np.uint16)), (norm, index, epi, kv8)
    finally:
        comm.close()


@pytest.mark.parametrize("exchanges", [2, 3])
@pytest.mark.parametrize("mc", [2, 9])
def test_fused_chain_equals_unfused(lib, cuda, mc, exchanges):
    """the decode layer's exchanges for 3 steps -- o_proj push, gate_up reduce-in (SWIGLU), down push, next qkv reduce-in
    (and, with 3 exchanges a step, one more push / reduce-in pair, so the slot parity flips from step to step) -- equal the
    tp_mode 0 GEMMs with zl_allreduce_one_shot(partial, residual) on the same comm, bit for bit"""
    from zhilight_b200 import ops
    dm, ff, nq = 1024, 1536, 1536
    rng = np.random.default_rng(mc * 10 + exchanges)
    mats = {}
    for name, (n, k) in dict(o=(dm, dm), gu=(2 * ff, dm), down=(dm, ff), qkv=(nq, dm)).items():
        q, z, s = C.weights(n, k, False, seed=len(mats) + 50)
        mats[name] = (_pack(q, z, s, False, cuda), n, k)
    ln1, ln2 = (_dev((1 + 0.1 * rng.standard_normal(dm)).astype(np.float16), cuda) for _ in range(2))
    odd = 512 if exchanges % 2 else 0
    comm = _Comm(cuda, 16 * 4096)
    try:
        def gemm(name, x, epi=0, ln=None, tp=None):
            packed, n, k = mats[name]
            y = torch.empty(x.shape[0], n // 2 if epi == ops.EPI_SWIGLU else n, dtype=torch.float16, device=cuda)
            assert _launch(x, packed, n, k, epi, y=None if tp and tp["mode"] == 2 else y, ln_w=ln, tp=tp)[0] == 0
            return y

        def run(fused):
            resid = _dev(C.activations("rand", mc, dm, seed=1), cuda)
            attn = _dev(C.activations("rand", mc, dm, seed=2), cuda)
            outs = []
            for _ in range(3):
                if fused:
                    comm.begin_step()
                pairs = [("o", "gu", ops.EPI_SWIGLU, ln1), ("down", "qkv", 0, ln2), ("o", "qkv", 0, ln2)][:exchanges]
                src = attn
                for j, (push, consume, epi, ln) in enumerate(pairs):
                    if push == "down":
                        src = outs[-1]
                    elif j == 2:
                        src = outs[-1][:, :dm].contiguous()
                    if fused:
                        gemm(push, src, tp=dict(comm=comm, mode=2, index=j | odd))
                        h = torch.empty(mc, dm, dtype=torch.float16, device=cuda)
                        y = gemm(consume, resid, epi, ln, tp=dict(comm=comm, mode=1, index=j | odd, h_out=h))
                    else:
                        h = comm.c.allreduce(gemm(push, src), resid)
                        torch.cuda.synchronize()
                        y = gemm(consume, h, epi, ln)
                    outs += [h.clone(), y]
                    resid = h
                attn = outs[-1][:, :dm].contiguous()
            return outs

        unfused = run(False)
        fused = run(True)
        assert len(fused) == len(unfused) == 3 * exchanges * 2
        for i, (a, b) in enumerate(zip(fused, unfused)):
            assert torch.isfinite(b.float()).all()
            assert torch.equal(a, b), i
    finally:
        comm.close()


def test_exchange_refusals(lib, cuda):
    """tp_mode 1 needs the activation row unpadded (ldx == K) and M * K fp16 values in a slot; tp_mode 2 M * N"""
    mc, n, k = 2, 2048, 1024
    q, z, s = C.weights(n, k, False, seed=3)
    packed = _pack(q, z, s, False, cuda)
    comm = _Comm(cuda, 1024)
    try:
        xp = torch.zeros(mc, k + 64, dtype=torch.float16, device=cuda)
        h = torch.empty(mc, k, dtype=torch.float16, device=cuda)
        y = torch.empty(mc, n, dtype=torch.float16, device=cuda)
        big = _Comm(cuda, 16 * 4096)
        try:
            rc, _ = _launch(xp[:, :k], packed, n, k, y=y, tp=dict(comm=big, mode=1, index=0, h_out=h))
            assert rc == -1
        finally:
            big.close()
        x = torch.zeros(mc, k, dtype=torch.float16, device=cuda)
        assert _launch(x, packed, n, k, y=y, tp=dict(comm=comm, mode=1, index=0, h_out=h))[0] == -1   # 2 * 1024 > 1024
        assert _launch(x, packed, n, k, tp=dict(comm=comm, mode=2, index=0))[0] == -1                 # 2 * 2048 > 1024
    finally:
        comm.close()
