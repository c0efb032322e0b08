"""The exact-integer W4A16 GEMM's int8-cache epilogue (zl_w4a16_gemm_fused with kv_int8): split + RoPE + quantise the K / V
rows into the int8 cache through the last-arriver protocol.  Its codes and scales must be the same GEMM's fp16 epilogue
rows quantised by zl_int8_quant_rows_u8, bit for bit."""
import numpy as np
import pytest
import torch

from oracle import gptq

pytestmark = pytest.mark.gpu

HQ, HKV, K, LEN = 4, 2, 512, 12


def _pack(cuda, k, n, row_map, seed=14):
    from zhilight_b200 import ops
    qw, qz, sc, gi = gptq.make_gptq_checkpoint(k, n, 128, False, seed=seed)
    o_qw, o_qz, o_sc, _ = gptq.to_k_major(qw, qz, sc, gi, 128)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    return ops.w4_pack(dev(o_qw.view(np.int32)), dev(o_qz), dev(o_sc), 128, False, row_map, variant=1)


def _quant_rows_u8(rows):
    from zhilight_b200 import _lib
    r = rows.reshape(-1, rows.shape[-1]).contiguous()
    q = torch.empty(r.shape, dtype=torch.uint8, device=r.device)
    s = torch.empty(r.shape[0], dtype=torch.float32, device=r.device)
    _lib.call("zl_int8_quant_rows_u8", r.data_ptr(), q.data_ptr(), s.data_ptr(), r.shape[0], r.shape[1], 0, None)
    torch.cuda.synchronize()
    return q.reshape(rows.shape), s.reshape(rows.shape[:-1])


def _case(cuda, m, d, norm_bias):
    from zhilight_b200 import ops
    n = (HQ + 2 * HKV) * d
    rm = ops.qkv_rope_row_map(HQ + 2 * HKV, d, cuda)
    packed = _pack(cuda, K, n, rm)
    g = torch.Generator().manual_seed(m * 1000 + d)
    x = torch.randn(m, K, generator=g).half().to(cuda)
    kw = {}
    if norm_bias:
        kw["ln_weight"] = (1.0 + 0.1 * torch.randn(K, generator=g)).half().to(cuda)
        kw["bias"] = ops.gather_rows_16((0.05 * torch.randn(n, generator=g)).half().to(cuda), rm)
    pos = torch.tensor([(5 * i) % 11 for i in range(m)], dtype=torch.int32, device=cuda)
    cos, sin = ops.rope_cos_sin(pos, d, 10000.0)
    tb = torch.tensor([i % 3 for i in range(m)], dtype=torch.int32, device=cuda)         # tasks interleaved
    pl = torch.tensor([-1 if i % 4 == 3 else i // 3 for i in range(m)], dtype=torch.int32, device=cuda)
    rope = dict(cos=cos, sin=sin, token_batch=tb, placement=pl, num_heads=HQ, num_kv_heads=HKV, dim_head=d)
    return packed, n, x, kw, rope, pl


@pytest.mark.parametrize("norm_bias", [False, True], ids=["plain", "norm+bias"])
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("m", [1, 2, 3, 4, 5, 8, 16])
def test_int8_epilogue_is_the_fp16_epilogue_quantised(lib, cuda, m, d, norm_bias):
    from zhilight_b200 import ops
    packed, n, x, kw, rope, pl = _case(cuda, m, d, norm_bias)
    kb16 = [torch.zeros(LEN, HKV, d, dtype=torch.float16, device=cuda) for _ in range(3)]
    vb16 = [torch.zeros(LEN, HKV, d, dtype=torch.float16, device=cuda) for _ in range(3)]
    q16 = ops.w4a16_gemm_fused(x, packed, n, K, epilogue=ops.EPI_QKV_ROPE, variant=1,
                               rope=dict(rope, k_bufs=kb16, v_bufs=vb16), **kw)
    # sentinels: rows the launch must not touch keep them
    kb8 = [torch.full((LEN, HKV, d), 77, dtype=torch.uint8, device=cuda) for _ in range(3)]
    vb8 = [torch.full((LEN, HKV, d), 77, dtype=torch.uint8, device=cuda) for _ in range(3)]
    sk = [torch.full((LEN, HKV), -1.0, device=cuda) for _ in range(3)]
    sv = [torch.full((LEN, HKV), -1.0, device=cuda) for _ in range(3)]
    stage = torch.empty(m, 2, HKV, d, dtype=torch.float16, device=cuda)
    cnt = torch.zeros(m, 2, HKV, dtype=torch.int32, device=cuda)
    kv8 = dict(sk_bufs=sk, sv_bufs=sv, stage=stage, counters=cnt)
    results = []
    for _ in range(2):     # back to back, counters not re-zeroed by the caller
        q8 = ops.w4a16_gemm_fused(x, packed, n, K, epilogue=ops.EPI_QKV_ROPE, variant=1,
                                  rope=dict(rope, k_bufs=kb8, v_bufs=vb8), kv8=kv8, **kw)
        torch.cuda.synchronize()
        assert int(cnt.abs().sum()) == 0, "counters must be back at zero"
        torch.testing.assert_close(q8, q16, rtol=0, atol=0)
        results.append([t.clone() for t in kb8 + vb8 + sk + sv])
    for a, b in zip(*results):
        torch.testing.assert_close(a, b, rtol=0, atol=0)
    written = {(int(t), int(p)) for t, p in zip(rope["token_batch"].tolist(), pl.tolist()) if p >= 0}
    for b in range(3):
        for bufs16, bufs8, scales in ((kb16, kb8, sk), (vb16, vb8, sv)):
            codes, sc = _quant_rows_u8(bufs16[b])
            for row in range(LEN):
                if (b, row) in written:
                    torch.testing.assert_close(bufs8[b][row], codes[row], rtol=0, atol=0)
                    torch.testing.assert_close(scales[b][row], sc[row], rtol=0, atol=0)
                else:
                    assert bool((bufs8[b][row] == 77).all()) and bool((scales[b][row] == -1.0).all()), (b, row)


def test_int8_epilogue_only_on_the_integer_route(lib, cuda):
    from zhilight_b200 import _lib, ops
    d = 64
    for m, extra in ((17, {}), (4, {"k_perm": torch.arange(K, dtype=torch.int32, device=cuda)})):
        packed, n, x, kw, rope, pl = _case(cuda, m, d, False)
        kb8 = [torch.zeros(LEN, HKV, d, dtype=torch.uint8, device=cuda) for _ in range(3)]
        sk = [torch.zeros(LEN, HKV, device=cuda) for _ in range(3)]
        kv8 = dict(sk_bufs=sk, sv_bufs=sk, stage=torch.empty(m, 2, HKV, d, dtype=torch.float16, device=cuda),
                   counters=torch.zeros(m, 2, HKV, dtype=torch.int32, device=cuda))
        with pytest.raises(_lib.ZLError) as e:
            ops.w4a16_gemm_fused(x, packed, n, K, epilogue=ops.EPI_QKV_ROPE, variant=1,
                                 rope=dict(rope, k_bufs=kb8, v_bufs=kb8), kv8=kv8, **extra)
        assert e.value.code == -2
