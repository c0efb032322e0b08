"""GPU: act-order (desc_act) GPTQ.  The exact-integer W4A16 kernel gathers x[:, k_perm] while it stages the activations
and must equal, bit for bit, the same launch on host-permuted activations; the other routes permute with
zl_gather_cols_16 first; layers.Linear and the decode driver serve act-order checkpoints end to end."""
import numpy as np
import pytest
import torch

from oracle import gptq, model as omodel
from tests.helpers import rel_l2
from tests.test_act_order_cpu import TINY, ActOrderOracle, act_order_g_idx, act_order_state_dict

pytestmark = pytest.mark.gpu

LAYERS8B = dict(num_layers=3, dim_model=4096, num_heads=32, num_kv_heads=8, dim_head=128, dim_ff=14336, vocab_size=2048,
                eps=1e-5, rope_theta=500000.0, rope_llama3=dict(factor=8.0, low=1.0, high=4.0, orig=8192.0))
_W = {}


def _weights(cuda, k, n, row_map=None, seed=0):
    """(packed ZLW4I of the sequentialised weights, k_perm, HF tensors, g_idx) of a random act-order Linear."""
    from zhilight_b200 import ops
    key = (k, n, None if row_map is None else row_map.numel(), seed)
    if key not in _W:
        qw, qz, sc, _ = gptq.make_gptq_checkpoint(k, n, 128, False, seed=seed)
        gi = act_order_g_idx(k, 128, np.random.default_rng(seed))
        t = [torch.from_numpy(a).to(cuda) for a in (qw, qz, sc)]
        kq, kz, ks, perm = ops.gptq_to_k_major_act_order(t[0], t[1], t[2], torch.from_numpy(gi))
        _W[key] = (ops.w4_pack(kq, kz, ks, 128, False, row_map, variant=1), perm, (qw, qz, sc), gi)
    return _W[key]


def _x(m, k, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(m, k, generator=g) * torch.logspace(-1, 0.5, k)[torch.randperm(k, generator=g)]).half()


# batch sizes the router sends to the integer kernel on each shape (larger ones go to the wgmma kernel); 1024 x 1024 takes
# the 16-token variants
@pytest.mark.parametrize("shape,m", [("4096x4096", 1), ("4096x4096", 2), ("4096x4096", 4), ("4096x4096", 7),
                                     ("swiglu28672x4096", 1), ("swiglu28672x4096", 4), ("swiglu28672x4096", 7),
                                     ("residual4096x14336", 1), ("residual4096x14336", 2),
                                     ("1024x1024", 8), ("1024x1024", 16)])
@pytest.mark.parametrize("norm", [False, True])
def test_integer_kernel_gather_is_bit_exact(lib, cuda, m, norm, shape):
    from zhilight_b200 import ops
    epi, n, k = {"4096x4096": (ops.EPI_NONE, 4096, 4096), "swiglu28672x4096": (ops.EPI_SWIGLU, 28672, 4096),
                 "residual4096x14336": (ops.EPI_RESIDUAL, 4096, 14336), "1024x1024": (ops.EPI_NONE, 1024, 1024)}[shape]
    assert lib.zl_w4_int_layout_route(m, n, k) == 3
    rm = ops.swiglu_row_map(n // 2, cuda) if epi == ops.EPI_SWIGLU else None
    packed, perm, (qw, qz, sc), gi = _weights(cuda, k, n, rm)
    x = _x(m, k, m).to(cuda)
    lw = (1 + 0.1 * torch.randn(k, generator=torch.Generator().manual_seed(3))).half().to(cuda) if norm else None
    res = torch.randn(m, n, generator=torch.Generator().manual_seed(4)).half().to(cuda) if epi == ops.EPI_RESIDUAL else None
    kw = dict(epilogue=epi, residual=res, eps=1e-5, variant=1)
    y = ops.w4a16_gemm_fused(x, packed, n, k, ln_weight=lw, k_perm=perm, **kw)
    pl = perm.long()
    y_host = ops.w4a16_gemm_fused(x[:, pl].contiguous(), packed, n, k, ln_weight=None if lw is None else lw[pl].contiguous(),
                                  **kw)
    torch.cuda.synchronize()
    assert torch.equal(y, y_host)
    if shape == "4096x4096" and not norm:   # and the act-order checkpoint itself
        ref = gptq.gemm_f32(x.cpu().numpy(), gptq.hf_dequant_f32(qw, qz, sc, gi, 128))
        assert rel_l2(y.float().cpu().numpy(), ref) <= 1e-3


@pytest.mark.parametrize("m", [1, 4, 7])
@pytest.mark.parametrize("norm", [False, True])
def test_integer_kernel_gather_qkv_rope_bit_exact(lib, cuda, m, norm):
    """6144 x 4096 qkv of Llama-3.1-8B with the RoPE / KV-append epilogue: q and the KV cache rows."""
    from zhilight_b200 import ops
    hq, hkv, d, k = 32, 8, 128, 4096
    n = (hq + 2 * hkv) * d
    assert lib.zl_w4_int_layout_route(m, n, k) == 3
    packed, perm, _, _ = _weights(cuda, k, n, ops.qkv_rope_row_map(hq + 2 * hkv, d, cuda), seed=1)
    x = _x(m, k, 10 + m).to(cuda)
    lw = (1 + 0.1 * torch.randn(k, generator=torch.Generator().manual_seed(3))).half().to(cuda) if norm else None
    pos = torch.tensor([(5 * i) % 11 for i in range(m)], dtype=torch.int32, device=cuda)
    cos, sin = ops.rope_cos_sin(pos, d, 500000.0)
    tb = torch.tensor([i % 4 for i in range(m)], dtype=torch.int32, device=cuda)
    pl = torch.tensor([i // 4 for i in range(m)], dtype=torch.int32, device=cuda)
    outs = []
    for gathered in (True, False):
        kb = [torch.zeros(8, hkv, d, dtype=torch.float16, device=cuda) for _ in range(4)]
        vb = [torch.zeros(8, hkv, d, dtype=torch.float16, device=cuda) for _ in range(4)]
        rope = dict(cos=cos, sin=sin, token_batch=tb, placement=pl, k_bufs=kb, v_bufs=vb, num_heads=hq, num_kv_heads=hkv,
                    dim_head=d)
        if gathered:
            q = ops.w4a16_gemm_fused(x, packed, n, k, epilogue=ops.EPI_QKV_ROPE, ln_weight=lw, variant=1, rope=rope,
                                     k_perm=perm)
        else:
            p = perm.long()
            q = ops.w4a16_gemm_fused(x[:, p].contiguous(), packed, n, k, epilogue=ops.EPI_QKV_ROPE,
                                     ln_weight=None if lw is None else lw[p].contiguous(), variant=1, rope=rope)
        outs.append([q] + kb + vb)
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_gather_cols_is_exact(lib, cuda):
    from zhilight_b200 import ops
    for m, k, ldx in ((1, 4096, 4096), (37, 14336, 14336), (5, 1024, 1536)):
        perm = torch.from_numpy(np.random.default_rng(k).permutation(k).astype(np.int32)).to(cuda)
        xs = torch.randn(m, ldx, generator=torch.Generator().manual_seed(m)).half().to(cuda)
        x = xs[:, :k]
        y = ops.gather_cols(x, perm)
        assert torch.equal(y, x[:, perm.long()])


@pytest.mark.parametrize("m", [17, 64, 300])
def test_gather_then_wgmma_is_bit_exact(lib, cuda, m):
    from zhilight_b200 import _lib, ops
    n, k = 4096, 4096
    assert lib.zl_w4_int_layout_route(m, n, k) == 4
    packed, perm, _, _ = _weights(cuda, k, n)
    x = _x(m, k, m).to(cuda)
    y = ops.w4a16_gemm_fused(ops.gather_cols(x, perm), packed, n, k, variant=1)
    y_host = ops.w4a16_gemm_fused(x[:, perm.long()].contiguous(), packed, n, k, variant=1)
    assert torch.equal(y, y_host)
    # k_perm is only gathered by the integer kernel
    with pytest.raises(_lib.ZLError) as e:
        ops.w4a16_gemm_fused(x, packed, n, k, variant=1, k_perm=perm)
    assert e.value.code == -2


def test_k_perm_refused_on_fp16_route_and_with_tp_mode(lib, cuda):
    import ctypes
    from zhilight_b200 import _lib, ops
    n, k = 256, 1024
    packed, perm, _, _ = _weights(cuda, k, n)
    x = _x(1, k, 0).to(cuda)
    with pytest.raises(_lib.ZLError) as e:   # variant 0: the fp16 mma.sync route
        ops.w4a16_gemm_fused(x, packed, n, k, variant=0, k_perm=perm)
    assert e.value.code == -2
    a = _lib.W4FusedArgs()
    y = torch.empty(1, n, dtype=torch.float16, device=cuda)
    a.x, a.ldx, a.packed, a.y, a.M, a.N, a.K, a.group_size, a.variant = (x.data_ptr(), k, packed.data_ptr(), y.data_ptr(),
                                                                          1, n, k, 128, 1)
    a.tp_mode, a.tp_comm, a.k_perm = 2, 16, perm.data_ptr()
    assert lib.zl_w4a16_gemm_fused(ctypes.byref(a), None) == -2


@pytest.mark.parametrize("m", [1, 5, 17])
def test_linear_gptq_act_order_matches_oracle(lib, cuda, m):
    from zhilight_b200 import _lib
    from zhilight_b200.layers import Linear
    k, n = 1024, 512
    qw, qz, sc, _ = gptq.make_gptq_checkpoint(k, n, 128, False, seed=4)
    gi = act_order_g_idx(k, 128, np.random.default_rng(4))
    sd = {"qweight": torch.from_numpy(qw), "qzeros": torch.from_numpy(qz), "scales": torch.from_numpy(sc),
          "g_idx": torch.from_numpy(gi)}
    lin = Linear(k, n, quant=5)
    lin.load_state_dict(sd)
    x = _x(m, k, m)
    y = lin(x.to(cuda)).float().cpu().numpy()
    ref = gptq.gemm_f32(x.numpy(), gptq.hf_dequant_f32(qw, qz, sc, gi, 128))
    assert rel_l2(y, ref) <= 1e-3
    with pytest.raises(_lib.ZLError):
        Linear(k, n, quant=8).load_state_dict(sd)


def _decoder(cfg, sd, **kw):
    from zhilight_b200.llama import LlamaDecoder
    sym = kw.pop("sym", False)
    dec = LlamaDecoder(quant_type=5, group_size=128, sym=sym, **dict(dict(max_batch=20, max_seq=64), **kw), **cfg)
    dec.load_state_dict(sd)
    return dec


def _steps(dec, orc, b, steps=4, seed=0, vocab=512):
    rng = np.random.default_rng(seed)
    tok = rng.integers(0, vocab, size=b).astype(np.int32)
    pos = np.zeros(b, np.int32)
    for _ in range(steps):
        nxt, logits = dec.decode(tok, pos, want_logits=True)
        ref = orc.decode(tok, pos)
        assert rel_l2(logits, ref) <= 3e-3
        tok = rng.integers(0, vocab, size=b).astype(np.int32)
        pos += 1
    return nxt


@pytest.mark.parametrize("b", [1, 20])
@pytest.mark.parametrize("fuse", [0, 1, 2])
def test_tiny_act_order_decode_matches_oracle(lib, cuda, b, fuse):
    sd = act_order_state_dict(TINY, omodel.make_state_dict(TINY, 5, 128, False, seed=3), seed=3)
    dec = _decoder(TINY, sd, fuse=fuse)
    _steps(dec, ActOrderOracle(TINY, sd, 5, 128, False, "f16", fuse_norm=fuse >= 1), b, vocab=TINY["vocab_size"])
    dec.close()


@pytest.mark.parametrize("b", [1, 20])
@pytest.mark.parametrize("fuse", [0, 2])
def test_llama8b_layers_act_order_decode_matches_oracle(lib, cuda, b, fuse):
    cfg = LAYERS8B
    key = ("sd8b",)
    if key not in _W:
        base = omodel.make_state_dict(cfg, 5, 128, True, seed=2, scale_range=(0.0003, 0.0008))
        sd = act_order_state_dict(cfg, base, seed=2)
        _W[key] = (sd, ActOrderOracle(cfg, sd, 5, 128, True, "f16", fuse_norm=True))
    sd, orc = _W[key]          # the dequantised weights are kept across runs; the KV state is not
    orc.fuse_norm = fuse >= 1
    orc.kv = {}
    dec = _decoder(cfg, sd, sym=True, fuse=fuse, max_seq=16)
    _steps(dec, orc, b, vocab=cfg["vocab_size"], seed=b)
    dec.close()


@pytest.mark.parametrize("b", [4, 20])   # integer kernel gathering in its staging loop / zl_gather_cols_16 + wgmma
def test_host_device_and_graph_stepping_agree(lib, cuda, b):
    sd = act_order_state_dict(TINY, omodel.make_state_dict(TINY, 5, 128, False, seed=5), seed=5)
    finals = []
    for graph, mode in ((True, "host"), (False, "host"), (True, "device")):
        dec = _decoder(TINY, sd, use_graph=graph)
        tok = np.arange(3, 3 + b, dtype=np.int32)
        pos = np.zeros(b, np.int32)
        seq = []
        if mode == "device":
            dec.set_state(tok, pos)
        for _ in range(6):
            if mode == "host":
                tok = dec.decode(tok, pos)
                pos = pos + 1
            else:
                dec.step_device(b)
                tok, pos = dec.get_state(b)
            seq.append(tok.copy())
        finals.append(np.array(seq))
        dec.close()
    np.testing.assert_array_equal(finals[0], finals[1])
    np.testing.assert_array_equal(finals[0], finals[2])


@pytest.mark.parametrize("dual", [False, True])
@pytest.mark.parametrize("chunk", [16, 64])
def test_chunked_prefill_matches_oracle(lib, cuda, monkeypatch, chunk, dual):
    """dual: the two-half, two-stream prefill pipeline (ZL_PREFILL_DUAL=1), which runs the GEMMs on half-chunks."""
    monkeypatch.setenv("ZL_PREFILL_DUAL", "1" if dual else "0")
    sd = act_order_state_dict(TINY, omodel.make_state_dict(TINY, 5, 128, False, seed=6), seed=6)
    dec = _decoder(TINY, sd, max_batch=2, max_seq=128, prefill_chunk=chunk)
    orc = ActOrderOracle(TINY, sd, 5, 128, False, "f16", fuse_norm=True)
    prompt = np.random.default_rng(6).integers(0, TINY["vocab_size"], size=40).astype(np.int32)
    nxt, logits = dec.prefill(1, prompt, want_logits=True)
    for i, t in enumerate(prompt):
        ref = orc.decode(np.array([t]), np.array([i]), tasks=[1])
    # the halves of one chunk can take different kernels (wgmma with a stand-alone RMSNorm vs the integer kernel with the
    # fused one), so the dual pipeline gets the tolerance tests/test_llama_gpu.py gives it against the oracle
    assert rel_l2(logits, ref) <= (5e-3 if dual else 3e-3)
    tok, pos = np.array([nxt], np.int32), np.array([40], np.int32)
    for _ in range(3):
        out, logits = dec.decode(np.array([0, tok[0]], np.int32), np.array([0, pos[0]], np.int32), want_logits=True)
        ref = orc.decode(tok, pos, tasks=[1])
        assert rel_l2(logits[1:], ref) <= 3e-3
        tok, pos = out[1:], pos + 1
    dec.close()


@pytest.mark.parametrize("b", [1, 16, 20])
def test_kernels_per_step(lib, cuda, b):
    base = omodel.make_state_dict(TINY, 5, 128, False, seed=7)
    counts = []
    for sd in (base, act_order_state_dict(TINY, base, seed=7)):
        dec = _decoder(TINY, sd)
        dec.decode(np.arange(b, dtype=np.int32), np.zeros(b, np.int32))
        counts.append(dec.stats(b)[1])
        dec.close()
    if b <= 16:
        assert counts[1] == counts[0]
    else:
        assert counts[0] < counts[1] <= counts[0] + 3 * TINY["num_layers"]


def test_sampled_task_draws_ops_sample(lib, cuda):
    from zhilight_b200 import ops
    sd = act_order_state_dict(TINY, omodel.make_state_dict(TINY, 5, 128, False, seed=8), seed=8)
    dec = _decoder(TINY, sd, max_batch=2)
    sp = dict(temperature=0.9, top_p=0.95, top_k=40, seed=11)
    dec.set_sampling(1, **sp)
    tok, pos = np.array([5, 9], np.int32), np.zeros(2, np.int32)
    for _ in range(4):
        nxt, logits = dec.decode(tok, pos, want_logits=True)
        want = ops.sample(torch.from_numpy(logits).to(cuda), [dict(temperature=0.0), sp],
                          counter=torch.from_numpy(pos).to(cuda)).cpu().numpy()
        np.testing.assert_array_equal(nxt, want)
        tok, pos = nxt, pos + 1
    dec.close()


def test_load_refusals(lib, cuda):
    from zhilight_b200 import _lib, dist
    from zhilight_b200.llama import LlamaDecoder
    base = omodel.make_state_dict(TINY, 5, 128, False, seed=9)
    sd = act_order_state_dict(TINY, base, seed=9)
    # mismatched q / k / v (and gate / up) permutations: the fused Linear has one input permutation
    for a, b in (("attn.project_q", "attn.project_k"), ("ff.w_in", "ff.w_gated")):
        bad = dict(sd)
        bad["layers.1.%s.g_idx" % b] = act_order_g_idx(TINY["dim_model"], 128, np.random.default_rng(1))
        dec = LlamaDecoder(quant_type=5, max_batch=1, max_seq=16, **TINY)
        with pytest.raises(_lib.ZLError) as e:
            dec.load_state_dict(bad)
        assert e.value.code == -2 and "layers.1.%s" % b in str(e.value)
        dec.close()
    # malformed: one group with 129 members and one with 127
    bad = dict(sd)
    gi = sd["layers.0.attn.attn_out.g_idx"].copy()
    gi[np.flatnonzero(gi == 1)[0]] = 0
    bad["layers.0.attn.attn_out.g_idx"] = gi
    dec = LlamaDecoder(quant_type=5, max_batch=1, max_seq=16, **TINY)
    with pytest.raises(_lib.ZLError) as e:
        dec.load_state_dict(bad)
    assert e.value.code == -1
    dec.close()
    # tensor parallelism: refused at load, before any exchange
    dec = LlamaDecoder(quant_type=5, max_batch=1, max_seq=16, tp_rank=0, tp_size=2, **TINY)
    with pytest.raises(_lib.ZLError) as e:
        dec.load_state_dict(dist.shard_state_dict(sd, 0, 2))
    assert e.value.code == -2
    dec.close()
