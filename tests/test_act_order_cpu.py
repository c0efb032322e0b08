"""Act-order (desc_act) GPTQ checkpoints without a GPU: the C-ABI struct mirror, argument checks of the column gather,
the act-order permutation of the Python front end, and the act-order test checkpoints and oracle that the GPU tests
(tests/test_act_order_gpu.py) compare against."""
import ctypes

import numpy as np
import pytest

from oracle import gptq, model as omodel
from zhilight_b200 import _lib

TINY = dict(num_layers=2, dim_model=256, num_heads=4, num_kv_heads=2, dim_head=64, dim_ff=512, vocab_size=512,
            eps=1e-5, rope_theta=10000.0, rope_llama3=None)

# Linears that share an input share its permutation: GPTQ's Hessian, and so desc_act's column order, is that of the input
INPUT_GROUPS = (("attn.project_q", "attn.project_k", "attn.project_v"), ("attn.attn_out",), ("ff.w_in", "ff.w_gated"),
                ("ff.w_out",))


def act_order_g_idx(k, group_size, rng):
    """g_idx as AutoGPTQ writes it for desc_act: columns quantised in the order perm, g_idx[perm[i]] = i // group_size."""
    perm = rng.permutation(k)
    g_idx = np.empty(k, np.int32)
    g_idx[perm] = np.arange(k) // group_size
    return g_idx


def act_order_state_dict(cfg, sd, seed=0, group_size=128):
    """A copy of a GPTQ state dict from oracle.model.make_state_dict with an act-order g_idx on every Linear: one random
    permutation per input (q/k/v, o, gate/up, down of each layer)."""
    rng = np.random.default_rng(1000 + seed)
    out = dict(sd)
    for l in range(cfg["num_layers"]):
        for group in INPUT_GROUPS:
            p = "layers.%d." % l
            k = sd[p + group[0] + ".qweight"].shape[0] * 8
            gi = act_order_g_idx(k, group_size, rng)
            for name in group:
                out[p + name + ".g_idx"] = gi
    return out


class ActOrderOracle(omodel.OracleLlama):
    """OracleLlama that honours each GPTQ Linear's g_idx: the weight is dequantised through the reference's act-order
    load (to_k_major with g_idx: rows gathered by argsort(g_idx)) and put back in checkpoint column order."""

    def _weight(self, prefix):
        gi = self.sd.get(prefix + ".g_idx")
        if self.quant_type != 5 or gi is None or prefix in self.w:
            return super()._weight(prefix)
        sd = self.sd
        qw, qz, sc, perm = gptq.to_k_major(sd[prefix + ".qweight"], sd[prefix + ".qzeros"], sd[prefix + ".scales"], gi,
                                           self.group_size)
        w_seq = gptq.dequant_k_major_f32(qw, qz, sc, self.sym)
        w = w_seq
        if perm is not None:
            w = np.empty_like(w_seq)
            w[:, perm] = w_seq
        self.w[prefix] = w
        return w


def test_w4_fused_args_mirror_matches_c_struct(lib):
    size, off = ctypes.c_size_t(), ctypes.c_size_t()
    assert lib.zl_w4_fused_args_layout(ctypes.byref(size), ctypes.byref(off)) == 0
    assert ctypes.sizeof(_lib.W4FusedArgs) == size.value
    assert _lib.W4FusedArgs.k_perm.offset == off.value
    assert lib.zl_w4_fused_args_layout(None, ctypes.byref(off)) == -1


def test_gather_cols_rejects_bad_arguments_without_gpu(lib):
    p, q = ctypes.c_void_p(256), ctypes.c_void_p(4096)
    ok = (p, 4096, q, p, 1, 4096, 0, None)
    for i, bad in ((0, None), (2, None), (3, None), (0, ctypes.c_void_p(258)), (2, ctypes.c_void_p(4100)),
                   (3, ctypes.c_void_p(264)), (1, 4095), (1, 4092), (5, 4092), (4, 0), (4, 70000)):
        args = list(ok)
        args[i] = bad
        assert lib.zl_gather_cols_16(*args) == -1, (i, bad)


def test_header_states_the_k_perm_contract():
    src = open(_lib.HEADER).read()
    for must in ("k_perm", "permute_input", "gptq/utils.cu:322-398", "make_sequential", "zl_gather_cols_16"):
        assert must in src, must


def test_act_order_perm_is_the_reference_bucket_sort():
    import torch
    from zhilight_b200 import ops
    rng = np.random.default_rng(0)
    for k in (256, 1024, 4096):
        gi = act_order_g_idx(k, 128, rng)
        perm = ops.act_order_perm(torch.from_numpy(gi))
        np.testing.assert_array_equal(perm.numpy(), gptq.argsort_g_idx(gi, 128))
    assert ops.act_order_perm(torch.arange(1024, dtype=torch.int32) // 128) is None
    bad = act_order_g_idx(1024, 128, rng)
    bad[bad == 3] = 2
    with pytest.raises(_lib.ZLError):
        ops.act_order_perm(torch.from_numpy(bad))
    with pytest.raises(_lib.ZLError):
        ops.act_order_perm(torch.full((1024,), 8, dtype=torch.int32))


def test_act_order_state_dict_groups():
    sd = act_order_state_dict(TINY, omodel.make_state_dict(TINY, 5, 128, False, seed=0))
    for l in range(TINY["num_layers"]):
        p = "layers.%d." % l
        gis = {}
        for group in INPUT_GROUPS:
            k = sd[p + group[0] + ".qweight"].shape[0] * 8
            gi = sd[p + group[0] + ".g_idx"]
            assert gi.shape == (k,) and gi.dtype == np.int32
            np.testing.assert_array_equal(gi[gptq.argsort_g_idx(gi, 128)], np.arange(k) // 128)
            assert not np.array_equal(gi, np.arange(k) // 128)
            for name in group[1:]:
                np.testing.assert_array_equal(sd[p + name + ".g_idx"], gi)
            gis[group[0]] = gi
        assert not np.array_equal(gis["attn.project_q"], gis["ff.w_in"])


def test_act_order_oracle_equals_checkpoint_dequant():
    cfg = TINY
    sd = act_order_state_dict(cfg, omodel.make_state_dict(cfg, 5, 128, False, seed=1))
    orc = ActOrderOracle(cfg, sd, 5, 128, False, "f16")
    rng = np.random.default_rng(2)
    x = rng.standard_normal((3, cfg["dim_model"])).astype(np.float16)
    for name in ("attn.project_q", "ff.w_in"):
        p = "layers.0." + name
        w = gptq.hf_dequant_f32(sd[p + ".qweight"], sd[p + ".qzeros"], sd[p + ".scales"], sd[p + ".g_idx"], 128)
        np.testing.assert_array_equal(orc._weight(p), w)
        y = (np.asarray(x, np.float32) @ w.T).astype(np.float16)
        np.testing.assert_array_equal(orc._linear(x, p), y)
    # the act-order g_idx changes the layer: the plain oracle reads the same tensors as a sequential checkpoint
    plain = omodel.OracleLlama(cfg, sd, 5, 128, False, "f16")
    assert not np.array_equal(plain._weight("layers.0.attn.project_q"), orc._weight("layers.0.attn.project_q"))


def test_gather_cols_checks_its_input_without_gpu():
    import torch
    from zhilight_b200 import ops
    perm = torch.arange(256, dtype=torch.int32)
    with pytest.raises(_lib.ZLError):   # 32-bit x
        ops.gather_cols(torch.zeros(2, 256), perm)
    with pytest.raises(_lib.ZLError):   # transposed view: column stride != 1
        ops.gather_cols(torch.zeros(256, 2, dtype=torch.float16).t(), perm)
    with pytest.raises(_lib.ZLError):   # int64 permutation
        ops.gather_cols(torch.zeros(2, 256, dtype=torch.float16), perm.long())
