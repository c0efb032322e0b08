"""int8 KV cache of the decode driver without a GPU: the config mirror, the configurations zl_llama_create refuses before
it touches the device, and the int8 oracle's cache rows against the reference's quantisation."""
import ctypes
import hashlib

import numpy as np
import pytest

from oracle import golden_cases as gc, model as omodel
from tests.kv8_oracle import Kv8OracleLlama, dequant_rows, quant_rows
from tests.helpers import rel_l2

TINY = dict(num_layers=2, dim_model=256, num_heads=4, num_kv_heads=2, dim_head=64, dim_ff=512, vocab_size=512,
            eps=1e-5, rope_theta=10000.0, rope_llama3=None)


def test_llama_config_mirror_matches_c_struct(lib):
    from zhilight_b200 import _lib
    size, off = ctypes.c_size_t(), ctypes.c_size_t()
    assert lib.zl_llama_config_layout(ctypes.byref(size), ctypes.byref(off)) == 0
    assert ctypes.sizeof(_lib.LlamaConfig) == size.value
    assert _lib.LlamaConfig.kv_int8.offset == off.value
    assert lib.zl_llama_config_layout(None, ctypes.byref(off)) == -1
    # appending kv_int8 left the GEMM argument struct as it was
    assert lib.zl_w4_fused_args_layout(ctypes.byref(size), ctypes.byref(off)) == 0
    assert ctypes.sizeof(_lib.W4FusedArgs) == size.value and _lib.W4FusedArgs.k_perm.offset == off.value


def _create(lib, **over):
    from zhilight_b200 import _lib
    c = dict(TINY, quant_type=5, group_size=128, sym=0, dtype=0, max_batch=2, max_seq=64, tp_rank=0, tp_size=1,
             use_pdl=1, use_graph=1, tp_int8=0, fuse=2, prefill_chunk=0, qkv_bias=0, kv_int8=1)
    c.update(over)
    l3 = c.pop("rope_llama3") or {}
    cfg = _lib.LlamaConfig(c["num_layers"], c["dim_model"], c["num_heads"], c["num_kv_heads"], c["dim_head"], c["dim_ff"],
                           c["vocab_size"], c["eps"], c["rope_theta"], float(l3.get("factor", 0.0)), 1.0, 4.0, 8192.0,
                           c["quant_type"], c["group_size"], c["sym"], c["dtype"], c["max_batch"], c["max_seq"],
                           c["tp_rank"], c["tp_size"], c["use_pdl"], c["use_graph"], c["tp_int8"], c["fuse"],
                           c["prefill_chunk"], c["qkv_bias"], c["kv_int8"])
    h = ctypes.c_void_p()
    return lib.zl_llama_create(ctypes.byref(cfg), ctypes.byref(h))


@pytest.mark.parametrize("over", [dict(dtype=1, quant_type=0), dict(dim_head=96, dim_model=384), dict(max_seq=65537),
                                  dict(dim_head=256, dim_model=1024)],
                         ids=["bf16", "dim_head96", "max_seq65537", "dim_head256"])
def test_create_refuses_unsupported_kv_int8_configs_before_touching_the_device(lib, over):
    assert _create(lib, **over) == -2
    assert b"kv_int8" in lib.zl_last_error()


def test_create_rejects_a_bad_kv_int8_flag(lib):
    assert _create(lib, kv_int8=2) == -1


def test_decoder_rejects_unknown_kv_cache_dtype():
    from zhilight_b200.llama import LlamaDecoder
    with pytest.raises(ValueError):
        LlamaDecoder(kv_cache_dtype="fp8", **TINY)


def test_oracle_cache_rows_match_the_reference_quantisation():
    """tests/golden/ref_kv8.npz holds the reference's quant_calc_scale(x, 127, 128) of these rows: sha256 of the uint8
    codes and the fp32 scales."""
    g = np.load("tests/golden/ref_kv8.npz")
    c = gc.case_kv8()
    for i, (k, v) in enumerate(zip(c["ks"], c["vs"])):
        for name, x in (("k", k), ("v", v)):
            codes, scales = quant_rows(x)
            assert codes.dtype == np.uint8 and codes.shape == x.shape and scales.shape == x.shape[:2]
            digest = np.frombuffer(hashlib.sha256(codes.reshape(-1).tobytes()).digest(), np.uint8)
            np.testing.assert_array_equal(g["%sq%d_sha256" % (name, i)], digest)
            np.testing.assert_array_equal(g["s%s%d" % (name, i)], scales)


def test_zero_row_decodes_to_zero():
    codes, scales = quant_rows(np.zeros((3, 64), np.float16))
    assert (scales == 0).all()
    assert (dequant_rows(codes, scales) == 0).all()


def test_kv8_oracle_stores_dequantised_rows_and_stays_near_fp16():
    sd = omodel.make_state_dict(TINY, 5, 128, False, seed=2)
    plain = omodel.OracleLlama(TINY, sd, 5, 128, False, "f16", fuse_norm=True)
    off = Kv8OracleLlama(TINY, sd, 5, 128, False, "f16", fuse_norm=True, kv_int8=False)
    kv8 = Kv8OracleLlama(TINY, sd, 5, 128, False, "f16", fuse_norm=True)
    rng = np.random.default_rng(0)
    spread = []
    for step in range(6):
        tok = rng.integers(0, TINY["vocab_size"], size=2)
        pos = [step, step]
        a = plain.decode(tok, pos)
        np.testing.assert_array_equal(off.decode(tok, pos), a)
        b = kv8.decode(tok, pos)
        spread.append(rel_l2(b, a))
    for task in (0, 1):
        for l in range(TINY["num_layers"]):
            kb, vb = kv8.kv[task][l]
            for pos, (kc, vc, ks, vs) in kv8.codes[(task, l)].items():
                np.testing.assert_array_equal(kb[pos], dequant_rows(kc, ks))
                np.testing.assert_array_equal(vb[pos], dequant_rows(vc, vs))
    # the int8 cache moves the logits of this model by 1-2.5 % (relative L2), ten times the 2e-3 the GPU tests allow between
    # the driver and this oracle: those tests can tell an int8 cache from an fp16 one
    assert 5e-3 < min(spread) and max(spread) < 5e-2, spread
