"""Loading and releasing a decoder: a checkpoint with an ill-shaped bias is refused before any copy reads past it, and a
model's device memory is returned when it is closed."""
import numpy as np
import pytest

from oracle import model as omodel

pytestmark = pytest.mark.gpu

TINY = dict(num_layers=2, dim_model=256, num_heads=4, num_kv_heads=2, dim_head=64, dim_ff=512, vocab_size=512,
            eps=1e-5, rope_theta=10000.0, rope_llama3=None)


@pytest.mark.parametrize("quant", [0, 5, 7], ids=["dense", "gptq", "fp8"])
def test_short_bias_is_refused(lib, cuda, quant):
    from zhilight_b200 import _lib
    from zhilight_b200.llama import LlamaDecoder
    sd = omodel.make_state_dict(TINY, quant, 128, False, seed=3)
    name = "layers.0.attn.project_q.bias"
    sd[name] = np.zeros(TINY["num_heads"] * TINY["dim_head"] - 1, np.float16)
    dec = LlamaDecoder(quant_type=quant, max_batch=1, max_seq=32, **TINY)
    with pytest.raises(_lib.ZLError) as e:
        dec.load_state_dict(sd)
    assert e.value.code == -1
    assert name in str(e.value)
    dec.close()


def test_close_returns_device_memory(lib, cuda):
    """create -> init_synthetic -> decode -> close, 20 times: the KV buffers (50 MB here), weights, activations and the
    argmax candidates all go back."""
    import torch
    from zhilight_b200.llama import LlamaDecoder

    def cycle():
        dec = LlamaDecoder(quant_type=5, max_batch=2, max_seq=24576, **TINY)
        dec.init_synthetic(0)
        dec.decode(np.array([1, 2], np.int32), np.array([0, 0], np.int32))
        dec.close()

    cycle()   # the first launches load kernel modules: device memory that is not the model's
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    for _ in range(20):
        cycle()
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    assert free0 - free1 <= 4 << 20
