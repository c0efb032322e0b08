"""The variable-length (k_varlen_attn, 64 KiB) and MLA (k_mla_decode_attn, ~217 KiB) attention kernels opt in to more
dynamic shared memory than the default 48 KiB.  That attribute belongs to the device that was current when it was set,
so each device must be set up on its first call there, not only the first device the process used.  Checked against
the float64 references of the boundary tests."""
import pytest
import torch

from tests.attn_check import assert_close
from tests.test_attn_boundaries_gpu import (BF16, DEVICE, F16, MLA_SCALE, MLA_TOL, VA_SETS, VA_TOL, _Mla, _plan_mla,
                                            _Varlen)

pytestmark = pytest.mark.gpu


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two CUDA devices")
def test_varlen_and_mla_on_two_devices(lib, cuda):
    from zhilight_b200 import ops
    va = _Varlen(VA_SETS["span"], 2, 8, 128, F16, seed=1)
    va_ref, _ = va.reference()
    lens = [3000, 65, 1]
    mla = _Mla(lens, 2, 16, BF16, "holes", [_plan_mla(len(lens), 2, 16, max(lens))], seed=2)
    mla_ref, _ = mla.reference()
    mla_mask = torch.cat([m.reshape(-1) for m in mla.masks]).to(torch.int8)
    for dev in ("cuda:0", "cuda:1"):
        with torch.cuda.device(dev):
            out = ops.varlen_attention(va.q.to(dev), va.table(), [k.to(dev) for k in va.k], [v.to(dev) for v in va.v],
                                       va.scale, va.hkv)
            assert_close(out.to(DEVICE), va_ref, VA_TOL[F16], ("varlen", dev))
            out = ops.mla_decode_attention(mla.q.to(dev), torch.tensor(lens, dtype=torch.int32, device=dev),
                                           [kv.to(dev) for kv in mla.kv], mla_mask.to(dev), MLA_SCALE, max(lens))
            assert_close(out.to(DEVICE), mla_ref, MLA_TOL[BF16], ("mla", dev))
