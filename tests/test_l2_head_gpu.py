"""The successor-GEMM L2 prefetch is a hint: decoding with it (ZL_W4_L2_HEAD / ZL_W4_L2_WHOLE_MB) and without it must
give bit-identical tokens and fp32 logits.  The settings are read once per process, so each arm runs in a process of its
own."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# every W4 GEMM of this model runs the exact-integer kernel at batch 1 and 2, so with the prefetch on every boundary of the
# chain issues it: o_proj (2 MB) as a whole blob, gate_up / down / next qkv as their per-warp heads
_DECODE = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from zhilight_b200.llama import LlamaDecoder
cfg = dict(num_layers=3, dim_model=2048, num_heads=16, num_kv_heads=8, dim_head=128, dim_ff=5632, vocab_size=8192,
           eps=1e-5, rope_theta=500000.0, rope_llama3=None)
out = {}
for B in (1, 2):
    dec = LlamaDecoder(quant_type=5, sym=True, max_batch=B, max_seq=64, **cfg)
    dec.init_synthetic(7)
    tok = np.arange(3, 3 + B, dtype=np.int32) * 101
    for step in range(6):
        tok, logits = dec.decode(tok, np.full(B, step, np.int32), want_logits=True)
        out["tok_%d_%d" % (B, step)] = tok.copy()
        out["logits_%d_%d" % (B, step)] = logits
    dec.close()
np.savez(sys.argv[2], **out)
"""


@pytest.mark.gpu
def test_l2_head_prefetch_leaves_decode_bit_identical(tmp_path):
    runs = {}
    for arm, depth, whole_mb in (("off", "0", "0"), ("on", "4", "4")):
        env = dict(os.environ)
        env["ZL_W4_L2_HEAD"] = depth
        env["ZL_W4_L2_WHOLE_MB"] = whole_mb
        path = str(tmp_path / (arm + ".npz"))
        r = subprocess.run([sys.executable, "-c", _DECODE, ROOT, path], env=env, capture_output=True, text=True,
                           timeout=600)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
        runs[arm] = np.load(path)
    off, on = runs["off"], runs["on"]
    assert sorted(off.files) == sorted(on.files)
    for k in off.files:
        assert np.isfinite(off[k]).all(), k
        assert np.array_equal(off[k].view(np.uint8), on[k].view(np.uint8)), k
