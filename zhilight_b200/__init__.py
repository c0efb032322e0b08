"""zhilight_b200 -- H100-native (sm_90a) quantized-decode hot path of ZhiLight.

Only what the hot path needs: `csrc/` (CUDA kernels + the C-ABI of include/zhilight_b200.h),
`ops` (torch-tensor front end), `layers` (mirror of the reference's test-facing operator API,
tests/py_export_internal), `llama` (decode driver).  Importing the package does not load the
shared library; the first op call does, and raises if it is missing -- there is no CPU fallback.
"""
from ._lib import ZLError, load, LIB_PATH  # noqa: F401

__version__ = "0.1.0"
