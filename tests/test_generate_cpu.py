"""Generate-until-stop without a GPU: the stop rule checks of LlamaDecoder.set_stop and the C-ABI refusals that run
before the model is touched."""
import ctypes

import numpy as np
import pytest

from zhilight_b200.llama import MAX_STOP_IDS, stop_rule

INVALID = -1


def test_stop_rule_accepts():
    ids, budget = stop_rule([2, 0, 511], 16, 512)
    assert ids.dtype == np.int32 and list(ids) == [2, 0, 511] and budget == 16
    ids, budget = stop_rule((), 0, 512)                       # no stop ids, no budget
    assert ids.size == 0 and budget == 0
    assert stop_rule(range(MAX_STOP_IDS), 1, 512)[0].size == MAX_STOP_IDS


@pytest.mark.parametrize("ids,budget", [
    ([512], 0), ([-1], 0),                # ids out of range
    ([3, 7, 3], 0),                       # repeated id
    (list(range(MAX_STOP_IDS + 1)), 0),   # more than 8 ids
    ([1], -1),                            # negative budget
    ([1], 2.5),                           # a budget that is not a whole number
])
def test_stop_rule_refuses(ids, budget):
    with pytest.raises(ValueError):
        stop_rule(ids, budget, 512)


def test_null_model_refusals(lib):
    """A NULL model is refused before anything else is looked at."""
    out = np.zeros(4, np.int32)
    p = out.ctypes.data_as(ctypes.c_void_p)
    steps = ctypes.c_int()
    assert lib.zl_llama_generate(None, 1, 1, p, p, p, ctypes.byref(steps)) == INVALID
    assert lib.zl_llama_generate(None, 0, 0, None, None, None, None) == INVALID
    ids = np.array([1, 2], np.int32)
    assert lib.zl_llama_set_stop(None, 0, ids.ctypes.data_as(ctypes.c_void_p), 2, 0) == INVALID
    assert lib.zl_llama_set_stop(None, 0, None, 0, 4) == INVALID
