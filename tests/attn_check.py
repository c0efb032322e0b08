"""Checks shared by the attention tests: which kernels a call launched, and closeness to a float64 reference over the
whole output and over every (task, query, head) row."""
import numpy as np
import torch


def launched(fn):
    """fn()'s result and the names of the kernels it launched.  The profiler now and then delivers a session's runtime
    calls without some or all of the kernels' device records; such a session is run again (fn is deterministic)."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        events = prof.key_averages()
        names = [e.key for e in events]
        launches = sum(e.count for e in events if e.key.startswith("cudaLaunchKernel"))
        kernels = sum(e.count for e in events
                      if e.device_type == DeviceType.CUDA and not e.key.startswith(("Memcpy", "Memset")))
        if kernels >= launches:
            break
    return out, names


def assert_close(out, ref, tol, what=""):
    """rel L2 <= tol over everything and <= 4 tol on each (task, query, head) row; rows whose reference is 0 (fully
    masked) must be exactly 0."""
    o = out.double()
    assert torch.isfinite(o).all(), what
    assert ((o - ref).norm() / ref.norm()).item() <= tol, (what, ((o - ref).norm() / ref.norm()).item())
    d = ref.shape[-1]
    rn, en = ref.reshape(-1, d).norm(dim=1), (o - ref).reshape(-1, d).norm(dim=1)
    dead = rn == 0
    assert (en[dead] == 0).all(), what
    if (~dead).any():
        rel = en[~dead] / rn[~dead]
        worst = int(rel.argmax())
        row = int(torch.nonzero(~dead)[worst])
        assert rel[worst].item() <= 4 * tol, (what, "row (task, query, head)", np.unravel_index(row, ref.shape[:-1]),
                                              rel[worst].item())
