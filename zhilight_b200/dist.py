"""Tensor-parallel plumbing: one process per GPU, torch.distributed for bootstrap only.

* `shard_state_dict` restates the reference's TP split of a checkpoint (column-parallel q/k/v/gate/up slice the
  output dim, row-parallel attn_out/w_out slice the input dim; src/nn/linear/linear.cpp:1212-1234,
  3rd/bmengine/bmengine/core/context.cpp:739-789, attention.cpp:96-99, feedforward.cpp:85-87), lm_head is
  vocab-parallel (src/nn/embedding/embedding.cu:353-392), the embedding table and the norms are replicated.
* `TPComm` owns the NVLink peer-memory exchange object (zl_comm_*): the symmetric buffers are mapped with
  CUDA IPC, the handles travel through `torch.distributed.all_gather_object` (gloo or nccl).
* `VocabGather` owns the vocabulary all-gather (zl_vocab_gather_*) that lets every rank sample from whole rows.
"""
import ctypes

import numpy as np

from . import _lib

COLUMN = ("attn.project_q", "attn.project_k", "attn.project_v", "ff.w_in", "ff.w_gated")
ROW = ("attn.attn_out", "ff.w_out")


def _slice(a, axis, rank, ws, unit=1):
    n = a.shape[axis]
    if n % (ws * unit) != 0:
        raise ValueError("dimension %d not divisible by tp=%d (unit %d)" % (n, ws, unit))
    step = n // ws
    idx = [slice(None)] * a.ndim
    idx[axis] = slice(rank * step, (rank + 1) * step)
    return np.ascontiguousarray(a[tuple(idx)])


def shard_tensor(name, a, rank, ws, group_size=128, is_awq=False):
    """Return rank's shard of checkpoint tensor `name` (numpy, HF/ZhiLight layout)."""
    a = np.asarray(a)
    if ws == 1:
        return a
    base, _, leaf = name.rpartition(".")
    col = any(base.endswith(s) for s in COLUMN)
    row = any(base.endswith(s) for s in ROW)
    if name == "lm_head.weight":
        return _slice(a, 0, rank, ws)                    # vocab-parallel rows
    if not (col or row):
        return a                                         # norms, embedding: replicated
    if leaf == "weight":                                 # dense (N, K)
        return _slice(a, 0 if col else 1, rank, ws)
    if leaf == "bias":
        return _slice(a, 0, rank, ws) if col else (a if rank == 0 else np.zeros_like(a))
    if leaf == "g_idx":
        return a if col else _slice(a, 0, rank, ws)
    if leaf in ("qweight", "qzeros", "scales"):
        if is_awq:
            # AWQ: qweight (K, N/8), qzeros (K/g, N/8), scales (K/g, N)
            if col:
                return _slice(a, 1, rank, ws)
            unit = {"qweight": group_size, "qzeros": 1, "scales": 1}[leaf]
            return _slice(a, 0, rank, ws, unit)
        # GPTQ: qweight (K/8, N), qzeros (K/g, N/8), scales (K/g, N)
        if col:
            return _slice(a, 1, rank, ws)                # last dim: N, N/8 words, N
        unit = {"qweight": group_size // 8, "qzeros": 1, "scales": 1}[leaf]   # (K/ws) % g == 0
        return _slice(a, 0, rank, ws, unit)
    return a


def shard_state_dict(sd, rank, ws, group_size=128, is_awq=False):
    return {k: shard_tensor(k, v, rank, ws, group_size, is_awq) for k, v in sd.items()}


def exchange_bytes(payload, group=None):
    """all-gather one bytes object per rank (rank order) over torch.distributed."""
    import torch.distributed as dist
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return [payload]
    out = [None] * dist.get_world_size(group)
    dist.all_gather_object(out, payload, group=group)
    return out


def _world(rank, world_size, group):
    import torch.distributed as dist
    if rank is None:
        rank = dist.get_rank(group) if dist.is_initialized() else 0
    if world_size is None:
        world_size = dist.get_world_size(group) if dist.is_initialized() else 1
    return rank, world_size


def open_ipc_peers(lib, prefix, handle, world_size, group=None):
    """Map every rank's symmetric buffer of a zl_<prefix> object into this process: all-gather the CUDA IPC handles
    (zl_<prefix>_get_ipc_handle), open them (zl_<prefix>_open_peers), then wait for every rank.  Collective."""
    import torch.distributed as dist
    if world_size == 1:
        return
    nb = lib.zl_comm_ipc_handle_bytes()
    buf = ctypes.create_string_buffer(nb)
    _lib.check(getattr(lib, "zl_%s_get_ipc_handle" % prefix)(handle, buf))
    all_h = exchange_bytes(buf.raw, group)
    assert len(all_h) == world_size and all(len(x) == nb for x in all_h)
    blob = ctypes.create_string_buffer(b"".join(all_h), nb * world_size)
    _lib.check(getattr(lib, "zl_%s_open_peers" % prefix)(handle, blob))
    dist.barrier(group)


class TPComm:
    """zl_comm wrapper.  max_elems = largest all-reduce message in 16-bit elements (max_batch * dim_model)."""

    def __init__(self, max_elems, rank=None, world_size=None, group=None):
        self.lib = _lib.load()
        rank, world_size = _world(rank, world_size, group)
        self.rank, self.world_size = rank, world_size
        h = ctypes.c_void_p()
        max_elems = (int(max_elems) + 31) // 32 * 32
        _lib.check(self.lib.zl_comm_create(rank, world_size, max_elems, ctypes.byref(h)))
        self.handle = h
        open_ipc_peers(self.lib, "comm", self.handle, world_size, group)

    def allreduce(self, partial, residual=None, int8=False, out=None):
        import torch
        from .ops import _dt, _p, _stream
        out = torch.empty_like(partial) if out is None else out
        _lib.call("zl_allreduce_one_shot", self.handle, _p(partial), _p(residual), _p(out), partial.numel(),
                  _dt(partial), int(int8), 0, _stream())
        return out

    def allgather(self, t):
        import torch
        from .ops import _p, _stream
        nbytes = t.numel() * t.element_size()
        out = torch.empty((self.world_size,) + tuple(t.shape), dtype=t.dtype, device=t.device)
        _lib.call("zl_allgather_small", self.handle, _p(t), _p(out), nbytes, 0, _stream())
        return out

    def close(self):
        if getattr(self, "handle", None):
            self.lib.zl_comm_destroy(self.handle)
            self.handle = None


class _DeviceArray:
    """__cuda_array_interface__ of a device buffer the library owns, for torch.as_tensor."""

    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = dict(shape=shape, typestr=typestr, data=(ptr, False), version=3, strides=None)


class VocabGather:
    """zl_vocab_gather wrapper: every rank's (rows, vocab / ws) fp32 logit shard into a (max_rows, vocab) buffer on every
    rank.  Collective: every rank constructs it with the same max_rows and vocab."""

    def __init__(self, max_rows, vocab, rank=None, ws=None, group=None):
        self.lib = _lib.load()
        rank, ws = _world(rank, ws, group)
        self.rank, self.world_size, self.max_rows, self.vocab = rank, ws, int(max_rows), int(vocab)
        h = ctypes.c_void_p()
        _lib.check(self.lib.zl_vocab_gather_create(rank, ws, self.max_rows, self.vocab, ctypes.byref(h)))
        self.handle = h
        open_ipc_peers(self.lib, "vocab_gather", self.handle, ws, group)

    def gather(self, shard, pdl=False):
        """Enqueue the all-gather of shard (rows, vocab / ws) fp32, a CUDA tensor with 16-byte aligned rows, on torch's
        current stream; -> buffer(rows)."""
        import torch
        from .ops import _stream
        if (not shard.is_cuda or shard.dtype != torch.float32 or shard.dim() != 2 or shard.stride(1) != 1
                or shard.shape[1] != self.vocab // self.world_size):
            raise _lib.ZLError(-1, "shard must be a (rows, vocab / ws) float32 CUDA tensor with unit column stride")
        rows, ld = shard.shape[0], shard.stride(0)
        _lib.call("zl_vocab_allgather", self.handle, ctypes.c_void_p(shard.data_ptr()), rows, ld, int(pdl), _stream())
        return self.buffer(rows)

    def buffer(self, rows=None):
        """The first rows (default max_rows) of this rank's gather buffer, as a float32 CUDA tensor that aliases it."""
        import torch
        rows = self.max_rows if rows is None else int(rows)
        ptr = self.lib.zl_vocab_gather_buffer(self.handle)
        return torch.as_tensor(_DeviceArray(ptr, (rows, self.vocab), "<f4"), device="cuda")

    def close(self):
        if getattr(self, "handle", None):
            self.lib.zl_vocab_gather_destroy(self.handle)
            self.handle = None
