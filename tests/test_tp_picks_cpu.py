"""Full-vocabulary picks under tensor parallelism without a GPU: the C-ABI of the vocabulary all-gather and of
zl_llama_set_vocab_gather, and the refusals that run before any device memory is touched."""
import ctypes

from zhilight_b200 import _lib

INVALID, UNSUPPORTED = -1, -2


def test_header_declares_the_gather():
    p = _lib.parse_header()
    assert [a for _, a in p["zl_vocab_gather_create"][1]] == ["rank", "world_size", "max_rows", "vocab", "out"]
    assert [a for _, a in p["zl_vocab_allgather"][1]] == ["g", "shard", "rows", "ld", "pdl", "stream"]
    assert [a for _, a in p["zl_llama_set_vocab_gather"][1]] == ["m", "g"]
    for name in ("zl_vocab_gather_destroy", "zl_vocab_gather_get_ipc_handle", "zl_vocab_gather_open_peers",
                 "zl_vocab_gather_info", "zl_vocab_gather_buffer"):
        assert name in p, name


def test_create_refusals(lib):
    h = ctypes.c_void_p()
    for args, code in [((0, 0, 4, 512), INVALID),          # world size
                       ((0, 9, 4, 512), INVALID),
                       ((2, 2, 4, 512), INVALID),          # rank
                       ((-1, 2, 4, 512), INVALID),
                       ((0, 1, 0, 512), INVALID),          # rows
                       ((0, 3, 4, 512), INVALID),          # vocab % world size
                       ((0, 1, 1 << 20, 1 << 12), INVALID),   # max_rows * vocab >= 2^31
                       ((0, 1, 4, 514), UNSUPPORTED),      # shard rows of 16-byte vectors
                       ((1, 2, 4, 1028), UNSUPPORTED),
                       ((0, 8, 4, 128256 + 8), UNSUPPORTED)]:
        assert lib.zl_vocab_gather_create(*args, ctypes.byref(h)) == code, args
    assert lib.zl_vocab_gather_create(0, 1, 4, 512, None) == INVALID


def test_null_object_refusals(lib):
    buf = ctypes.create_string_buffer(64)
    i = ctypes.c_int()
    assert lib.zl_vocab_allgather(None, None, 1, 512, 0, None) == INVALID
    assert lib.zl_vocab_gather_get_ipc_handle(None, buf) == INVALID
    assert lib.zl_vocab_gather_open_peers(None, buf) == INVALID
    assert lib.zl_vocab_gather_info(None, ctypes.byref(i), ctypes.byref(i), ctypes.byref(i), ctypes.byref(i)) == INVALID
    assert not lib.zl_vocab_gather_buffer(None)
    lib.zl_vocab_gather_destroy(None)
    assert lib.zl_llama_set_vocab_gather(None, None) == INVALID
