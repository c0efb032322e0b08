"""CPU checks of the prompt prefix cache: the chained-key trie and LRU policy (zhilight_b200/prefix_cache.py), and the
C-ABI of the device block pool refusing bad arguments without a GPU."""
import ctypes
import random

import pytest

from zhilight_b200 import _lib
from zhilight_b200.prefix_cache import PrefixCache

BT = 4


def blk(v):
    """one block of BT tokens, all equal to v"""
    return [v] * BT


A, B, C, D, E, F = (blk(v) for v in (1, 2, 3, 4, 5, 6))


def test_chained_keys_never_match_a_block_after_another_prefix():
    pc = PrefixCache(8, BT)
    # cached with its tail: A and A/B are cached
    assert pc.insert(A + B + [9]) == [(0, 0), (1, 1)]
    # a per-block-index key would now find "B at index 1" after C; the trie only finds C
    assert pc.insert(C + [9]) == [(0, 2)]
    assert pc.match(C + B + [7, 7]) == [2]
    # the [A, B], [C, B], [C, B, ...] case: prompts of exactly two blocks cache their first block only
    pc = PrefixCache(8, BT)
    pc.insert(A + B)
    pc.insert(C + B)
    assert pc.match(C + B + [7]) == [pc.match(C + [0])[0]]
    assert len(pc.match(C + B + [7])) == 1
    # and B after C, once cached, is its own block, distinct from B after A
    pc = PrefixCache(8, BT)
    ab = pc.insert(A + B + [0])
    cb = pc.insert(C + B + [0])
    assert [b for _, b in ab] == [0, 1] and [b for _, b in cb] == [2, 3]
    assert pc.match(C + B + [5]) == [2, 3] and pc.match(A + B + [5]) == [0, 1]


def test_a_prompt_of_whole_blocks_leaves_its_last_block_to_prefill():
    pc = PrefixCache(8, BT)
    pc.insert(A + B + C + [0])
    for k in (1, 2, 3):
        assert len(pc.match((A + B + C)[:k * BT])) == k - 1
    assert len(pc.match(A + B + C + [0])) == 3
    assert pc.match([]) == [] and pc.match([1]) == []
    assert pc.insert(A) == []          # nothing match() could serve


def test_eviction_is_lru_over_leaves_and_parents_outlive_children():
    pc = PrefixCache(3, BT)
    assert pc.insert(A + B + [0]) == [(0, 0), (1, 1)]
    assert pc.insert(C + [0]) == [(0, 2)]
    # pool full.  A is the least recently used block but has a cached child: the LRU leaf is A/B (block 1)
    assert pc.insert(D + [0]) == [(0, 1)]
    assert pc.match(A + B + [0]) == [0]          # A survived, A/B went
    # now LRU order: C, D, A.  No leaf is older than C
    assert pc.insert(E + [0]) == [(0, 2)]
    assert pc.match(C + [0]) == []
    # a match refreshes: touch D, then the LRU leaf is A
    assert pc.match(D + [0]) == [1]
    assert pc.insert(F + [0]) == [(0, 0)]
    assert pc.match(A + [0]) == [] and pc.match(D + [0]) == [1] and pc.match(E + [0]) == [2]


def test_insert_never_evicts_its_own_path():
    pc = PrefixCache(2, BT)
    assert pc.insert(A + B + [0]) == [(0, 0), (1, 1)]
    # A/B/C needs a third block: the only leaf is on the prompt's own path, so insertion stops
    assert pc.insert(A + B + C + [0]) == []
    assert pc.match(A + B + C + [0]) == [0, 1]
    # a one-block prompt elsewhere takes the leaf A/B (its parent A stays while A/B exists, then becomes a leaf)
    assert pc.insert(D + [0]) == [(0, 1)]
    assert pc.match(A + B + [0]) == [0]


def test_identical_call_sequences_make_identical_decisions():
    def run(seed):
        rng = random.Random(seed)
        pc = PrefixCache(6, BT)
        log = []
        stems = [[rng.randrange(5) for _ in range(BT * rng.randrange(1, 4))] for _ in range(4)]
        for _ in range(200):
            prompt = list(rng.choice(stems)) + [rng.randrange(5) for _ in range(rng.randrange(1, 3 * BT))]
            log.append(("m", tuple(pc.match(prompt))))
            log.append(("i", tuple(pc.insert(prompt))))
            assert len(pc) <= 6
        return log

    assert run(1) == run(1)
    assert run(2) == run(2)


def test_header_exports_the_pool_entry_points(lib):
    protos = _lib.parse_header()
    for name in ("zl_llama_kv_pool_create", "zl_llama_kv_blocks_save", "zl_llama_kv_blocks_load",
                 "zl_llama_kv_blocks_bench"):
        assert name in protos, name
        assert hasattr(lib, name), name
    src = open(_lib.HEADER).read()
    assert "prefix_cache.hpp:35-117" in src and "batch_generator.cpp:626-645" in src and ":1213-1224" in src


def test_pool_entry_points_refuse_bad_arguments_without_a_gpu(lib):
    INVALID = -1
    blocks = (ctypes.c_int32 * 2)(0, 1)
    assert lib.zl_llama_kv_pool_create(None, 4, 128) == INVALID
    assert lib.zl_llama_kv_pool_create(None, 0, 128) == INVALID
    assert lib.zl_llama_kv_pool_create(None, 4, 100) == INVALID
    for fn in (lib.zl_llama_kv_blocks_save, lib.zl_llama_kv_blocks_load):
        assert fn(None, 0, blocks, blocks, 2) == INVALID
    ms, by = ctypes.c_float(), ctypes.c_double()
    assert lib.zl_llama_kv_blocks_bench(None, 0, blocks, blocks, 2, 1, 0, 1, ctypes.byref(ms), ctypes.byref(by)) == INVALID
    assert b"invalid argument" in lib.zl_last_error()


def test_prefill_cached_without_a_pool_is_refused():
    from zhilight_b200.llama import LlamaDecoder
    dec = LlamaDecoder.__new__(LlamaDecoder)      # no device needed: the check is on the host
    with pytest.raises(RuntimeError):
        dec.prefill_cached(0, [1, 2, 3])
