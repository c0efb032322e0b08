"""KV arena placement decisions (zl_kv_arena_replay), no device: grants, growth, release and compaction keep live tasks
disjoint, move every row a task holds to its new place, zero-fill what they grant, and refuse a call exactly when the
least sizes of its tasks exceed the free rows plus their own."""
import numpy as np
import pytest

from zhilight_b200 import _lib
from zhilight_b200.llama import KV_FULL, kv_arena_replay

G = 64   # grant unit


def rup(x):
    return -(-x // G) * G


def overlap(a0, n0, a1, n1):
    return n0 > 0 and n1 > 0 and a0 < a1 + n1 and a1 < a0 + n0


def _pairs(call):
    return [tuple(call)] if np.ndim(call) == 1 else [tuple(p) for p in call]


def check_replay(kv_rows, max_batch, max_seq, ops):
    """ops: calls, each (task, rows) or a list of them.  -> per call: result, extents after it; and the moves"""
    res_p, ext_p, moves = kv_arena_replay(kv_rows, max_batch, max_seq, ops)
    starts = np.cumsum([0] + [len(_pairs(c)) for c in ops])[:-1]
    for c, i0 in enumerate(starts):   # every pair of a call reports the call's result and extents
        k = len(_pairs(ops[c]))
        assert (res_p[i0:i0 + k] == res_p[i0]).all() and (ext_p[i0:i0 + k] == ext_p[i0]).all()
    res, ext = res_p[starts], ext_p[starts]
    rows = rup(kv_rows)
    mem = np.zeros(rows, np.int64)          # tag of what each row holds: task * 10^6 + row + 1, 0 = zero
    first = np.zeros(max_batch, np.int64)
    cap = np.zeros(max_batch, np.int64)
    by_op = {}
    first_op = {int(i0): c for c, i0 in enumerate(starts)}
    for m in moves:
        by_op.setdefault(first_op[int(m[0])], []).append(m)
    for i, call in enumerate(ops):
        pairs = _pairs(call)
        needs = {}
        for t, r in pairs:
            needs[t] = max(needs.get(t, 0), r)
        task, need = pairs[0]
        # the op's moves, launch by launch: every launch reads its sources before it writes
        launches = {}
        for m in by_op.get(i, []):
            launches.setdefault(int(m[1]), []).append(m)
        for lid in sorted(launches):
            l = launches[lid]
            for a in range(len(l)):
                _, _, s, d, c, z = (int(x) for x in l[a])
                assert c == 0 or not overlap(s, c, d, c + z), ("a move overlaps its own source", l[a])
                assert d >= 0 and d + c + z <= rows and s >= 0 and s + c <= rows
                assert (c + z) % G == 0 and d % G == 0
                for b in range(a + 1, len(l)):
                    _, _, s2, d2, c2, z2 = (int(x) for x in l[b])
                    assert not overlap(d, c + z, s2, c2) and not overlap(s, c, d2, c2 + z2), "moves of a launch clash"
                    assert not overlap(d, c + z, d2, c2 + z2), "two moves of a launch write the same rows"
            reads = [mem[int(m[2]):int(m[2]) + int(m[4])].copy() for m in l]
            for m, r in zip(l, reads):
                d, c, z = int(m[3]), int(m[4]), int(m[5])
                mem[d:d + c] = r
                mem[d + c:d + c + z] = 0
        f1, c1 = ext[i, :, 0].astype(np.int64), ext[i, :, 1].astype(np.int64)
        if need == 0:
            assert len(pairs) == 1 and res[i] == 0 and c1[task] == 0
        else:
            short = sum(rup(r) - cap[t] for t, r in needs.items() if r > cap[t]) > rows - cap.sum()
            assert (res[i] == KV_FULL) == short, (i, needs, res[i], cap, rows)
            if res[i] == KV_FULL:
                assert not by_op.get(i) and (f1 == first).all() and (c1 == cap).all(), "a refusal changed the arena"
            else:
                assert all(c1[t] >= r and c1[t] % G == 0 for t, r in needs.items())
        # live extents: in range and disjoint; every task kept its rows' contents, and what it gained is zero
        live = [t for t in range(max_batch) if c1[t] > 0]
        for t in live:
            assert 0 <= f1[t] and f1[t] + c1[t] <= rows
            for u in live:
                assert t == u or not overlap(f1[t], c1[t], f1[u], c1[u]), (t, u, f1, c1)
            old = cap[t] if not (need == 0 and t == task) else 0
            kept = min(old, c1[t])
            want = t * 10**6 + np.arange(kept) + 1
            assert (mem[f1[t]:f1[t] + kept] == want).all(), ("task %d lost rows" % t, i)
            if c1[t] > old:
                assert (mem[f1[t] + old:f1[t] + c1[t]] == 0).all(), ("granted rows not zero-filled", t, i)
        for t in live:   # the tasks write every row they hold
            mem[f1[t]:f1[t] + c1[t]] = t * 10**6 + np.arange(c1[t]) + 1
        first, cap = f1, c1
    return res, ext, moves


def random_ops(rng, max_batch, max_seq, n):
    ops, cap = [], [0] * max_batch
    for _ in range(n):
        t = int(rng.integers(max_batch))
        if rng.random() < 0.2:
            ops.append((t, 0))
            cap[t] = 0
        else:
            need = min(max_seq, cap[t] + int(rng.integers(1, max_seq // 2 + 2)))
            ops.append((t, need))
            cap[t] = max(cap[t], need)
    return ops


def random_calls(rng, max_batch, max_seq, n):
    """calls of up to max_batch tasks growing together, as a decode step, generate or a joined step grants them"""
    calls, cap = [], [0] * max_batch
    for _ in range(n):
        if rng.random() < 0.2:
            t = int(rng.integers(max_batch))
            calls.append((t, 0))
            cap[t] = 0
            continue
        tasks = rng.choice(max_batch, int(rng.integers(1, max_batch + 1)), replace=False)
        call = []
        for t in tasks:
            need = min(max_seq, cap[t] + int(rng.integers(1, max_seq // 3 + 2)))
            call.append((int(t), need))
            cap[t] = max(cap[t], need)
        calls.append(call)
    return calls


@pytest.mark.parametrize("kv_rows,max_batch,max_seq", [(1024, 4, 512), (1000, 8, 300), (4096, 16, 1024), (640, 6, 640)])
@pytest.mark.parametrize("seed", range(6))
def test_random_sequences(kv_rows, max_batch, max_seq, seed):
    rng = np.random.default_rng(seed * 131 + kv_rows)
    check_replay(kv_rows, max_batch, max_seq, random_ops(rng, max_batch, max_seq, 120))


@pytest.mark.parametrize("kv_rows,max_batch,max_seq", [(1024, 4, 512), (1000, 8, 300), (4096, 16, 1024), (640, 6, 640)])
@pytest.mark.parametrize("seed", range(6))
def test_random_multi_task_calls(kv_rows, max_batch, max_seq, seed):
    rng = np.random.default_rng(seed * 977 + kv_rows)
    res, _, _ = check_replay(kv_rows, max_batch, max_seq, random_calls(rng, max_batch, max_seq, 80))
    assert (res == 0).any() and (res == KV_FULL).any()


def test_multi_task_call_falls_back_to_least_sizes():
    # tasks 0 and 1 hold 128 rows each of 384; both need 129: doubling task 0 to 256 would starve task 1, but two least
    # grants of 192 fill the arena exactly
    res, ext, _ = check_replay(384, 2, 512, [(0, 128), (1, 128), [(0, 129), (1, 129)]])
    assert list(res) == [0, 0, 0] and list(ext[-1, :, 1]) == [192, 192]
    # one row more than fits is refused
    res, _, _ = check_replay(384, 2, 512, [(0, 128), (1, 128), [(0, 129), (1, 193)]])
    assert res[-1] == KV_FULL


def test_decisions_are_a_function_of_the_calls():
    ops = random_ops(np.random.default_rng(7), 8, 512, 200)
    a = kv_arena_replay(2048, 8, 512, ops)
    b = kv_arena_replay(2048, 8, 512, ops)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def test_compaction_slides_in_pieces():
    # [free 64][task 1: 192][free 64] and task 0 needs 128: task 1 must move by 64 rows, less than its length
    ops = [(0, 64), (1, 192), (0, 0), (2, 64), (2, 0), (0, 128)]
    res, ext, moves = check_replay(320, 3, 256, ops)
    assert res[-1] == 0
    pieces = [m for m in moves if m[0] == len(ops) - 1 and m[4] > 0]
    assert len(pieces) >= 2 and all(m[4] <= abs(m[2] - m[3]) for m in pieces)
    assert len({int(m[1]) for m in pieces}) == len(pieces), "overlapping pieces share no launch"


def test_full_arena_refuses_then_serves_after_release():
    ops = [(0, 128), (1, 128), (2, 1), (1, 0), (2, 1)]
    res, ext, _ = check_replay(256, 3, 128, ops)
    assert list(res) == [0, 0, KV_FULL, 0, 0]


def test_geometric_growth_moves_a_task_logarithmically():
    max_seq = 4096
    ops = [(0, r) for r in range(1, max_seq + 1)] + [(1, 64)]
    ops = [(1, 64)] + ops   # a neighbour right after task 0 forces every growth to move
    res, ext, moves = kv_arena_replay(max_seq + 4 * G, 2, max_seq, ops)
    assert (res == 0).all()
    grants = len({int(m[0]) for m in moves if m[2] != m[3] or m[5] > 0})
    assert grants <= 2 + int(np.log2(max_seq // G)) + 1, grants


def test_fixed_layout():
    res, ext, moves = kv_arena_replay(0, 4, 100, [(0, 100), (1, 0), (3, 1)])
    assert (res == 0).all() and len(moves) == 0
    assert (ext[:, :, 0] == np.arange(4) * 100).all() and (ext[:, :, 1] == 100).all()


@pytest.mark.parametrize("kv_rows", [-1, 4 * 100 + 1])
def test_bad_kv_rows(kv_rows):
    with pytest.raises(_lib.ZLError):
        kv_arena_replay(kv_rows, 4, 100, [(0, 1)])
