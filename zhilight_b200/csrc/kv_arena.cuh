// Placement of every task's KV rows in the decode driver's per-layer row space (kv_arena.cu).  The row space has the same
// layout in every layer and in K, V and the int8 scales, so one placement serves them all; the per-layer device pointer
// tables (Layer::k_addrs ...) hold base + first[task] * row bytes and are rewritten by k_kv_relocate when a task moves.
//
// Fixed layout (kv_rows = 0): task t owns rows [t max_seq, (t + 1) max_seq) for good; nothing ever grows or moves.
// Arena (kv_rows > 0): tasks start empty and are granted rows in units of kGrant as their writes reach them.  A grant grows
// a task geometrically, to min(max(need, 2 cap), max_seq) rounded up to kGrant, or to the least multiple of kGrant that
// holds `need` when that does not fit.  It takes, in this order: the free rows right after the task (in place), the
// smallest free extent that holds it (best fit, the lowest on a tie; the task's rows move there), or a compaction that
// packs the tasks below the growing one downwards and those above it upwards so that every free row lies right after it.
// A compaction move whose destination overlaps its source is split into pieces no longer than the distance moved, so the
// destination of every move is disjoint from its source.  A call that grants several tasks is planned with the geometric
// sizes first and, when they do not all fit, again from the start with every task at its least size; it is refused
// exactly when the least sizes exceed the free rows plus the tasks' own.
#pragma once
#include <cstdint>
#include <utility>
#include <vector>

namespace zl {

// One extent of a relocation, in rows of the row space: rows [src, src + copy) move to [dst, dst + copy), then rows
// [dst + copy, dst + copy + zero) are zero-filled.  copy = 0: a zero fill only (src = dst).
struct KvMove {
    int32_t src, dst, copy, zero;
};

struct KvArena {
    // grant unit: 64 rows keeps every task base 16-byte aligned for any row and scale-row size (64 x 4-byte scales),
    // holds any prefix-cache block of up to 64 tokens whole, and bounds a task's moves to log2(max_seq / 64) + 1
    static constexpr int kGrant = 64;

    bool fixed = true;
    int rows = 0;        // rows of the row space
    int max_seq = 0;
    std::vector<int32_t> first, cap;   // per task; cap 0: no rows (first 0)

    // kv_rows 0: the fixed layout; else kv_rows (1 .. max_batch * max_seq) rounded up to kGrant.  ZL_ERR_INVALID_ARG
    // outside that range.
    int init(int kv_rows, int max_batch, int max_seq);
    // rows granted in units of: kGrant, or max_seq in the fixed layout
    int unit() const { return fixed ? max_seq : kGrant; }
    int free_rows() const;
    // Plans giving every task of `needs` {task, rows (<= max_seq)} at least that many rows (a task named twice gets the
    // larger).  On success stores the arena after the grants in *next, appends the relocation to *launches (launch i must
    // complete before launch i + 1 starts: no move of a launch overlaps another of the same launch, in source or
    // destination) and returns ZL_OK; else returns ZL_ERR_KV_FULL.  Changes nothing itself: the caller commits *next.
    int plan(const std::vector<std::pair<int, int>>& needs, KvArena* next,
             std::vector<std::vector<KvMove>>* launches) const;
    // returns the task's rows to the free space (a no-op in the fixed layout)
    void release(int task);

   private:
    bool grow(int task, int need, bool least_only, std::vector<KvMove>* seq);
    bool place(int task, int size, bool compact, std::vector<KvMove>* seq);
};

}  // namespace zl
