// Host-side KV arena of the decode driver: which rows of the per-layer row space each task holds (kv_arena.cuh).
#include "common.cuh"
#include "kv_arena.cuh"

#include <algorithm>
#include <climits>

namespace zl {
namespace {

int round_up(int x, int g) { return (x + g - 1) / g * g; }

bool overlap(int a0, int n0, int a1, int n1) { return n0 > 0 && n1 > 0 && a0 < a1 + n1 && a1 < a0 + n0; }

// two moves that may not share a launch: one writes rows the other reads or writes
bool conflict(const KvMove& a, const KvMove& b) {
    return overlap(a.dst, a.copy + a.zero, b.src, b.copy) || overlap(a.src, a.copy, b.dst, b.copy + b.zero) ||
           overlap(a.dst, a.copy + a.zero, b.dst, b.copy + b.zero);
}

// rows [s, s + n) to [d, d + n): one move when the ranges are disjoint, else pieces no longer than |s - d| in the order
// that reads every piece before a later one overwrites it
void slide(int s, int d, int n, std::vector<KvMove>* seq) {
    if (s == d || n == 0) return;
    const int k = s > d ? s - d : d - s;
    if (k >= n) {
        seq->push_back({s, d, n, 0});
    } else if (d < s) {
        for (int o = 0; o < n; o += k) seq->push_back({s + o, d + o, std::min(k, n - o), 0});
    } else {
        for (int o = n; o > 0; o -= k) {
            const int len = std::min(k, o);
            seq->push_back({s + o - len, d + o - len, len, 0});
        }
    }
}

struct Ext {
    int first, len, task;
};

}  // namespace

int KvArena::init(int kv_rows, int max_batch, int max_seq_) {
    const long long all = (long long)max_batch * max_seq_;
    if (kv_rows < 0 || kv_rows > all || all > INT_MAX - kGrant) return ZL_ERR_INVALID_ARG;
    fixed = kv_rows == 0;
    max_seq = max_seq_;
    first.assign(max_batch, 0);
    cap.assign(max_batch, 0);
    if (fixed) {
        rows = (int)all;
        for (int t = 0; t < max_batch; ++t) {
            first[t] = t * max_seq;
            cap[t] = max_seq;
        }
    } else {
        rows = round_up(kv_rows, kGrant);
    }
    return ZL_OK;
}

int KvArena::free_rows() const {
    if (fixed) return 0;
    int used = 0;
    for (int c : cap) used += c;
    return rows - used;
}

void KvArena::release(int task) {
    if (fixed) return;
    first[task] = 0;
    cap[task] = 0;
}

bool KvArena::place(int task, int size, bool compact, std::vector<KvMove>* seq) {
    const int f = first[task], c = cap[task];
    std::vector<Ext> live;   // the other tasks' extents by address
    for (int t = 0; t < (int)cap.size(); ++t)
        if (t != task && cap[t] > 0) live.push_back({first[t], cap[t], t});
    std::sort(live.begin(), live.end(), [](const Ext& a, const Ext& b) { return a.first < b.first; });
    if (!compact) {
        if (c > 0) {   // in place: the free rows right after the task
            int next = rows;
            for (const Ext& e : live)
                if (e.first >= f + c) {
                    next = e.first;
                    break;
                }
            if (next - f >= size) {
                seq->push_back({f + c, f + c, 0, size - c});
                cap[task] = size;
                return true;
            }
        }
        // best fit among the free extents (the task's own rows are not free: the move's destination avoids its source)
        std::vector<Ext> all = live;
        if (c > 0) all.push_back({f, c, task});
        std::sort(all.begin(), all.end(), [](const Ext& a, const Ext& b) { return a.first < b.first; });
        int best = -1, best_len = INT_MAX, at = 0;
        for (size_t i = 0; i <= all.size(); ++i) {
            const int end = i < all.size() ? all[i].first : rows;
            if (end - at >= size && end - at < best_len) {
                best = at;
                best_len = end - at;
            }
            if (i < all.size()) at = all[i].first + all[i].len;
        }
        if (best < 0) return false;
        seq->push_back({c > 0 ? f : best, best, c, size - c});
        first[task] = best;
        cap[task] = size;
        return true;
    }
    if (free_rows() + c < size) return false;
    // compaction: the tasks below this one pack downwards from row 0, this one follows them, the tasks above it pack
    // upwards from the end; every free row then lies right after this task
    const int key = c > 0 ? f : INT_MAX;   // a task without rows packs after all others
    int p = 0;
    for (const Ext& e : live)
        if (e.first < key) {
            slide(e.first, p, e.len, seq);
            first[e.task] = p;
            p += e.len;
        }
    slide(f, p, c, seq);
    int q = rows;
    for (auto it = live.rbegin(); it != live.rend(); ++it)
        if (it->first > key) {
            q -= it->len;
            slide(it->first, q, it->len, seq);
            first[it->task] = q;
        }
    seq->push_back({p + c, p + c, 0, size - c});
    first[task] = p;
    cap[task] = size;
    return true;
}

// least_only: the least multiple of kGrant that holds `need`, never the geometric target
bool KvArena::grow(int task, int need, bool least_only, std::vector<KvMove>* seq) {
    const int c = cap[task];
    if (c >= need) return true;
    const int least = round_up(need, kGrant);
    const int target = least_only ? least : round_up(std::min(std::max(need, 2 * c), max_seq), kGrant);
    for (bool compact : {false, true}) {
        if (place(task, target, compact, seq)) return true;
        if (least != target && place(task, least, compact, seq)) return true;
    }
    return false;
}

int KvArena::plan(const std::vector<std::pair<int, int>>& needs, KvArena* next,
                  std::vector<std::vector<KvMove>>* launches) const {
    std::vector<std::pair<int, int>> merged;   // one need per task, the largest, in order of first appearance
    for (const auto& n : needs) {
        auto it = std::find_if(merged.begin(), merged.end(), [&](const std::pair<int, int>& m) { return m.first == n.first; });
        if (it == merged.end())
            merged.push_back(n);
        else
            it->second = std::max(it->second, n.second);
    }
    *next = *this;
    bool met = true;
    for (const auto& n : merged) met = met && cap[n.first] >= n.second;
    if (met) return ZL_OK;
    // geometric sizes first: an early task's doubling can starve a later one, so the whole call is planned again at the
    // least sizes before it is refused; a plan at the least sizes exists whenever they fit the free rows plus the tasks' own
    std::vector<KvMove> seq;
    bool ok = false;
    for (bool least_only : {false, true}) {
        *next = *this;
        seq.clear();
        ok = true;
        for (const auto& n : merged)
            if (!next->grow(n.first, n.second, least_only, &seq)) {
                ok = false;
                break;
            }
        if (ok) break;
    }
    if (!ok) {
        *next = *this;
        return ZL_ERR_KV_FULL;
    }
    // a move joins the current launch unless it touches rows a move of that launch reads or writes
    bool fresh = true;
    for (const KvMove& mv : seq) {
        bool clash = fresh;
        if (!clash)
            for (const KvMove& o : launches->back())
                if (conflict(mv, o)) {
                    clash = true;
                    break;
                }
        if (clash) launches->emplace_back();
        launches->back().push_back(mv);
        fresh = false;
    }
    return ZL_OK;
}

}  // namespace zl

extern "C" int zl_kv_arena_replay(int kv_rows, int max_batch, int max_seq, const int32_t* ops, int n_ops,
                                  int32_t* results, int32_t* extents, int32_t* moves, int max_moves, int* n_moves) {
    ZL_CHECK_ARG(max_batch > 0 && max_seq > 0 && n_ops >= 0 && (n_ops == 0 || (ops && results && extents)));
    ZL_CHECK_ARG(max_moves >= 0 && (max_moves == 0 || moves) && n_moves);
    zl::KvArena a;
    ZL_CHECK_ARG(a.init(kv_rows, max_batch, max_seq) == ZL_OK);
    for (int i = 0; i < n_ops; ++i) {
        const int32_t* o = ops + 3 * i;   // {call, task, rows}
        ZL_CHECK_ARG(o[1] >= 0 && o[1] < max_batch && o[2] >= 0 && o[2] <= max_seq);
        ZL_CHECK_ARG(o[2] > 0 || ((i == 0 || ops[3 * i - 3] != o[0]) && (i + 1 == n_ops || ops[3 * i + 3] != o[0])));
    }
    int nm = 0, nl = 0;
    for (int i = 0; i < n_ops;) {
        int j = i + 1;   // the call: ops i .. j - 1
        while (j < n_ops && ops[3 * j] == ops[3 * i]) ++j;
        int rc = ZL_OK;
        if (ops[3 * i + 2] == 0) {
            a.release(ops[3 * i + 1]);
        } else {
            std::vector<std::pair<int, int>> needs;
            for (int k = i; k < j; ++k) needs.push_back({ops[3 * k + 1], ops[3 * k + 2]});
            std::vector<std::vector<zl::KvMove>> launches;
            zl::KvArena next;
            rc = a.plan(needs, &next, &launches);
            a = std::move(next);
            for (const auto& l : launches) {
                for (const zl::KvMove& mv : l) {
                    if (nm < max_moves) {
                        int32_t* o = moves + 6 * (size_t)nm;
                        o[0] = i;
                        o[1] = nl;
                        o[2] = mv.src;
                        o[3] = mv.dst;
                        o[4] = mv.copy;
                        o[5] = mv.zero;
                    }
                    ++nm;
                }
                ++nl;
            }
        }
        for (int k = i; k < j; ++k) {
            results[k] = rc;
            for (int t = 0; t < max_batch; ++t) {
                extents[((size_t)k * max_batch + t) * 2] = a.first[t];
                extents[((size_t)k * max_batch + t) * 2 + 1] = a.cap[t];
            }
        }
        i = j;
    }
    *n_moves = nm;
    ZL_CHECK_ARG(nm <= max_moves);
    return ZL_OK;
}
