"""numpy restatement of the sampling contract (include/zhilight_b200.h, zl_sample), for the sampling tests.

Philox4x32-10 and u, the penalties, the exact float64 probability of every token, and the inverse-CDF pick for a given
u with a flag for targets that fall within 1e-5 * P' of a cumulative boundary (where fp32 and float64 sums may
legitimately disagree).
"""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
MASK32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: 4 arrays of uint32 words, key: 2 arrays; -> 4 arrays (curand_philox4x32_x.h's round and key schedule)."""
    c = [np.asarray(w, dtype=np.uint64) & MASK32 for w in ctr]
    k0, k1 = [np.asarray(w, dtype=np.uint64) & MASK32 for w in key]
    for i in range(10):
        if i:
            k0 = (k0 + W0) & MASK32
            k1 = (k1 + W1) & MASK32
        p0 = M0 * c[0]
        p1 = M1 * c[2]
        c = [((p1 >> np.uint64(32)) ^ c[1] ^ k0) & MASK32, p1 & MASK32,
             ((p0 >> np.uint64(32)) ^ c[3] ^ k1) & MASK32, p0 & MASK32]
    return [w.astype(np.uint32) for w in c]


def uniform_r(seed, counter):
    """r = first Philox output word for key (seed lo, seed hi), counter (counter, 0, 0, 0); vectorised."""
    seed = np.asarray(seed, dtype=np.uint64)
    counter = np.asarray(counter, dtype=np.uint64)
    z = np.zeros(np.broadcast(seed, counter).shape, dtype=np.uint64)
    return philox4x32_10([counter + z, z, z, z], [seed & MASK32, seed >> np.uint64(32)])[0]


def uniform(seed, counter):
    """u = ((r >> 8) + 1) * 2^-24 in (0, 1]."""
    r = uniform_r(seed, counter).astype(np.uint64)
    return ((r >> np.uint64(8)) + np.uint64(1)).astype(np.float64) * 2.0 ** -24


def penalise(logits, history_tokens, repetition_penalty=1.0, presence_penalty=0.0):
    """fp32 copy of one row with the reference's penalty (beam_util.cu:212-219) on every distinct history token."""
    l = np.array(logits, dtype=np.float32, copy=True)
    toks = np.unique(np.asarray(list(history_tokens), dtype=np.int64))
    if toks.size == 0:
        return l
    v = l[toks]
    if presence_penalty != 0:
        v = v - np.float32(presence_penalty)
    else:
        rp = np.float32(repetition_penalty)
        v = np.where(v < 0, v * rp, v / rp).astype(np.float32)
    l[toks] = v
    return l


def greedy(l):
    """zl_argmax's pick: the maximum, ties to the lowest index; NaN never wins."""
    l = np.where(np.isnan(l), -np.inf, l).astype(np.float32)
    return int(np.argmax(l))


def is_greedy(temperature, top_k):
    return not temperature > 0 or top_k == 1


def _order(l, temperature):
    x = (np.asarray(l, dtype=np.float32) / np.float32(temperature)).astype(np.float32)
    x = np.where(np.isnan(x), np.float32(-np.inf), x)
    idx = np.arange(x.size)
    order = np.lexsort((idx, -x))   # descending x, ties by ascending index
    return x, order


def _cumulative(l, temperature, top_p, top_k):
    """-> (order, C (float64 inclusive cumulative weights in that order), P') or None for a greedy fallback row."""
    x, order = _order(l, temperature)
    xmax = x[order[0]]
    if not np.isfinite(xmax):
        return None
    w = np.exp(x[order].astype(np.float64) - np.float64(xmax))
    C = np.cumsum(w)
    Z = C[-1]
    P = top_p * Z
    if 0 < top_k < x.size:
        P = min(P, C[top_k - 1])
    return order, C, P


def probs(l, temperature, top_p=1.0, top_k=0):
    """Exact float64 probability of each token of an (already penalised) fp32 row."""
    V = len(l)
    p = np.zeros(V, dtype=np.float64)
    if is_greedy(temperature, top_k):
        p[greedy(l)] = 1.0
        return p
    cum = _cumulative(l, temperature, top_p, top_k)
    if cum is None:
        p[greedy(l)] = 1.0
        return p
    order, C, P = cum
    hi = np.minimum(C, P)
    lo = np.concatenate([[0.0], hi[:-1]])
    p[order] = (hi - lo) / P
    return p


def pick(l, temperature, top_p, top_k, u, margin=1e-5):
    """-> (token, ambiguous): the first j in order with C_j >= u * P', and whether u * P' lies within margin * P' of a
    cumulative boundary."""
    if is_greedy(temperature, top_k):
        return greedy(l), False
    cum = _cumulative(l, temperature, top_p, top_k)
    if cum is None:
        return greedy(l), False
    order, C, P = cum
    target = u * P
    j = int(np.searchsorted(C, target, side="left"))
    j = min(j, len(C) - 1)
    near = abs(C[j] - target) <= margin * P or (j > 0 and abs(target - C[j - 1]) <= margin * P)
    return int(order[j]), bool(near)


def reference_binary_search(l, temperature, top_p, top_k, u):
    """random_util.cu:81-106 on float64 softmax probabilities: probs_cum normalised, top_p clipped by probs_cum[k-1],
    v_p = u * top_p * probs_cum[-1], then the binary search for the first probs_cum[idx] >= v_p (vectorised over u)."""
    x, order = _order(l, temperature)
    w = np.exp(x[order].astype(np.float64) - np.float64(x[order[0]]))
    cum = np.cumsum(w / w.sum())
    tp = top_p
    if 0 < top_k < len(cum):   # the reference asserts top_k < V; the contract treats top_k >= V as off
        tp = min(cum[top_k - 1], tp)
    v_p = np.asarray(u, dtype=np.float64) * tp * cum[-1]
    lf = np.full(v_p.shape, -1)
    rt = np.full(v_p.shape, len(cum) - 1)
    while np.any(lf + 1 < rt):
        go = lf + 1 < rt
        mid = (lf + rt) // 2
        below = cum[np.maximum(mid, 0)] < v_p
        lf = np.where(go & below, mid, lf)
        rt = np.where(go & ~below, mid, rt)
    return order[rt]


def history_bitmap(token_lists, V):
    """(tasks, ceil(V/32)) int32 bitmap with the given tokens set."""
    words = (V + 31) // 32
    h = np.zeros((len(token_lists), words), dtype=np.uint32)
    for t, toks in enumerate(token_lists):
        for tok in toks:
            h[t, tok >> 5] |= np.uint32(1) << np.uint32(tok & 31)
    return h.view(np.int32)


def bitmap_tokens(row, V):
    row = np.asarray(row).view(np.uint32)
    bits = np.unpackbits(row.view(np.uint8), bitorder="little")[:V]
    return set(np.nonzero(bits)[0].tolist())
