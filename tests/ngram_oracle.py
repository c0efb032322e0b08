"""numpy restatement of the logits processors (include/zhilight_b200.h, zl_sample_processed), for the processor tests.

The n-gram levels restate calc_repetition_ngram (reference src/generator/beam_util.cu:318-350) over the task's tokens
most recent first (apply_beam_repetition_penalty, beam_util.cu:352-375, reads them with get_hypothesis_tokens(..., true));
the factor is powf(ngram_penalty, level + 1) * repetition_penalty applied as beam_repetition_penalty does
(beam_util.cu:212-219).  The bias follows the penalties (SearcherImplV1::pick_top_k, batch_generator.cpp:1764-1766, with
add_logit_bias at :1709-1728), then the pick is tests/sampling_oracle.py's.
"""
import numpy as np

from tests import sampling_oracle as so


def kmp_levels(r):
    """calc_repetition_ngram's ngrams[] for r (most recent first): KMP next[], then ngrams[i - L] = max(., L)."""
    n = len(r)
    if n == 0:
        return []
    nxt = [0] * n
    nxt[0] = -1
    for i in range(n - 1):
        p = nxt[i]
        while p >= 0:
            if r[p + 1] == r[i + 1]:
                break
            p = nxt[p]
        nxt[i + 1] = p + 1 if r[p + 1] == r[i + 1] else -1
    lev = [0] * n
    for i in range(n):
        L = nxt[i] + 1
        lev[i - L] = max(lev[i - L], L)
    return lev


def z_levels(r):
    """The parallel form k_ngram_levels computes: z the Z-function of r, R(s) = max(0, max over s' < s of
    s' + z[s'] - 1); lev[s-1] = z[s] where z[s] > 0 and s + z[s] - 1 > R(s), every other entry 0."""
    n = len(r)
    lev = [0] * n
    R = 0
    for s in range(1, n):
        z = 0
        while s + z < n and r[s + z] == r[z]:
            z += 1
        if z > 0 and s + z - 1 > R:
            lev[s - 1] = z
        R = max(R, s + z - 1)
    return lev


def ngram_factors(seq, ngram_penalty, repetition_penalty):
    """{token: f} for a task's sequence (oldest first): f = max over occurrences of
    powf(ngram_penalty, lev + 1) * repetition_penalty, in fp32."""
    r = list(seq)[::-1]
    lev = kmp_levels(r)
    ng, rp = np.float32(ngram_penalty), np.float32(repetition_penalty)
    out = {}
    for tok, l in zip(r, lev):
        f = np.float32(np.power(ng, np.float32(l + 1), dtype=np.float32) * rp)
        out[tok] = max(out.get(tok, np.float32(0)), f)
    return out


def process(logits, seq, repetition_penalty=1.0, presence_penalty=0.0, ngram_penalty=1.0, bias=None):
    """fp32 copy of one row with the task's penalties (n-gram rule when ngram_penalty > 1, else the bitmap rule over the
    sequence's distinct tokens) and then its bias {token: value}."""
    if ngram_penalty > 1:
        l = np.array(logits, dtype=np.float32, copy=True)
        for tok, f in ngram_factors(seq, ngram_penalty, repetition_penalty).items():
            v = l[tok]
            l[tok] = v * f if v < 0 else v / f
    else:
        l = so.penalise(logits, set(seq), repetition_penalty, presence_penalty)
    for tok, b in (bias or {}).items():
        l[tok] = np.float32(l[tok] + np.float32(b))
    return l


def pick(logits, seq, params, counter, ngram_penalty=1.0, bias=None):
    """-> (token, ambiguous) for one row: process, then sampling_oracle.pick with the row's u."""
    p = dict(dict(temperature=0.0, top_p=1.0, top_k=0, repetition_penalty=1.0, presence_penalty=0.0, seed=0), **params)
    l = process(logits, seq, p["repetition_penalty"], p["presence_penalty"], ngram_penalty, bias)
    u = float(so.uniform(p["seed"], int(counter)))
    return so.pick(l, p["temperature"], p["top_p"], p["top_k"], u)
