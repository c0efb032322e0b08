"""numpy restatement of the masked pick (include/zhilight_b200.h, zl_sample_masked) on top of tests/ngram_oracle.py.

The row is processed as zl_sample_processed processes it, then only the allowed tokens remain: the pick is
sampling_oracle.pick over the sub-row of allowed tokens (so top-k counts allowed tokens only, and masked tokens get no
mass), with an allowed NaN counted as -inf, mapped back to its token id.  A sub-row whose tokens are all -inf takes its
first entry: the smallest allowed token.
"""
import numpy as np

from tests import ngram_oracle as ng
from tests import sampling_oracle as so


def masked_pick(logits, allowed, seq=(), params=None, counter=0, ngram_penalty=1.0, bias=None):
    """-> (token, ambiguous) for one row; allowed: the allowed token ids (non-empty; bitmask_tokens of a mask)."""
    toks = np.unique(np.asarray(allowed, dtype=np.int64))
    p = dict(dict(temperature=0.0, top_p=1.0, top_k=0, repetition_penalty=1.0, presence_penalty=0.0, seed=0),
             **(params or {}))
    raw = np.asarray(logits, np.float32)
    raw = np.where(np.isnan(raw), np.float32(-np.inf), raw)
    with np.errstate(over="ignore", invalid="ignore"):
        l = ng.process(raw, list(seq), p["repetition_penalty"], p["presence_penalty"], ngram_penalty, bias)
    sub = l[toks]
    u = float(so.uniform(p["seed"], int(counter)))
    j, amb = so.pick(sub, p["temperature"], p["top_p"], p["top_k"], u)
    return int(toks[j]), amb


def run_automaton(automaton, tokens):
    """the states an automaton passes through on a token sequence, start first"""
    s = [automaton.start]
    for t in tokens:
        s.append(automaton.next_state(s[-1], int(t)))
    return s
