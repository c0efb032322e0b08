"""Token automata for constrained decoding (zl_llama_set_constraint in include/zhilight_b200.h).

An automaton over a vocabulary of V tokens has S >= 1 states.  State s allows the tokens of a bitmask A(s): ceil(V/32)
uint32 words, bit j of word i = token 32 i + j, non-empty, with no bit at or past V.  Its edges are (token, next) pairs
with distinct tokens of A(s) in ascending order, kept as CSR arrays (row_ptr, edge_tok, edge_next).  Picking token x in
state s moves to the next state of x's edge, or to default_next[s] when x has none.  The decoder masks each pick of a
constrained task with its state's set and moves the state on the device.

Two builders cover the common requests: `allowed` (a fixed set of tokens, one state) and `choices` (answer with one of
these token sequences).  Compiling regular expressions, JSON schemas or grammars needs a tokenizer's strings and stays
with host grammar engines, which drive the decoder with a one-state `allowed` mask per step.
"""
import numpy as np


def mask_words(vocab_size):
    return (int(vocab_size) + 31) // 32


def token_bitmask(tokens, vocab_size):
    """(ceil(V/32),) uint32 bitmask of the given token ids (each in [0, V))."""
    t = np.asarray(list(tokens) if not isinstance(tokens, np.ndarray) else tokens, dtype=np.int64).reshape(-1)
    if t.size and (t.min() < 0 or t.max() >= vocab_size):
        raise ValueError("token ids must lie in [0, %d)" % vocab_size)
    m = np.zeros(mask_words(vocab_size), np.uint32)
    np.bitwise_or.at(m, t >> 5, (np.uint32(1) << (t & 31).astype(np.uint32)))
    return m


def bitmask_tokens(mask):
    """the ascending token ids set in a uint32 bitmask"""
    bits = np.unpackbits(np.asarray(mask, np.uint32).view(np.uint8), bitorder="little")
    return np.flatnonzero(bits)


class TokenAutomaton:
    """A validated token automaton: masks (S, ceil(V/32)) uint32, row_ptr (S + 1), edge_tok / edge_next (E) and
    default_next (S) int32, and the start state.  The constructor refuses a malformed automaton with ValueError, with
    the same rules as zl_token_automaton_check."""

    def __init__(self, vocab_size, masks, row_ptr, edge_tok, edge_next, default_next, start=0):
        self.vocab_size = int(vocab_size)
        self.masks = np.ascontiguousarray(masks, dtype=np.uint32)
        self.row_ptr = np.ascontiguousarray(row_ptr, dtype=np.int32).reshape(-1)
        self.edge_tok = np.ascontiguousarray(edge_tok, dtype=np.int32).reshape(-1)
        self.edge_next = np.ascontiguousarray(edge_next, dtype=np.int32).reshape(-1)
        self.default_next = np.ascontiguousarray(default_next, dtype=np.int32).reshape(-1)
        self.start = int(start)
        self._validate()

    @property
    def n_states(self):
        return self.masks.shape[0]

    @property
    def n_edges(self):
        return self.edge_tok.size

    def _validate(self):
        V, W = self.vocab_size, mask_words(self.vocab_size)
        if V <= 0:
            raise ValueError("vocab_size must be positive")
        if self.masks.ndim != 2 or self.masks.shape[0] < 1 or self.masks.shape[1] != W:
            raise ValueError("masks must have shape (n_states >= 1, %d)" % W)
        S, E = self.masks.shape[0], self.edge_tok.size
        if self.row_ptr.size != S + 1 or self.default_next.size != S or self.edge_next.size != E:
            raise ValueError("row_ptr needs n_states + 1 entries, default_next n_states, edge_next one per edge")
        if not 0 <= self.start < S:
            raise ValueError("start state out of range")
        if self.row_ptr[0] != 0 or self.row_ptr[-1] != E or np.any(np.diff(self.row_ptr) < 0):
            raise ValueError("row_ptr must start at 0, never decrease and end at the number of edges")
        if not self.masks.any(axis=1).all():
            raise ValueError("every state must allow at least one token")
        if V % 32 and np.any(self.masks[:, -1] >> np.uint32(V % 32)):
            raise ValueError("a mask has bits at or past vocab_size")
        for arr, what in ((self.default_next, "default_next"), (self.edge_next, "edge_next")):
            if arr.size and (arr.min() < 0 or arr.max() >= S):
                raise ValueError(what + " names a state out of range")
        for s in range(S):
            t = self.edge_tok[self.row_ptr[s]:self.row_ptr[s + 1]].astype(np.int64)
            if t.size == 0:
                continue
            if t.min() < 0 or t.max() >= V:
                raise ValueError("edge token out of range")
            if np.any(np.diff(t) <= 0):
                raise ValueError("a state's edge tokens must be distinct and ascending")
            if not np.all((self.masks[s, t >> 5] >> (t & 31).astype(np.uint32)) & 1):
                raise ValueError("an edge token is outside its state's allowed set")

    def allowed_tokens(self, state):
        return bitmask_tokens(self.masks[state])

    def next_state(self, state, token):
        """the state after picking `token` in `state`"""
        a, b = self.row_ptr[state], self.row_ptr[state + 1]
        k = a + int(np.searchsorted(self.edge_tok[a:b], token))
        return int(self.edge_next[k]) if k < b and self.edge_tok[k] == token else int(self.default_next[state])


def allowed(tokens=None, vocab_size=None, bitmask=None):
    """A one-state automaton that allows the same tokens at every step: the given token ids, or (bitmask=) a
    (ceil(V/32),) uint32 bitmask as a grammar engine emits it.  Exactly one of the two is given."""
    if vocab_size is None or (tokens is None) == (bitmask is None):
        raise ValueError("allowed() takes vocab_size and exactly one of tokens and bitmask")
    if bitmask is not None:
        m = np.asarray(bitmask)
        if m.dtype != np.uint32 or m.shape != (mask_words(vocab_size),):
            raise ValueError("bitmask must be a (%d,) uint32 array" % mask_words(vocab_size))
    else:
        m = token_bitmask(np.asarray(tokens).reshape(-1), vocab_size)
    return TokenAutomaton(vocab_size, m[None, :], [0, 0], [], [], [0], 0)


def choices(token_seqs, end_ids, vocab_size):
    """An automaton that emits exactly one of `token_seqs` (non-empty token id sequences), then one of `end_ids`.

    The states are the nodes of the sequences' token trie (the root is the start) and one final state.  A node allows
    the tokens of its children; a node where a choice is complete also allows `end_ids`, which lead to the final state,
    so a choice that is a prefix of another may either end or go on.  The final state allows `end_ids` and stays."""
    ends = sorted({int(e) for e in end_ids})
    if not ends:
        raise ValueError("choices needs at least one end id")
    seqs = [tuple(int(t) for t in s) for s in token_seqs]
    if not seqs or any(len(s) == 0 for s in seqs):
        raise ValueError("choices needs at least one non-empty token sequence")
    for t in ends + [t for s in seqs for t in s]:
        if not 0 <= t < vocab_size:
            raise ValueError("token ids must lie in [0, %d)" % vocab_size)
    if set(ends) & {t for s in seqs for t in s}:
        raise ValueError("an end id may not occur inside a choice")
    children, complete = [{}], [False]   # node 0: the root
    for s in seqs:
        node = 0
        for t in s:
            if t not in children[node]:
                children[node][t] = len(children)
                children.append({})
                complete.append(False)
            node = children[node][t]
        complete[node] = True
    final = len(children)
    masks, row_ptr, edge_tok, edge_next = [], [0], [], []
    for node, ch in enumerate(children):
        toks = sorted(ch)
        masks.append(token_bitmask(toks + (ends if complete[node] else []), vocab_size))
        edge_tok += toks
        edge_next += [ch[t] for t in toks]
        row_ptr.append(len(edge_tok))
    masks.append(token_bitmask(ends, vocab_size))
    row_ptr.append(len(edge_tok))
    return TokenAutomaton(vocab_size, np.stack(masks), row_ptr, edge_tok, edge_next, [final] * (final + 1), 0)
