"""Beam search over the decode driver's beam steps: the host policy and the slot planner.

The policy is the reference's SearcherImplV1::pick_top_k (src/generator/batch_generator.cpp:1762-1852) with its early
stop (:1564-1574) and BeamSearchResultManager (src/generator/beam_result_manager.hpp:94-125).  The selection itself runs
on the GPU (zl_beam_topk inside zl_llama_beam_step).

Each beam owns a task slot: group g (one prompt) uses slots [g W, (g + 1) W).  Where the reference keeps one tree buffer
per task and attends with an ancestor mask, a fork here copies the KV rows in which two slots' token histories differ
(zl_llama_kv_copy_rows), and every attention route stays as it is.
"""
import numpy as np

MAX_WIDTH = 16   # zl_beam_topk's largest group
MAX_K = 32


class BeamResults:
    """BeamSearchResultManager (beam_result_manager.hpp:94-125): at most num_results finished hypotheses; once full, a
    result must score at least the current minimum and replaces the first result holding it if it scores more."""

    def __init__(self, num_results):
        self.num_results = num_results
        self.items = []                   # [tokens, score, cum_logprob]
        self.min_score = np.float32(1e10)

    def full(self):
        return len(self.items) >= self.num_results

    def accept_score(self, score):
        return not self.full() or score >= self.min_score

    def add_result(self, tokens, cum, score):
        if not self.full():
            self.items.append([tokens, score, cum])
            if score < self.min_score:
                self.min_score = score
            return
        if score < self.min_score:
            return
        i = min(range(len(self.items)), key=lambda j: (self.items[j][1], j))   # get_min_score_idx: the first minimum
        if score > self.items[i][1]:
            self.items[i] = [tokens, score, cum]
        self.min_score = min(it[1] for it in self.items)

    def best(self):
        """(tokens, score, cum_logprob) tuples, best score first"""
        return [(list(t), float(s), float(c)) for t, s, c in sorted(self.items, key=lambda it: -it[1])]


def select(parent, token, cum, t, width, max_new_tokens, eos_id, results, gen):
    """One group's pick_top_k (batch_generator.cpp:1799-1850) over its candidates, best first: parent[k] (-1: none), token[k]
    and cum[k] the cumulative log-probability.  gen[j] are the generated tokens of the beam in the group's row j.  A
    candidate whose token is EOS, or any candidate at the last step, is offered to `results` with score cum / (t + 1) (the
    EOS itself is not kept); any other becomes a live beam, until `width` are live.  Returns the live (parent, token, cum),
    or none when the best of them is not accepted (the early stop, batch_generator.cpp:1564-1574)."""
    live = []
    for p, v, c in zip(parent, token, cum):
        if p < 0:
            break
        c = np.float32(c)
        score = c / np.float32(t + 1)
        if v == eos_id or t + 1 == max_new_tokens:
            if results.accept_score(score):
                results.add_result(gen[p] + ([] if v == eos_id else [int(v)]), c, score)
        else:
            live.append((int(p), int(v), c))
        if len(live) >= width:
            break
    if live and not results.accept_score(live[0][2] / np.float32(t + 1)):
        return []
    return live


def lcp(a, b):
    n = min(len(a), len(b))
    i = 0
    while i < n and a[i] == b[i]:
        i += 1
    return i


def plan_slots(parents, kv):
    """Slots for the children of one group.  parents[c]: the row (slot within the group) of child c's parent; kv[j]: the
    tokens whose KV rows slot j holds.  A parent's first child keeps the parent's slot; every other child takes the next
    slot, in ascending order, whose beam left no child, and needs the rows [lcp(kv[parent], kv[slot]), len(kv[parent]))
    copied from its parent.  So no destination is a source and one copy launch per step is race-free.
    Returns (slot of each child, [(src, dst, row0, row1), ...])."""
    with_child = set(parents)
    free = [j for j in range(len(kv)) if j not in with_child]
    kept, slots, copies = set(), [], []
    for p in parents:
        if p not in kept:
            kept.add(p)
            slots.append(p)
            continue
        d = free.pop(0)
        slots.append(d)
        row0 = lcp(kv[p], kv[d])
        if row0 < len(kv[p]):
            copies.append((p, d, row0, len(kv[p])))
    return slots, copies


def beam_search(step, copy_rows, prefill, prompts, beam_width, max_new_tokens, eos_id, num_results=1, trace=None):
    """The search loop over a driver's entry points:
      step(tokens, positions, groups, cum, K) -> (parent, token, score), each (G, K)   -- zl_llama_beam_step
      copy_rows(ranges (n, 4) {src, dst, row0, row1})                                 -- zl_llama_kv_copy_rows
      prefill(slot, tokens)                                                           -- zl_llama_prefill at pos0 0
    Returns, per prompt, up to num_results (tokens, score, cum_logprob) best first.  trace: a list that gets one dict per
    step (inputs, candidates and the beams after the pick)."""
    W, G = int(beam_width), len(prompts)
    if not 1 <= W <= MAX_WIDTH:
        raise ValueError("beam_width must be 1 .. %d, not %d" % (MAX_WIDTH, W))
    if max_new_tokens < 1 or num_results < 1 or G < 1:
        raise ValueError("need at least one prompt, max_new_tokens >= 1 and num_results >= 1")
    B, K = G * W, min(2 * W, MAX_K)   # batch_generator.cpp:1771
    groups = np.array([[g * W, W] for g in range(G)], dtype=np.int32)
    kv = [[] for _ in range(B)]       # tokens whose KV rows each slot holds
    seq = [None] * B                  # a live slot's prompt + generated tokens; the last one is the next input
    gen = [None] * B                  # ... and its generated tokens alone
    cum = np.full(B, -np.inf, dtype=np.float32)
    results = [BeamResults(num_results) for _ in range(G)]
    done = [False] * G
    for g, p in enumerate(prompts):
        p = [int(x) for x in p]
        if not p:
            raise ValueError("prompt %d is empty" % g)
        s = g * W
        if len(p) > 1:
            prefill(s, p[:-1])
        kv[s], seq[s], gen[s], cum[s] = p[:-1], p, [], 0.0
    for t in range(max_new_tokens):
        # a dead slot steps at the row after its history, which no history holds, with token 0
        tokens = np.array([seq[s][-1] if seq[s] else 0 for s in range(B)], dtype=np.int32)
        positions = np.array([len(kv[s]) for s in range(B)], dtype=np.int32)
        parent, token, score = step(tokens, positions, groups, cum, K)
        for s in range(B):
            if seq[s] is not None:
                kv[s] = seq[s]
        rec = dict(t=t, tokens=tokens, positions=positions, cum=cum.copy(), parent=parent, token=token, score=score,
                   slots=[None if seq[s] is None else list(seq[s]) for s in range(B)], beams=[])
        ranges = []
        n_seq, n_gen = [None] * B, [None] * B
        n_cum = np.full(B, -np.inf, dtype=np.float32)
        for g in range(G):
            live = [] if done[g] else select(parent[g], token[g], score[g], t, W, max_new_tokens, eos_id, results[g],
                                              gen[g * W:(g + 1) * W])
            rec["beams"].append([(list(seq[g * W + p]) + [v], float(c)) for p, v, c in live])
            if not live:
                done[g] = True
                continue
            slots, copies = plan_slots([p for p, _, _ in live], kv[g * W:(g + 1) * W])
            for (p, v, c), d in zip(live, slots):
                s, ps = g * W + d, g * W + p
                n_seq[s], n_gen[s], n_cum[s] = seq[ps] + [v], gen[ps] + [v], c
            for p, d, r0, r1 in copies:
                ranges.append((g * W + p, g * W + d, r0, r1))
                kv[g * W + d] = list(kv[g * W + p])
        if trace is not None:
            rec["ranges"] = list(ranges)
            trace.append(rec)
        seq, gen, cum = n_seq, n_gen, n_cum
        if ranges:
            copy_rows(np.array(ranges, dtype=np.int32))
        if all(done):
            break
    return [r.best() for r in results]
