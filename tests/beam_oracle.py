"""numpy restatement of the reference's beam search: SearcherImplV1::pick_top_k (src/generator/batch_generator.cpp:1762-1852),
its early stop (:1564-1574) and BeamSearchResultManager (src/generator/beam_result_manager.hpp:94-125), written over plain
hypothesis lists -- no task slots, no KV copies -- as the yardstick of zhilight_b200/beam_search.py."""
import numpy as np


class ResultManager:
    def __init__(self, n):
        self.n, self.tokens, self.scores, self.cums = n, [], [], []
        self.min_score = np.float32(1e10)

    def accept(self, score):
        return len(self.scores) < self.n or score >= self.min_score

    def add(self, tokens, cum, score):
        if len(self.scores) < self.n:
            self.tokens.append(tokens)
            self.scores.append(score)
            self.cums.append(cum)
            self.min_score = min(self.min_score, score)
            return
        if score < self.min_score:
            return
        i = int(np.argmin(self.scores))   # the first minimum
        if score > self.scores[i]:
            self.tokens[i], self.scores[i], self.cums[i] = tokens, score, cum
        self.min_score = min(self.scores)

    def best(self):
        order = sorted(range(len(self.scores)), key=lambda i: (-self.scores[i], i))
        return [(list(self.tokens[i]), float(self.scores[i]), float(self.cums[i])) for i in order]


def pick(cands, gens, t, width, max_new, eos, mgr):
    """cands: [(parent, token, cum)] best first (parent -1: none); gens[parent]: its generated tokens.
    -> the live [(parent, token, cum)] after the pick and the early stop"""
    live = []
    for parent, tok, cum in cands:
        if parent < 0:
            break
        cum = np.float32(cum)
        score = cum / np.float32(t + 1)
        last = t + 1 == max_new
        if tok == eos or last:
            if mgr.accept(score):
                mgr.add(list(gens[parent]) + ([] if tok == eos else [int(tok)]), cum, score)
        else:
            live.append((int(parent), int(tok), cum))
        if len(live) >= width:
            break
    if live and not mgr.accept(live[0][2] / np.float32(t + 1)):
        live = []
    return live


def log_softmax_f32(x):
    """beam_util.cu:30-45 in fp32: x - max - log(1e-20 + sum exp(x - max))"""
    x = np.asarray(x, np.float32)
    m = x.max()
    return (x - m) - np.float32(np.log(np.float32(1e-20) + np.exp(x - m).sum(dtype=np.float32)))


def topk(rows, cums, k):
    """flat top-k of cum[i] + logp[i][v] over live rows: (score desc, i * V + v asc) -> [(i, v, score)], padded with
    (-1, -1, -inf)"""
    scores, keys = [], []
    for i, (lp, c) in enumerate(zip(rows, cums)):
        if not c > -np.inf:
            continue
        s = (lp + np.float32(c)).astype(np.float32)
        ok = np.isfinite(s)
        scores.append(s[ok])
        keys.append(i * len(lp) + np.nonzero(ok)[0])
    if not scores:
        return [(-1, -1, -np.inf)] * k
    s, key = np.concatenate(scores), np.concatenate(keys)
    order = np.lexsort((key, -s.astype(np.float64)))[:k]
    V = len(rows[0])
    out = [(int(key[j] // V), int(key[j] % V), np.float32(s[j])) for j in order]
    return out + [(-1, -1, -np.inf)] * (k - len(out))


def search(logits_fn, prompts, width, max_new, eos, num_results):
    """Beam search of each prompt on its own: logits_fn(tokens) -> the next-token logits after `tokens`."""
    k = min(2 * width, 32)
    out = []
    for prompt in prompts:
        prompt = [int(x) for x in prompt]
        hyps = [([], np.float32(0))]   # (generated tokens, cum)
        mgr = ResultManager(num_results)
        for t in range(max_new):
            rows = [log_softmax_f32(logits_fn(prompt + g)) for g, _ in hyps]
            cands = topk(rows, [c for _, c in hyps], k)
            live = pick(cands, [g for g, _ in hyps], t, width, max_new, eos, mgr)
            if not live:
                break
            hyps = [(hyps[p][0] + [v], c) for p, v, c in live]
        out.append(mgr.best())
    return out


def replay(trace, prompts, width, max_new, eos, num_results):
    """Replays the per-step candidates a search recorded (beam_search's trace) through pick(): -> (results, beams per
    step and group) to compare with the search's own"""
    mgrs = [ResultManager(num_results) for _ in prompts]
    done = [False] * len(prompts)
    beams = []
    for rec in trace:
        t, step = rec["t"], []
        for g, prompt in enumerate(prompts):
            rows = rec["slots"][g * width:(g + 1) * width]
            gens = [None if r is None else r[len(prompt):] for r in rows]
            cands = list(zip(rec["parent"][g], rec["token"][g], rec["score"][g]))
            live = [] if done[g] else pick(cands, gens, t, width, max_new, eos, mgrs[g])
            done[g] = done[g] or not live
            step.append([(list(rows[p]) + [v], float(c)) for p, v, c in live])
        beams.append(step)
    return [m.best() for m in mgrs], beams
