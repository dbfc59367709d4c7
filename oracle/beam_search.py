"""ORACLE (test infrastructure, not product code): CPU restatement of the reference's beam search, PaddleNLP
generation/utils.py (beam_search :1484-1649, BeamHypotheses / BeamSearchScorer :98-316, reorder_cache :1480-1482,
get_scale_by_dtype transformers/utils.py:91-112), with the choices the reference leaves open pinned down the way
b200mix_beam_search_step makes them:
  - step scores are log(exp(x - max) / sum) in fp32, then the repetition penalty, then + the beam score;
  - among equal scores the lower flat index (beam * V + token) ranks first; with diversity_rate > 0 the lower position
    in the row-major (beam, rank) list ranks first, and rank * diversity_rate is an fp32 product;
  - the scorer's arithmetic is Python double, as in the reference.
"""
from typing import Callable, Optional

import numpy as np

from .generation import repetition_penalty

BEAM_INIT, WORST_INIT = -1e6, 1e6
# The device's fp32 step scores differ from numpy's by a few ulps (expf / logf and the order of the row sum), about
# 1e-7 relative; two candidates closer than NEAR (relative) may be ranked either way. 1e-6 keeps a tenfold margin while
# flagging few items: with 2 * nb + 1 adjacent pairs per item (and per row with diversity_rate > 0), 1e-5 would flag
# tens of percent of the items at nb = 16 on N(0, 9) logits.
NEAR = 1e-6


def _close(a: float, b: float) -> bool:
    """Different but within NEAR (relative): fp32 rounding may swap them. Exact ties are ranked the same on both sides."""
    return a != b and abs(a - b) <= NEAR * max(abs(a), abs(b))


def beam_step_scores(logits: np.ndarray, beam_scores: np.ndarray, presence: Optional[np.ndarray], penalty=1.0):
    """:1561-1564 on fp32 [rows, V] logits: log(softmax) as log(exp(x - max) / sum), the penalty, + beam_scores [rows]."""
    x = logits.astype(np.float32)
    e = np.exp(x - x.max(-1, keepdims=True)).astype(np.float32)
    with np.errstate(divide="ignore"):
        s = np.log((e / e.sum(-1, keepdims=True, dtype=np.float32)).astype(np.float32)).astype(np.float32)
    if penalty != 1.0:
        s = repetition_penalty(s, presence, penalty)
    return (s + beam_scores.astype(np.float32)[:, None]).astype(np.float32)


def _top(values: np.ndarray, k: int):
    """Indices of the k + 1 largest of a 1-D fp32 array by (value desc, index asc) (k + 1 for the boundary check)."""
    n = min(k + 1, values.size)
    kth = np.partition(values, values.size - n)[values.size - n]
    cand = np.nonzero(values >= kth)[0]
    order = np.lexsort((cand, -values[cand]))
    return cand[order[:n]]


def _near_pairs(v: np.ndarray, n: int) -> np.ndarray:
    """near[i]: ranks i and i + 1 of the sorted values v lie within NEAR, for i < n."""
    return np.array([_close(float(v[i]), float(v[i + 1])) for i in range(min(n, len(v) - 1))], bool)


def beam_step(logits, beam_scores, presence, num_beams, penalty=1.0, diversity_rate=0.0, eos_token_id=None):
    """Selection of one step: (scores fp32 [B, 2nb], tokens [B, 2nb], beams [B, 2nb] (within the item), near bool [B]).
    near: two candidates whose order can change the result lie within NEAR of each other. process() consumes the
    first nb + (eos candidates among them) ranks, so those ranks and the one after them count; with diversity_rate > 0,
    so do the neighbours in their row's own ranking of every candidate the diversified list consumes."""
    s = beam_step_scores(logits, beam_scores, presence, penalty)
    rows, V = s.shape
    nb, K = num_beams, 2 * num_beams
    B = rows // nb
    scores = np.zeros((B, K), np.float32)
    tokens = np.zeros((B, K), np.int64)
    beams = np.zeros((B, K), np.int64)
    near = np.zeros(B, bool)
    def consumed(toks):  # ranks process() reads before its nb slots are full
        return min(K, nb + int(np.sum(toks[:K] == eos_token_id)) if eos_token_id is not None else nb)

    for b in range(B):
        if diversity_rate == 0.0:
            flat = s[b * nb:(b + 1) * nb].reshape(-1)
            idx = _top(flat, K)
            near[b] = _near_pairs(flat[idx], consumed(idx % V)).any()
            idx = idx[:K]
            scores[b], tokens[b], beams[b] = flat[idx], idx % V, idx // V
        else:
            sib_s = np.zeros((nb, K), np.float32)
            sib_t = np.zeros((nb, K), np.int64)
            row_near = np.zeros((nb, K + 1), bool)  # [j, r]: row j's ranks r and r + 1 are close
            for j in range(nb):
                idx = _top(s[b * nb + j], K)
                pairs = _near_pairs(s[b * nb + j][idx], K)
                row_near[j, :len(pairs)] = pairs
                sib_s[j], sib_t[j] = s[b * nb + j][idx[:K]], idx[:K]
            sibling = (np.arange(1, K + 1).astype(np.float32) * np.float32(diversity_rate)).astype(np.float32)
            div = (sib_s - sibling[None]).astype(np.float32).reshape(-1)
            pos = _top(div, K)
            n = consumed(sib_t.reshape(-1)[pos])
            near[b] = _near_pairs(div[pos], n).any()
            for p in pos[:n + 1]:
                j, r = divmod(int(p), K)
                near[b] |= row_near[j, r] or (r > 0 and row_near[j, r - 1])
            pos = pos[:K]
            scores[b], tokens[b], beams[b] = sib_s.reshape(-1)[pos], sib_t.reshape(-1)[pos], pos // K
    return scores, tokens, beams, near


class BeamHypotheses:
    """The n-best list of one item (the rules of BeamHypotheses :98-143), in Python double. `beams` holds (score, hyp)
    in insertion order, hyp being any payload (the token ids here); scores are normalised by ((n + 5) / 6) ** lp for
    n generated tokens. While the list has room every hypothesis enters and worst_score (1e6 while empty) is the running
    minimum. A full list takes a newcomer only when it beats worst_score; it then loses its lowest entry (lowest
    score, earliest position among equals) and worst_score becomes the score ranked next. `near` is set when such a
    comparison was within NEAR (relative)."""

    def __init__(self, num_beams, length_penalty, early_stopping):
        self.capacity, self.lp, self.stop_early = num_beams, length_penalty, early_stopping
        self.beams = []
        self.worst_score = WORST_INIT
        self.near = False

    def normalised(self, sum_logprobs, n_generated):
        return sum_logprobs / ((n_generated + 5) / 6) ** self.lp

    def add(self, hyp, sum_logprobs, n_generated):
        score = self.normalised(sum_logprobs, n_generated)
        if len(self.beams) < self.capacity:
            self.beams.append((score, hyp))
            self.worst_score = min(self.worst_score, score)
            return
        self.near |= _close(score, self.worst_score)
        if not score > self.worst_score:
            return
        self.beams.append((score, hyp))
        scores = np.array([b[0] for b in self.beams])
        rank = np.lexsort((np.arange(len(scores)), scores))  # ascending score, then position
        self.worst_score = float(scores[rank[1]])
        self.beams.pop(int(rank[0]))

    def is_done(self, best_sum_logprobs, n_generated):
        """Enough hypotheses, and early stopping or none of the running beams can still beat the worst one."""
        if len(self.beams) < self.capacity:
            return False
        if self.stop_early:
            return True
        bound = self.normalised(best_sum_logprobs, n_generated)
        self.near |= _close(self.worst_score, bound)
        return self.worst_score >= bound


def beam_process(hyps, done, input_ids, scores, tokens, beams, step, eos_token_id=None, pad_token_id=0):
    """BeamSearchScorer.process (:196-262) for candidates from beam_step. input_ids [B*nb, S + step]; done bool [B]
    (updated in place). Returns (next scores fp32 [B*nb], next tokens [B*nb], next global row indices [B*nb])."""
    B, K = scores.shape
    nb = K // 2
    ns = np.zeros(B * nb, np.float32)
    nt = np.zeros(B * nb, np.int64)
    ni = np.zeros(B * nb, np.int64)
    for b in range(B):
        if done[b]:
            ns[b * nb:(b + 1) * nb], nt[b * nb:(b + 1) * nb], ni[b * nb:(b + 1) * nb] = 0, pad_token_id, 0
            continue
        slot = 0
        for rank in range(K):
            tok, sc, row = int(tokens[b, rank]), scores[b, rank], b * nb + int(beams[b, rank])
            if eos_token_id is not None and tok == eos_token_id:
                if rank >= nb:
                    continue
                hyps[b].add(input_ids[row].copy(), float(sc), step)
            else:
                ns[b * nb + slot], nt[b * nb + slot], ni[b * nb + slot] = sc, tok, row
                slot += 1
            if slot == nb:
                break
        if hyps[b].is_done(float(scores[b].max()), step):
            done[b] = True
    return ns, nt, ni


def beam_finalize(hyps, done, input_ids, beam_scores, origin_len, max_length, num_return_sequences, pad_token_id,
                  eos_token_id):
    """BeamSearchScorer.finalize (:264-316) with input_ids [B*nb, cur_len] (prompt included). Returns (decoded int64
    [B * nrs, width] with the prompt, scores fp32 [B * nrs])."""
    B = len(hyps)
    nb = input_ids.shape[0] // B
    for b, h in enumerate(hyps):
        if done[b]:
            continue
        for j in range(nb):
            h.add(input_ids[b * nb + j].copy(), float(beam_scores[b * nb + j]), input_ids.shape[1] - origin_len)
    best = []
    for h in hyps:  # highest score first; among equal scores the later insertion first
        scores = np.array([b[0] for b in h.beams])
        for i in np.lexsort((-np.arange(len(scores)), -scores))[:num_return_sequences]:
            best.append((h.beams[i][1], h.beams[i][0]))
    lengths = [len(hyp) for hyp, _ in best]
    width = min(max(lengths) + 1, max_length)
    decoded = np.full((len(best), width), pad_token_id if min(lengths) != max(lengths) else 0, np.int64)
    for i, (hyp, _) in enumerate(best):
        decoded[i, :lengths[i]] = hyp
        if lengths[i] < max_length:
            decoded[i, lengths[i]] = eos_token_id
    return decoded, np.array([s for _, s in best], np.float32)


def beam_search(logits_fn: Callable, input_ids: np.ndarray, max_new_tokens: int, vocab_size: int, num_beams: int, *,
                penalty=1.0, diversity_rate=0.0, length_penalty=1.0, early_stopping=False, num_return_sequences=1,
                eos_token_id: Optional[int] = None, pad_token_id=0):
    """The beam_search loop (:1529-1649). logits_fn(step, tokens [B*nb] or None, rows [B*nb] or None) -> fp32 [B*nb, V]
    logits of the newest position, where tokens / rows are the previous step's choices and the global rows
    (index_select order) the caller reorders its cache by. Returns (decoded [B*nrs, width], scores fp32 [B*nrs],
    excused bool [B]: a selection or scorer comparison of the item was within NEAR, info dict)."""
    B, S = input_ids.shape
    nb = num_beams
    ids = np.repeat(input_ids, nb, 0)
    beam_scores = np.zeros((B, nb), np.float32)
    beam_scores[:, 1:] = BEAM_INIT
    beam_scores = beam_scores.reshape(-1)
    hyps = [BeamHypotheses(nb, length_penalty, early_stopping) for _ in range(B)]
    done = np.zeros(B, bool)
    excused = np.zeros(B, bool)
    tokens = rows = None
    steps = 0
    for step in range(max_new_tokens):
        logits = logits_fn(step, tokens, rows)
        presence = None
        if penalty != 1.0:
            presence = np.zeros((B * nb, vocab_size), bool)
            presence[np.arange(B * nb)[:, None], ids] = True
        sc, tk, bm, near = beam_step(logits, beam_scores, presence, nb, penalty, diversity_rate, eos_token_id)
        excused |= near & ~done
        beam_scores, tokens, rows = beam_process(hyps, done, ids, sc, tk, bm, step, eos_token_id, pad_token_id)
        ids = np.concatenate([ids[rows], tokens[:, None]], 1)
        steps += 1
        if done.all():
            break
    excused |= np.array([h.near for h in hyps])
    decoded, scores = beam_finalize(hyps, done, ids, beam_scores, S, S + max_new_tokens, num_return_sequences,
                                    pad_token_id, eos_token_id)
    excused |= np.array([h.near for h in hyps])
    return decoded, scores, excused, dict(done=done, hyps=hyps, steps=steps, ids=ids, beam_scores=beam_scores)
