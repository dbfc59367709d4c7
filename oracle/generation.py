"""ORACLE (test infrastructure, not product code): CPU restatement of the reference's decoding loop, PaddleNLP
generation/utils.py (greedy_search :1028-1127, sample :1129-1271, get_unfinished_flag :67-95) and
generation/logits_process.py (RepetitionPenaltyLogitsProcessor :89-110, TopKProcess :293-305, TopPProcess :308-341),
with the choices the reference leaves open pinned down the way b200mix_sample_tokens makes them:
  - probabilities are fp32 softmax(l / T) = exp(x - max) / sum (IEEE fp32 division);
  - top-p ranks equal probabilities by ascending token id (the reference's argsort order is unspecified);
  - masses are added as floor(p * 2^48) integers (exact for p >= 2^-25), so a sum does not depend on its order;
  - paddle.multinomial is replaced by one Philox4x32-10 draw per (seed, step, row): counter = (step, row, 0, 0),
    key = the 64-bit seed, u = (x0 >> 8) * 2^-24, and the token is the first kept id (ascending id order) whose
    inclusive prefix mass exceeds u * kept mass.
"""
from typing import Callable, List, Optional

import numpy as np

FX = 2.0 ** 48
_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """Random123 philox4x32-10. ctr: 4 words, key: 2 words (ints or equal-shape integer arrays). Returns 4 uint64
    arrays holding the 32-bit output words."""
    c = [np.asarray(x, dtype=np.uint64) & _M32 for x in ctr]
    k0, k1 = (np.asarray(x, dtype=np.uint64) & _M32 for x in key)
    for r in range(10):
        if r:
            k0 = (k0 + np.uint64(0x9E3779B9)) & _M32
            k1 = (k1 + np.uint64(0xBB67AE85)) & _M32
        p0 = c[0] * np.uint64(0xD2511F53)
        p1 = c[2] * np.uint64(0xCD9E8D57)
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _M32]
    return c


def uniform(seed: int, step: int, rows) -> np.ndarray:
    """u in [0, 1) (24 bits) for each row index of `rows` at `step`: float64 array."""
    rows = np.asarray(rows, dtype=np.uint64)
    x0 = philox4x32_10((np.full_like(rows, step), rows, 0, 0), (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF))[0]
    return (x0 >> np.uint64(8)).astype(np.float64) * 2.0 ** -24


def repetition_penalty(logits: np.ndarray, presence: np.ndarray, penalty: float) -> np.ndarray:
    """:104-110 on fp32 [B, V] logits; presence bool [B, V] = ids seen so far (every id of the prompt included)."""
    p = np.float32(penalty)
    pen = np.where(logits < 0, logits * p, logits / p).astype(np.float32)
    return np.where(presence, pen, logits)


def softmax_t(logits: np.ndarray, temperature: float) -> np.ndarray:
    x = (logits / np.float32(temperature)).astype(np.float32)
    e = np.exp(x - x.max(-1, keepdims=True)).astype(np.float32)
    return (e / e.sum(-1, keepdims=True, dtype=np.float32)).astype(np.float32)


def top_k_process(probs: np.ndarray, top_k: int) -> np.ndarray:
    """TopKProcess: keep p >= the k-th largest p (ties at that value all kept); top_k = 0 disables it."""
    if top_k == 0:
        return probs
    k = min(max(top_k, 1), probs.shape[-1])
    kth = -np.sort(-probs, axis=-1)[..., k - 1:k]
    return np.where(probs >= kth, probs, np.float32(0)).astype(np.float32)


def fixed_point(probs: np.ndarray) -> np.ndarray:
    return np.floor(probs.astype(np.float64) * FX).astype(np.int64)


def top_p_keep(probs: np.ndarray, top_p: float) -> np.ndarray:
    """TopPProcess as a keep mask over [B, V] (applied to the top-k output as it is, not renormalised): ids sorted by
    descending p, lower id first among equals; an id is dropped when the mass ranked above it exceeds top_p."""
    if top_p >= 1.0:
        return np.ones(probs.shape, dtype=bool)
    tp = np.floor(np.float64(np.float32(top_p)) * FX)
    keep = np.zeros(probs.shape, dtype=bool)
    for b in range(probs.shape[0]):
        order = np.lexsort((np.arange(probs.shape[1]), -probs[b]))
        w = fixed_point(probs[b][order])
        excl = np.cumsum(w) - w
        keep[b, order] = excl <= tp
    return keep


def draw_row(probs: np.ndarray, keep: np.ndarray, u: np.ndarray):
    """Inverse-CDF choice over the kept, unnormalised mass of ONE row (probs, keep [V]) for each u of `u` [n].
    Returns (tokens int64 [n], near-boundary bool [n]: the target lies within 1e-5, relative to the kept mass, of a
    prefix boundary)."""
    cum = np.cumsum(np.where(keep, fixed_point(probs), 0))
    K = np.float64(cum[-1])
    target = np.asarray(u, dtype=np.float64) * K
    cumf = cum.astype(np.float64)
    tok = np.searchsorted(cumf, target, side="right")
    lo = np.where(tok > 0, cumf[np.maximum(tok - 1, 0)], -np.inf)
    near = np.minimum(cumf[tok] - target, target - lo) <= 1e-5 * K
    return tok.astype(np.int64), near


def draw(probs: np.ndarray, keep: np.ndarray, u: np.ndarray):
    """draw_row for each row of probs / keep [B, V] with its own u [B]."""
    res = [draw_row(probs[b], keep[b], u[b:b + 1]) for b in range(len(u))]
    return np.concatenate([r[0] for r in res]), np.concatenate([r[1] for r in res])


def top_p_near_boundary(probs: np.ndarray, top_p: float) -> np.ndarray:
    """Rows whose top-p cut lies within 1e-5 (relative) of top_p: rounding may move it by one id there."""
    if top_p >= 1.0:
        return np.zeros(probs.shape[0], dtype=bool)
    tp = np.float64(np.float32(top_p)) * FX
    near = np.zeros(probs.shape[0], dtype=bool)
    for b in range(probs.shape[0]):
        w = fixed_point(-np.sort(-probs[b]))
        excl = (np.cumsum(w) - w).astype(np.float64)
        near[b] = bool((np.abs(excl[1:] - tp) <= 1e-5 * tp).any())
    return near


def next_tokens(logits: np.ndarray, presence: np.ndarray, *, do_sample: bool, temperature=1.0, top_k=0, top_p=1.0,
                penalty=1.0, seed=0, step=0, rows=None):
    """One step over fp32 [B, V] logits -> (tokens int64 [B], excused bool [B]). Greedy: argmax of the penalised
    logits (lowest id on ties). Sampling: temperature, softmax, top-k, top-p, Philox inverse-CDF draw."""
    l = repetition_penalty(logits.astype(np.float32), presence, penalty) if penalty != 1.0 else logits.astype(np.float32)
    if not do_sample:
        return l.argmax(-1).astype(np.int64), np.zeros(l.shape[0], dtype=bool)
    probs = top_k_process(softmax_t(l, temperature), top_k)
    keep = top_p_keep(probs, top_p)
    u = uniform(seed, step, np.arange(l.shape[0]) if rows is None else rows)
    tok, near = draw(probs, keep, u)
    return tok, near | top_p_near_boundary(probs, top_p)


def get_unfinished_flag(last_tokens: np.ndarray, unfinished: np.ndarray, eos_token_id: List[int]) -> np.ndarray:
    """:67-95 for an int or a flat list of ids: a row stays unfinished unless its newest token is any of them."""
    return unfinished & ~np.isin(last_tokens, np.asarray(eos_token_id, dtype=np.int64))


def generate(logits_fn: Callable[[int, np.ndarray], np.ndarray], input_ids: np.ndarray, max_new_tokens: int, vocab_size: int,
             *, do_sample=False, temperature=1.0, top_k=0, top_p=1.0, penalty=1.0, eos_token_id: Optional[List[int]] = None,
             pad_token_id=0, seed=0):
    """greedy_search / sample: logits_fn(step, newest tokens or None) -> fp32 [B, V] logits of the newest position.
    Finished rows emit pad_token_id (:1239-1240) and the loop stops once every row has finished (:1253-1256).
    Returns (ids [B, S + n], presence bool [B, V] after the loop, finished bool [B], excused bool [B])."""
    B = input_ids.shape[0]
    presence = np.zeros((B, vocab_size), dtype=bool)
    presence[np.arange(B)[:, None], input_ids] = True
    unfinished = np.ones(B, dtype=bool)
    excused = np.zeros(B, dtype=bool)
    new, last = [], None
    for step in range(max_new_tokens):
        tok, near = next_tokens(logits_fn(step, last), presence, do_sample=do_sample, temperature=temperature,
                                top_k=top_k, top_p=top_p, penalty=penalty, seed=seed, step=step)
        excused |= near & unfinished
        if eos_token_id:
            tok = np.where(unfinished, tok, pad_token_id)
        presence[np.arange(B), tok] = True
        new.append(tok)
        last = tok
        if eos_token_id:
            unfinished = get_unfinished_flag(tok, unfinished, eos_token_id)
            if not unfinished.any():
                break
    return np.concatenate([input_ids, np.stack(new, 1)], 1), presence, ~unfinished, excused
