"""Beam search for generate() (PaddleNLP GenerationMixin.beam_search, generation/utils.py:1484-1649, with
BeamHypotheses / BeamSearchScorer :98-316 and the GenerationConfig defaults of configuration_utils.py:149-173).

resolve_beam_search_args() checks the arguments without touching a device. BeamSearcher holds the per-call device state
of b200mix_beam_search_step and b200mix_kv_reorder: a call selects the next tokens of every beam and reorders the
generated part of the KV cache, with no host round trip, so it can sit inside the graphed decode step. finalize()
copies the small tables to the host once and applies BeamSearchScorer.finalize."""
import math
from dataclasses import dataclass
from typing import List, Optional, Tuple

import torch

MAX_BEAMS = 16  # 2 * num_beams candidates per item fit one warp
WORST_INIT = 1e6  # get_scale_by_dtype() for fp32 (transformers/utils.py:91-112): BeamHypotheses.worst_score
BEAM_INIT = -1e6  # initial score of beams 1 .. nb-1 (:1523-1526)


@dataclass(frozen=True)
class BeamSearchArgs:
    num_beams: int
    num_return_sequences: int
    length_penalty: float
    early_stopping: bool
    diversity_rate: float
    repetition_penalty: float
    eos_token_id: Optional[int]
    pad_token_id: int


def resolve_beam_search_args(num_beams=1, num_return_sequences=1, length_penalty=1.0, early_stopping=False,
                             diversity_rate=0.0, num_beam_groups=1, repetition_penalty=1.0, eos_token_id=None,
                             pad_token_id=None) -> BeamSearchArgs:
    """The reference's checks (BeamSearchScorer :177-190, generate :958-969) plus what this implementation leaves out:
    group beam search, an eos list and early_stopping="never" raise NotImplementedError."""
    if isinstance(num_beams, bool) or not isinstance(num_beams, int) or num_beams <= 1:
        raise ValueError(f"`num_beams` has to be an integer strictly greater than 1, but received {num_beams!r}. "
                         "For `num_beams` == 1, use decode_strategy='greedy_search' instead.")
    if num_beams > MAX_BEAMS:
        raise NotImplementedError(f"num_beams={num_beams}: beam search supports at most {MAX_BEAMS} beams")
    if num_beam_groups != 1:
        raise NotImplementedError("group beam search (num_beam_groups > 1) is not supported")
    if isinstance(num_return_sequences, bool) or not isinstance(num_return_sequences, int) or \
            not 1 <= num_return_sequences <= num_beams:
        raise ValueError(f"`num_return_sequences` has to be an integer in [1, num_beams={num_beams}], "
                         f"but received {num_return_sequences!r}")
    length_penalty, diversity_rate, penalty = float(length_penalty), float(diversity_rate), float(repetition_penalty)
    if not math.isfinite(length_penalty):
        raise ValueError(f"`length_penalty` has to be finite, but is {length_penalty}")
    if not math.isfinite(diversity_rate) or diversity_rate < 0.0:
        raise ValueError(f"`diversity_rate` has to be finite and >= 0, but is {diversity_rate}")
    if early_stopping == "never":
        raise NotImplementedError("early_stopping='never' is not supported (the reference treats it as True)")
    if not isinstance(early_stopping, bool):
        raise ValueError(f"`early_stopping` has to be a bool, but is {early_stopping!r}")
    if not penalty > 0.0 or penalty == float("inf"):
        raise ValueError(f"`penalty` has to be a strictly positive float, but is {penalty}")
    if eos_token_id is not None and not isinstance(eos_token_id, int):
        raise NotImplementedError("beam search takes one int eos_token_id, not a list")
    if pad_token_id is None:
        pad_token_id = eos_token_id
    return BeamSearchArgs(num_beams=num_beams, num_return_sequences=num_return_sequences,
                          length_penalty=length_penalty, early_stopping=early_stopping,
                          diversity_rate=diversity_rate, repetition_penalty=penalty, eos_token_id=eos_token_id,
                          pad_token_id=0 if pad_token_id is None else int(pad_token_id))


def length_factor(n_generated: int, length_penalty: float) -> float:
    """GNMT length normalisation: a hypothesis of n generated tokens has score sum_logprobs / ((n + 5) / 6) ** lp."""
    return ((n_generated + 5) / 6) ** length_penalty


def lowest_entry(scores: List[float], skip: int = -1) -> int:
    """Position of the lowest score (the earliest position among equal scores), position `skip` left out."""
    pick = -1
    for i, sc in enumerate(scores):
        if i != skip and (pick < 0 or sc < scores[pick]):
            pick = i
    return pick


class BeamHypotheses:
    """The n-best list of one item in Python double, the rules of the reference's BeamHypotheses (:98-143): entries
    (score, ref) in insertion order, at most num_beams of them, and `worst_score` (1e6 while empty). A new score is
    kept while the list has room, or when it beats worst_score; a full list then drops its lowest (score, position)
    entry and worst_score becomes the next lowest score. A ref is (generated length, beam slot): the tokens are
    recovered from the token / parent tables."""

    def __init__(self, num_beams, length_penalty, entries=(), worst_score=WORST_INIT):
        self.capacity, self.length_penalty = num_beams, length_penalty
        self.entries: List[Tuple[float, tuple]] = list(entries)
        self.worst_score = worst_score

    def add(self, sum_logprobs, n_generated, ref):
        score = sum_logprobs / length_factor(n_generated, self.length_penalty)
        full = len(self.entries) >= self.capacity
        if full and not score > self.worst_score:
            return
        self.entries.append((score, ref))
        if not full:
            self.worst_score = min(self.worst_score, score)
            return
        scores = [e[0] for e in self.entries]
        drop = lowest_entry(scores)
        self.worst_score = scores[lowest_entry(scores, skip=drop)]
        del self.entries[drop]

    def best(self, n: int):
        """The n highest entries, highest first; among equal scores the later insertion first."""
        order = sorted(range(len(self.entries)), key=lambda i: (-self.entries[i][0], -i))
        return [self.entries[i] for i in order[:n]]


def finalize_tables(prompt_ids: torch.Tensor, tokens: torch.Tensor, parents: torch.Tensor, beam_scores: torch.Tensor,
                    hyp_score: torch.Tensor, hyp_step: torch.Tensor, hyp_slot: torch.Tensor, hyp_count: torch.Tensor,
                    hyp_worst: torch.Tensor, done: torch.Tensor, n_steps: int, max_new_tokens: int,
                    args: BeamSearchArgs):
    """BeamSearchScorer.finalize (:264-316) on host copies of the device tables. prompt_ids [B, S]; tokens / parents
    [max_new, B * nb]; n_steps = selections made. Returns (ids int64 [B * nrs, S + L], scores fp32 [B * nrs])."""
    B, S = prompt_ids.shape
    nb, nrs = args.num_beams, args.num_return_sequences
    tokens, parents = tokens.tolist(), parents.tolist()
    best = []
    for b in range(B):
        n = int(hyp_count[b])
        hyps = BeamHypotheses(nb, args.length_penalty,
                              [(float(hyp_score[b, i]), (int(hyp_step[b, i]), int(hyp_slot[b, i]))) for i in range(n)],
                              float(hyp_worst[b]))
        if not int(done[b]):  # the open beams join the list with their running scores
            for j in range(nb):
                hyps.add(float(beam_scores[b * nb + j]), n_steps, (n_steps, j))
        for score, (length, slot) in hyps.best(nrs):
            seq = []
            for s in range(length - 1, -1, -1):  # backtrack through the parent table
                r = b * nb + slot
                seq.append(tokens[s][r])
                slot = parents[s][r]
            best.append((b, seq[::-1], score))
    lengths = [S + len(seq) for _, seq, _ in best]
    max_length = S + max_new_tokens
    width = min(max(lengths) + 1, max_length)
    fill = args.pad_token_id if min(lengths) != max(lengths) else 0
    out = torch.full((len(best), width), fill, dtype=torch.int64)
    for i, (b, seq, _) in enumerate(best):
        out[i, :S] = prompt_ids[b]
        out[i, S:lengths[i]] = torch.tensor(seq, dtype=torch.int64)
        if lengths[i] < max_length and args.eos_token_id is not None:
            out[i, lengths[i]] = args.eos_token_id
    return out, torch.tensor([s for _, _, s in best], dtype=torch.float32)


def expand_cache(cache, num_beams: int):
    """expand_inputs_for_generation (:413-423) for a filled KVCache: each item's rows repeated num_beams times
    (repeat_interleave order), key_bias included."""
    from .qwen2_vl.modeling_qwen2_vl import KVCache
    n_kv, hd = cache.k[0].shape[2:]
    out = KVCache(0, cache.batch * num_beams, cache.max_len, n_kv, hd, cache.k[0].device)
    out.k = [k.repeat_interleave(num_beams, 0) for k in cache.k]
    out.v = [v.repeat_interleave(num_beams, 0) for v in cache.v]
    out.length = cache.length
    out.key_bias = None if cache.key_bias is None else cache.key_bias.repeat_interleave(num_beams, 0)
    return out


class BeamSearcher:
    """Device state of one beam-search generate() call over B prompts of S tokens and an expanded cache of B * nb rows.
    Calling it with fp32 logits [B * nb, V] (any row stride) enqueues b200mix_beam_search_step and then
    b200mix_kv_reorder on the cache: the chosen ids go to `ids` (int64 [B * nb], what the next decode step embeds)."""

    def __init__(self, prompt_ids: torch.Tensor, vocab_size: int, max_new_tokens: int, args: BeamSearchArgs, cache,
                 device):
        from . import ops
        B, S = prompt_ids.shape
        nb = args.num_beams
        rows = B * nb
        if int(prompt_ids.min()) < 0 or int(prompt_ids.max()) >= vocab_size:
            raise ValueError(f"prompt ids must lie in [0, {vocab_size})")
        if not 0 <= args.pad_token_id < vocab_size or not (args.eos_token_id is None or
                                                             0 <= args.eos_token_id < vocab_size):
            raise ValueError(f"eos / pad token ids must lie in [0, {vocab_size})")
        if cache.batch != rows or cache.length != S or cache.max_len < S + max_new_tokens:
            raise ValueError(f"the cache must hold {rows} rows of {S} + {max_new_tokens} positions")
        self.prompt_ids, self.args, self.max_new_tokens, self.cache = prompt_ids.cpu(), args, int(max_new_tokens), cache
        # the small tables share one allocation, so that finalize() needs a single device-to-host copy
        self._fields = [("state", torch.int64, (4,)), ("ids", torch.int64, (rows,)),
                        ("tokens", torch.int64, (self.max_new_tokens, rows)),
                        ("parents", torch.int32, (self.max_new_tokens, rows)), ("beam_scores", torch.float32, (rows,)),
                        ("hyp_score", torch.float64, (B, nb)), ("hyp_step", torch.int32, (B, nb)),
                        ("hyp_slot", torch.int32, (B, nb)), ("hyp_count", torch.int32, (B,)),
                        ("hyp_worst", torch.float64, (B,)), ("done", torch.int32, (B,))]
        words = sum((math.prod(shape) * dt.itemsize + 7) // 8 for _, dt, shape in self._fields)
        self.arena = torch.zeros(words, dtype=torch.int64, device=device)
        self.t = self._views(self.arena)
        self.t["beam_scores"].view(B, nb)[:, 1:] = BEAM_INIT
        self.t["hyp_worst"].fill_(WORST_INIT)
        self.ids = self.t["ids"]
        self.presence = None
        if args.repetition_penalty != 1.0:
            from .sampling import presence_bitmap
            bm = presence_bitmap(self.prompt_ids.repeat_interleave(nb, 0), vocab_size)
            self.presence = torch.stack([bm, torch.zeros_like(bm)]).to(device)
        self.workspace = torch.empty(ops.beam_search_workspace_bytes(B, nb, vocab_size), dtype=torch.uint8,
                                     device=device)
        self.layer_kv = torch.tensor([t.data_ptr() for kv in zip(cache.k, cache.v) for t in kv], dtype=torch.int64,
                                     device=device)

    def _views(self, arena):
        out, o = {}, 0
        for name, dt, shape in self._fields:
            n = math.prod(shape)
            w = (n * dt.itemsize + 7) // 8
            out[name] = arena[o:o + w].view(dt)[:n].view(shape)
            o += w
        return out

    def __call__(self, logits: torch.Tensor):
        from . import ops
        a, t = self.args, self.t
        ops.beam_search_step(logits, a.num_beams, self.workspace, state=t["state"], next_ids=t["ids"],
                             beam_scores=t["beam_scores"], tokens=t["tokens"], parents=t["parents"],
                             hyp_score=t["hyp_score"], hyp_step=t["hyp_step"], hyp_slot=t["hyp_slot"],
                             hyp_count=t["hyp_count"], hyp_worst=t["hyp_worst"], done=t["done"],
                             presence=self.presence, eos_token_id=-1 if a.eos_token_id is None else a.eos_token_id,
                             pad_token_id=a.pad_token_id, repetition_penalty=a.repetition_penalty,
                             diversity_rate=a.diversity_rate, length_penalty=a.length_penalty,
                             early_stopping=a.early_stopping)
        ops.kv_reorder(self.layer_kv, self.cache.k[0], a.num_beams, self.prompt_ids.shape[1], t["parents"], t["state"],
                       t["done"])

    def all_done(self) -> bool:
        return bool(self.t["state"][2].item())

    def finalize(self):
        """-> (ids int64 [B * num_return_sequences, S + L] with the prompt, scores fp32 [B * num_return_sequences])."""
        h = self._views(self.arena.cpu())
        n_steps = min(int(h["state"][0]), self.max_new_tokens)
        return finalize_tables(self.prompt_ids, h["tokens"], h["parents"], h["beam_scores"], h["hyp_score"],
                               h["hyp_step"], h["hyp_slot"], h["hyp_count"], h["hyp_worst"], h["done"], n_steps,
                               self.max_new_tokens, self.args)
