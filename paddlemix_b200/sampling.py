"""Decoding settings and on-device token selection for generate() (PaddleNLP GenerationMixin.generate,
generation/utils.py, with the GenerationConfig defaults of configuration_utils.py:138-163).

resolve_generation_args() checks the arguments without touching a device. TokenSampler holds the per-call device state
of b200mix_sample_tokens (presence bitmap, finished flags, step counter, output buffer) so that a whole decode loop can
run as CUDA-graph replays with no host round trip per token."""
from dataclasses import dataclass
from typing import List, Optional

import torch

# generate() reads the all-finished flag once per this many decode steps: one 32-byte D2H copy
FINISH_CHECK_INTERVAL = 8


@dataclass(frozen=True)
class GenerationArgs:
    do_sample: bool
    temperature: float
    top_k: int
    top_p: float
    repetition_penalty: float
    eos_token_id: List[int]
    pad_token_id: int
    # False when the call only uses what plain greedy generate() always took (no penalty, no sampling, eos None or an
    # int, no pad_token_id): that path is kept as it is
    on_device: bool


def resolve_generation_args(decode_strategy="greedy_search", do_sample=False, temperature=1.0, top_k=50, top_p=1.0,
                            repetition_penalty=1.0, eos_token_id=None, pad_token_id=None) -> GenerationArgs:
    """Validates generate()'s decoding arguments (the reference's checks: RepetitionPenaltyLogitsProcessor
    logits_process.py:99-101, TopPProcess / temperature ranges, pad defaulting at utils.py:873-875)."""
    if decode_strategy == "beam_search":
        raise NotImplementedError("decode_strategy='beam_search' is not supported")
    if decode_strategy not in ("greedy_search", "sampling"):
        raise ValueError(f"decode_strategy must be 'greedy_search' or 'sampling', got {decode_strategy!r}")
    sampling = bool(do_sample) or decode_strategy == "sampling"
    temperature, top_p, penalty = float(temperature), float(top_p), float(repetition_penalty)
    if not temperature > 0.0 or temperature == float("inf"):
        raise ValueError(f"`temperature` has to be a strictly positive float, but is {temperature}")
    if not 0.0 < top_p <= 1.0:
        raise ValueError(f"`top_p` has to be a float in (0, 1], but is {top_p}")
    if top_k is None:
        top_k = 0
    if int(top_k) != top_k or top_k < 0:
        raise ValueError(f"`top_k` has to be a non-negative integer, but is {top_k}")
    if not penalty > 0.0 or penalty == float("inf"):
        raise ValueError(f"`penalty` has to be a strictly positive float, but is {penalty}")
    eos_list = eos_token_id is not None and not isinstance(eos_token_id, int)
    eos = [] if eos_token_id is None else ([int(eos_token_id)] if not eos_list else [int(e) for e in eos_token_id])
    on_device = sampling or penalty != 1.0 or eos_list or pad_token_id is not None
    if pad_token_id is None and eos:
        if eos_list:
            raise ValueError("pad_token_id is required when eos_token_id is a list")
        pad_token_id = eos[0]
    return GenerationArgs(do_sample=sampling, temperature=temperature, top_k=int(top_k), top_p=top_p,
                          repetition_penalty=penalty, eos_token_id=eos,
                          pad_token_id=0 if pad_token_id is None else int(pad_token_id), on_device=on_device)


def seed_from(generator: Optional[torch.Generator] = None) -> int:
    """A 63-bit Philox key drawn from `generator` (torch's default CPU generator when None)."""
    dev = generator.device if generator is not None else "cpu"
    return int(torch.randint(0, 2 ** 63 - 1, (1,), generator=generator, device=dev).item())


def presence_bitmap(ids: torch.Tensor, vocab_size: int) -> torch.Tensor:
    """int32 [B, ceil(V/32)]: bit i of word i // 32 is set when id i occurs in the row of ids [B, S]."""
    B = ids.shape[0]
    words = (vocab_size + 31) // 32
    seen = torch.zeros(B, words * 32, dtype=torch.bool)
    seen.scatter_(1, ids.cpu().long(), True)
    w = (seen.view(B, words, 32).long() << torch.arange(32)).sum(-1)  # < 2^32
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


class TokenSampler:
    """Device state of one generate() call. Calling it with fp32 logits [B, V] (any row stride) enqueues one
    b200mix_sample_tokens launch: the chosen ids go to `ids` (int64 [B], what the next decode step embeds) and to column
    `step` of `out` (int64 [B, max_new_tokens])."""

    def __init__(self, prompt_ids: torch.Tensor, vocab_size: int, max_new_tokens: int, args: GenerationArgs, seed: int,
                 device):
        B = prompt_ids.shape[0]
        if int(prompt_ids.min()) < 0 or int(prompt_ids.max()) >= vocab_size:
            raise ValueError(f"prompt ids must lie in [0, {vocab_size})")
        if args.eos_token_id and not 0 <= args.pad_token_id < vocab_size:
            raise ValueError(f"pad_token_id={args.pad_token_id} must lie in [0, {vocab_size})")
        self.args, self.seed, self.max_new_tokens = args, int(seed), int(max_new_tokens)
        self.presence = presence_bitmap(prompt_ids, vocab_size).to(device)
        self.finished = torch.zeros(B, dtype=torch.int32, device=device)
        self.state = torch.zeros(4, dtype=torch.int64, device=device)
        self.out = torch.zeros(B, self.max_new_tokens, dtype=torch.int64, device=device)
        self.ids = torch.zeros(B, dtype=torch.int64, device=device)
        self.eos = torch.tensor(args.eos_token_id, dtype=torch.int64, device=device) if args.eos_token_id else None

    def __call__(self, logits: torch.Tensor):
        from . import ops
        a = self.args
        ops.sample_tokens(logits, self.presence, self.finished, self.state, self.out, self.ids, self.eos,
                          a.pad_token_id, do_sample=a.do_sample, temperature=a.temperature, top_k=a.top_k,
                          top_p=a.top_p, repetition_penalty=a.repetition_penalty, seed=self.seed)

    def all_finished(self) -> bool:
        return self.eos is not None and bool(self.state[2].item())

    def n_generated(self) -> int:
        """Tokens that belong to the result: up to and including the step at which the last row finished (the
        reference's stopping rule), else every step taken (at most max_new_tokens)."""
        s = self.state.cpu()
        n = int(s[3]) + 1 if int(s[2]) else int(s[0])
        return min(n, self.max_new_tokens)
