"""b200mix_sample_tokens and Qwen2-VL generate() with sampling / repetition penalty / EOS lists, against the CPU
oracle (oracle/generation.py). Draws are compared id for id. A row may differ from the oracle (is excused) only when its
target lies within 1e-5 of a CDF boundary (relative to the kept mass) or its top-p cut lies within 1e-5 (relative) of
top_p, where fp32 rounding of the probabilities (device expf and summation order against the CPU's) may move the
result by one id; fewer than 1 % of the rows may be excused."""
import numpy as np
import pytest
import torch

from oracle import generation as G
from oracle import qwen2vl as O

pytestmark = pytest.mark.gpu


def _args(do_sample=True, temperature=1.0, top_k=0, top_p=1.0, penalty=1.0, eos=(), pad=0):
    from paddlemix_b200.sampling import GenerationArgs
    return GenerationArgs(do_sample=do_sample, temperature=temperature, top_k=top_k, top_p=top_p,
                          repetition_penalty=penalty, eos_token_id=list(eos), pad_token_id=pad, on_device=True)


def _presence(prompt, V):
    p = np.zeros((prompt.shape[0], V), dtype=bool)
    p[np.arange(prompt.shape[0])[:, None], prompt.numpy()] = True
    return p


SETTINGS = [  # (penalty, temperature, top_k, top_p)
    (1.0, 1.0, 0, 1.0),
    (1.05, 0.7, 50, 0.9),
    (1.3, 1.5, 0, 0.6),
    (1.0, 0.5, 1000, 0.95),
    (2.0, 1.0, 7, 1.0),
]


@pytest.mark.parametrize("V", [1024, 32001, 152064])
def test_sampled_ids_equal_oracle(V):
    """One logits row replicated into 4096 rows: every row draws with its own Philox counter (step, row)."""
    from paddlemix_b200.sampling import TokenSampler
    B, step = 4096, 3
    g = torch.Generator().manual_seed(V)
    row = torch.randn(V, generator=g) * 3
    prompt = torch.randint(0, V, (1, 64), generator=g)
    logits = row.cuda().repeat(B, 1)
    pres = _presence(prompt, V)
    for i, (pen, T, k, p) in enumerate(SETTINGS):
        seed = 0x9E3779B97F4A7C15 + 977 * i
        s = TokenSampler(prompt.expand(B, -1), V, step + 1, _args(True, T, k, p, pen), seed, "cuda")
        s.state[0] = step
        s(logits)
        got = s.out[:, step].cpu().numpy()
        assert np.array_equal(s.ids.cpu().numpy(), got)
        l = G.repetition_penalty(row.numpy()[None], pres, pen)
        probs = G.top_k_process(G.softmax_t(l, T), k)
        keep = G.top_p_keep(probs, p)
        want, near = G.draw_row(probs[0], keep[0], G.uniform(seed, step, np.arange(B)))
        near |= G.top_p_near_boundary(probs, p)[0]
        differ = got != want
        assert not (differ & ~near).any(), (V, (pen, T, k, p), int((differ & ~near).sum()))
        assert differ.mean() < 0.01, (V, (pen, T, k, p), differ.mean())  # excused rows
        assert len(set(got.tolist())) > 1  # real draws, not one id


def test_greedy_with_penalty_is_exact_argmax():
    from paddlemix_b200.sampling import TokenSampler
    B, V = 64, 32001
    g = torch.Generator().manual_seed(1)
    logits = torch.randn(B, V, generator=g) * 2
    prompt = torch.randint(0, V, (B, 200), generator=g)
    prompt[0].clamp_(min=21)  # ids 10 and 20 of row 0 are not penalised
    top = logits.max(1).values
    logits[0, 10] = logits[0, 20] = top[0] + 1  # tie: the lower id wins
    ids0 = prompt[1, 0]
    logits[1, ids0] = top[1] + 0.5  # the best logit, but seen in the prompt: divided by 3 it falls below the runner-up
    s = TokenSampler(prompt, V, 1, _args(False, penalty=3.0), 0, "cuda")
    s(logits.cuda())
    want, _ = G.next_tokens(logits.numpy(), _presence(prompt, V), do_sample=False, penalty=3.0)
    got = s.out[:, 0].cpu().numpy()
    assert np.array_equal(got, want) and got[0] == 10 and got[1] != ids0


def test_top_k_ties_and_top_p_boundaries():
    from paddlemix_b200.sampling import TokenSampler
    B, V = 4096, 1024
    g = torch.Generator().manual_seed(2)
    prompt = torch.zeros(1, 1, dtype=torch.long)
    # top-k = 5 with the 5th value shared by three ids: all seven ids survive
    row = -5 + 0.1 * torch.randn(V, generator=g)
    row[[5, 17, 300, 301]] = 10.0
    row[[400, 401, 402]] = 9.0
    s = TokenSampler(prompt.expand(B, -1), V, 1, _args(True, top_k=5), 11, "cuda")
    s(row.cuda().repeat(B, 1))
    got = s.out[:, 0].cpu().numpy()
    assert set(got.tolist()) == {5, 17, 300, 301, 400, 401, 402}
    probs = G.top_k_process(G.softmax_t(row.numpy()[None], 1.0), 5)
    want, near = G.draw_row(probs[0], np.ones(V, dtype=bool), G.uniform(11, 0, np.arange(B)))
    assert not ((got != want) & ~near).any()
    # four equal probabilities 0.25: masses above them are 0, .25, .5, .75 in id order
    row = torch.full((V,), float("-inf"))
    row[[3, 8, 100, 700]] = 0.0
    for top_p, kept in ((0.5, {3, 8, 100}), (0.3, {3, 8}), (1e-6, {3})):
        s = TokenSampler(prompt.expand(B, -1), V, 1, _args(True, top_p=top_p), 12, "cuda")
        s(row.cuda().repeat(B, 1))
        assert set(s.out[:, 0].cpu().tolist()) == kept, top_p


def _step_logits(B, V, steps, finish_at, eos, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for t in range(steps):
        l = torch.randn(B, V, generator=g)
        for b, f in enumerate(finish_at):
            if f == t:
                l[b, eos[b % len(eos)]] = 50.0
        out.append(l.numpy())
    return out


@pytest.mark.parametrize("finish_at", [[2, 5, 5, 8, 100, 0], [2, 5, 5, 8, 3, 0]])
def test_multi_step_eos_pad_and_bookkeeping(finish_at):
    """Rows finishing at different steps: pad fill, finished flags, the last-finish step and the presence bitmap match
    the oracle loop; steps past the end do not change the result."""
    from paddlemix_b200.sampling import TokenSampler, presence_bitmap
    B, V, steps, eos, pad = 6, 1000, 12, [7, 11], 0
    g = torch.Generator().manual_seed(4)
    prompt = torch.randint(0, V, (B, 30), generator=g)
    L = _step_logits(B, V, steps, finish_at, eos, seed=5)
    kw = dict(do_sample=True, temperature=0.8, top_k=20, top_p=0.95, penalty=1.1)
    seed = 1234567
    s = TokenSampler(prompt, V, steps, _args(True, 0.8, 20, 0.95, 1.1, eos, pad), seed, "cuda")
    for t in range(steps):
        s(torch.from_numpy(L[t]).cuda())
    ids, presence, finished, excused = G.generate(lambda t, last: L[t], prompt.numpy(), steps, V, eos_token_id=eos,
                                                  pad_token_id=pad, seed=seed, **kw)
    assert not excused.any()
    n = ids.shape[1] - prompt.shape[1]
    assert s.n_generated() == n
    assert np.array_equal(s.out[:, :n].cpu().numpy(), ids[:, prompt.shape[1]:])
    assert np.array_equal(s.finished.cpu().numpy().astype(bool), finished)
    st = s.state.cpu().tolist()
    assert st[0] == steps and st[1] == 0 and st[2] == int(finished.all())
    if finished.all():
        assert st[3] == n - 1 and (s.out[:, n:].cpu() == pad).all()
        bm = presence_bitmap(torch.cat([prompt, s.out.cpu()], 1), V)  # the extra steps emitted pad only
    else:
        bm = presence_bitmap(torch.from_numpy(ids), V)
    assert torch.equal(s.presence.cpu(), bm)


def test_graph_replays_equal_eager_launches():
    from paddlemix_b200.sampling import TokenSampler
    B, V, n = 16, 32001, 6
    g = torch.Generator().manual_seed(6)
    logits = (torch.randn(B, V, generator=g) * 2).cuda()
    prompt = torch.randint(0, V, (B, 40), generator=g)
    a = _args(True, 0.9, 40, 0.9, 1.5, [5], 0)
    eager = TokenSampler(prompt, V, n, a, 99, "cuda")
    for _ in range(n):
        eager(logits)
    graphed = TokenSampler(prompt, V, n, a, 99, "cuda")
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        graphed(logits)
    assert int(graphed.state[0]) == 0  # capture does not run the kernel
    for _ in range(n):
        graph.replay()
    assert torch.equal(graphed.out, eager.out) and torch.equal(graphed.presence, eager.presence)
    assert len(set(eager.out[0].tolist())) > 1


def test_sample_tokens_rejects_bad_arguments():
    from paddlemix_b200 import _lib
    from paddlemix_b200.sampling import TokenSampler
    B, V = 2, 64
    s = TokenSampler(torch.zeros(B, 1, dtype=torch.long), V, 2, _args(), 0, "cuda")
    logits = torch.zeros(B, V, device="cuda")
    from paddlemix_b200 import ops
    for kw in (dict(temperature=0.0), dict(top_p=0.0), dict(top_p=1.5), dict(top_k=-1), dict(repetition_penalty=0.0)):
        with pytest.raises(_lib.B200MixError):
            ops.sample_tokens(logits, s.presence, s.finished, s.state, s.out, s.ids, do_sample=True, **kw)
    big = torch.zeros(1, (1 << 20) + 1, device="cuda")
    pres = torch.zeros(1, ((1 << 20) + 32) // 32, dtype=torch.int32, device="cuda")
    with pytest.raises(_lib.B200MixError):
        ops.sample_tokens(big, pres, s.finished[:1], s.state, s.out[:1], s.ids[:1])
    eos = torch.tensor([3], dtype=torch.int64, device="cuda")
    with pytest.raises(_lib.B200MixError):  # pad id outside the vocabulary
        ops.sample_tokens(logits, s.presence, s.finished, s.state, s.out, s.ids, eos, V)


# ---- Qwen2-VL generate ----------------------------------------------------------------------------------------------

def _padded(cfg, grid, n_text, seed=7):
    """Left-padded prompts with images: ids [B, S], attention_mask [B, S], pixel values."""
    g = torch.Generator().manual_seed(seed)
    m2 = cfg["vision"]["spatial_merge_size"] ** 2
    T = sum(t * h * w for t, h, w in grid)
    pv = torch.randn(T, 3 * 2 * 14 * 14, generator=g)
    seqs = [[cfg["vision_start_token_id"]] + [cfg["image_token_id"]] * (t * h * w // m2) + [cfg["vision_end_token_id"]] +
            torch.randint(0, 1000, (nt,), generator=g).tolist() for (t, h, w), nt in zip(grid, n_text)]
    S = max(len(x) for x in seqs)
    ids, am = torch.zeros(len(seqs), S, dtype=torch.long), torch.zeros(len(seqs), S, dtype=torch.long)
    for i, x in enumerate(seqs):
        ids[i, S - len(x):], am[i, S - len(x):] = torch.tensor(x), 1
    return ids, am, pv


def _tiny_model(seed):
    from paddlemix_b200.qwen2_vl import Qwen2VLForConditionalGeneration
    cfg = O.QWEN2VL_CONFIGS["tiny"]
    return cfg, Qwen2VLForConditionalGeneration(cfg).load_state_dict(O.init_qwen2vl_params(cfg, seed=seed), device=0)


def test_qwen2vl_generate_instruct_settings_match_host_loop():
    """Instruct-style settings, do_sample with top_k=1, top_p=0.001, T=0.1, repetition penalty 1.05, a list of EOS ids
    and a pad id: generate() equals a host loop of eager forward() calls plus the
    oracle's processors, token for token."""
    from paddlemix_b200.sampling import seed_from
    cfg, model = _tiny_model(3)
    grid = [[1, 8, 8], [1, 4, 8], [1, 8, 8]]
    ids, am, pv = _padded(cfg, grid, [20, 9, 14])
    V, max_new = cfg["vocab_size"], 12
    kw = dict(do_sample=True, temperature=0.1, top_k=1, top_p=0.001, penalty=1.05)

    def host_loop(eos, pad, seed):
        model.cache_headroom = max_new
        out = model(input_ids=ids, attention_mask=am, pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid),
                    use_cache=True)
        cache, deltas = out.past_key_values, out.rope_deltas
        first = out.logits[:, -1].cpu().numpy()

        def logits_fn(step, last):
            if step == 0:
                return first
            o = model(input_ids=torch.from_numpy(last)[:, None], past_key_values=cache, rope_deltas=deltas, use_cache=True)
            return o.logits[:, 0].cpu().numpy()
        return G.generate(logits_fn, ids.numpy(), max_new, V, eos_token_id=eos, pad_token_id=pad, seed=seed, **kw)

    free, _, _, _ = host_loop(None, 0, 0)
    S = ids.shape[1]
    eos = [int(free[0, S + 2]), int(free[1, S + 5])]  # rows finish at different steps
    pad = 0
    seed = seed_from(torch.Generator().manual_seed(3))
    want, _, finished, excused = host_loop(eos, pad, seed)
    assert not excused.any()
    gen = model.generate(ids, pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid), attention_mask=am,
                         max_new_tokens=max_new, do_sample=True, temperature=0.1, top_k=1, top_p=0.001,
                         repetition_penalty=1.05, eos_token_id=eos, pad_token_id=pad,
                         generator=torch.Generator().manual_seed(3))
    assert torch.equal(gen, torch.from_numpy(want)), (gen[:, S:], want[:, S:])
    # greedy with the same penalty / eos list follows the same host loop (do_sample=False ignores T / top-k / top-p)
    gen_g = model.generate(ids, pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid), attention_mask=am,
                           max_new_tokens=max_new, repetition_penalty=1.05, eos_token_id=eos, pad_token_id=pad)
    assert torch.equal(gen_g, gen)
    with pytest.raises(ValueError):
        model.generate(ids, attention_mask=am, max_new_tokens=2, eos_token_id=eos)  # a list of EOS ids needs pad


def test_qwen2vl_generate_sampling_seeds_and_stopping_rule():
    cfg, model = _tiny_model(4)
    grid = [[1, 8, 8], [1, 8, 8]]
    ids, am, pv = _padded(cfg, grid, [10, 16], seed=8)
    B, S = ids.shape
    eos, pad, max_new = list(range(0, cfg["vocab_size"], 7)), 1, 40

    def run(seed):
        return model.generate(ids, pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid), attention_mask=am,
                              max_new_tokens=max_new, do_sample=True, temperature=1.0, top_k=50, top_p=0.9,
                              repetition_penalty=1.05, eos_token_id=eos, pad_token_id=pad,
                              generator=torch.Generator().manual_seed(seed))
    a, b, c = run(7), run(7), run(8)
    assert torch.equal(a, b)
    assert not (a.shape == c.shape and torch.equal(a, c))
    for out in (a, c):
        new = out[:, S:]
        n = new.shape[1]
        first_eos = []
        for r in range(B):
            hit = [j for j in range(n) if int(new[r, j]) in eos]
            first_eos.append(hit[0] if hit else None)
            if hit:
                assert (new[r, hit[0] + 1:] == pad).all()
        if all(f is not None for f in first_eos):
            assert n == max(first_eos) + 1
        else:
            assert n == max_new
