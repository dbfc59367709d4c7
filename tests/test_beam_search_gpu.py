"""b200mix_beam_search_step, b200mix_kv_reorder and Qwen2-VL generate(decode_strategy="beam_search") against the CPU
oracle (oracle/beam_search.py). Tokens and parents are compared exactly and scores within 1e-5. An item may differ
from the oracle (is excused) only when two candidates whose order can change the result, or the two sides of a scorer
comparison, lie within oracle.beam_search.NEAR (1e-6 relative) of each other, where fp32 rounding (device expf / logf
and summation order against the CPU's) may swap them; fewer than 1 % of the items may be excused."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import beam_search as G
from oracle import qwen2vl as O

pytestmark = pytest.mark.gpu


def _cache(rows, max_len, n_layers=1, n_kv=1, hd=8, seed=0):
    from paddlemix_b200.qwen2_vl.modeling_qwen2_vl import KVCache
    c = KVCache(0, rows, max_len, n_kv, hd, "cuda")
    g = torch.Generator(device="cuda").manual_seed(seed)
    c.k = [torch.randn(rows, max_len, n_kv, hd, generator=g, device="cuda").to(torch.bfloat16) for _ in range(n_layers)]
    c.v = [torch.randn(rows, max_len, n_kv, hd, generator=g, device="cuda").to(torch.bfloat16) for _ in range(n_layers)]
    return c


def _searcher(prompt, V, nb, max_new, **kw):
    from paddlemix_b200.beam_search import BeamSearcher, resolve_beam_search_args
    args = resolve_beam_search_args(num_beams=nb, **kw)
    B, S = prompt.shape
    cache = _cache(B * nb, S + max_new)
    cache.length = S
    return BeamSearcher(prompt, V, max_new, args, cache, "cuda")


def _presence_np(bm, V):
    """int32 [rows, words] bitmap -> bool [rows, V]."""
    w = bm.cpu().numpy().view(np.uint32)
    return ((w[:, :, None] >> np.arange(32, dtype=np.uint32)) & 1).astype(bool).reshape(w.shape[0], -1)[:, :V]


SETTINGS = [  # (B, penalty, diversity_rate, eos)
    (1, 1.0, 0.0, None),
    (8, 1.3, 0.0, 3),
    (32, 1.0, 0.7, 3),
    (8, 1.05, 0.3, None),
]


@pytest.mark.parametrize("nb", [2, 4, 8, 16])
@pytest.mark.parametrize("V", [1024, 32001, 152064])
def test_step_equals_oracle(V, nb):
    g = torch.Generator().manual_seed(V + nb)
    step, items, excused_items = 3, 0, 0
    for B, pen, div, eos in SETTINGS:
        if V * B * nb > 152064 * 8 * 16:
            B = 8  # keeps the CPU oracle's memory bounded
        rows = B * nb
        prompt = torch.randint(0, V, (B, 40), generator=g)
        s = _searcher(prompt, V, nb, step + 1, repetition_penalty=pen, diversity_rate=div, eos_token_id=eos)
        logits = torch.randn(rows, V, generator=g) * 3
        if eos is not None:
            logits[:, eos] += 8.0  # eos candidates at several ranks
        bs = -torch.rand(rows, generator=g) * 5
        s.t["beam_scores"].copy_(bs)
        s.t["state"][0] = step
        presence = None
        if pen != 1.0:  # the bitmaps of step 3 live in buffer 1
            bm = (torch.randint(0, 2 ** 31, (rows, (V + 31) // 32), generator=g) & torch.randint(
                0, 2 ** 31, (rows, (V + 31) // 32), generator=g)).to(torch.int32)
            s.presence[1].copy_(bm)
            presence = _presence_np(bm, V)
        s(logits.cuda())
        sc, tk, bm_, near = G.beam_step(logits.numpy(), bs.numpy(), presence, nb, pen, div, eos)
        hyps = [G.BeamHypotheses(nb, 1.0, False) for _ in range(B)]
        done = np.zeros(B, bool)
        ns, nt, ni = G.beam_process(hyps, done, np.arange(rows)[:, None], sc, tk, bm_, step, eos, 0)
        excused = near | np.array([h.near for h in hyps])
        got_t = s.t["tokens"][step].cpu().numpy()
        got_p = s.t["parents"][step].cpu().numpy()
        got_s = s.t["beam_scores"].cpu().numpy()
        assert np.array_equal(s.ids.cpu().numpy(), got_t)
        want_p = ni - np.repeat(np.arange(B), nb) * nb
        for b in range(B):
            r = slice(b * nb, (b + 1) * nb)
            if excused[b]:
                continue
            assert np.array_equal(got_t[r], nt[r]) and np.array_equal(got_p[r], want_p[r]), (B, pen, div, b)
            np.testing.assert_allclose(got_s[r], ns[r], rtol=1e-5, atol=1e-5)
            assert int(s.t["hyp_count"][b]) == len(hyps[b].beams) and bool(s.t["done"][b]) == bool(done[b])
            for i, (score, hyp) in enumerate(hyps[b].beams):
                assert abs(float(s.t["hyp_score"][b, i]) - score) <= 1e-5 * abs(score)
                assert int(s.t["hyp_step"][b, i]) == step and int(s.t["hyp_slot"][b, i]) == int(hyp[0]) - b * nb
        if presence is not None and not excused.any():  # children = parent bitmap + the new id, into buffer 0
            want = presence[ni]
            want[np.arange(rows), nt] = True
            assert np.array_equal(_presence_np(s.presence[0], V), want)
        items += B
        excused_items += int(excused.sum())
    assert excused_items <= 0.01 * items, (excused_items, items)


def test_engineered_ties_take_the_lowest_flat_index():
    B, nb, V = 2, 4, 1000
    g = torch.Generator().manual_seed(1)
    row = -5 + torch.rand(V, generator=g)
    row[[9, 3, 7]] = 5.0
    s = _searcher(torch.zeros(B, 1, dtype=torch.long), V, nb, 2)
    s.t["beam_scores"].zero_()  # identical beams
    s(row.cuda().repeat(B * nb, 1))
    # candidates (beam, token): (0,3) (0,7) (0,9) (1,3) (1,7) (1,9) (2,3) (2,7); the first four fill the slots
    assert s.t["tokens"][0].tolist() == [3, 7, 9, 3] * B and s.t["parents"][0].tolist() == [0, 0, 0, 1] * B
    s = _searcher(torch.zeros(B, 1, dtype=torch.long), V, nb, 2, diversity_rate=0.0)
    s.t["beam_scores"].zero_()
    flat = torch.zeros(B * nb, V)  # every score equal: flat indices 0, 1, 2, 3
    s(flat.cuda())
    assert s.t["tokens"][0].tolist() == [0, 1, 2, 3] * B and s.t["parents"][0].tolist() == [0] * nb * B


def test_engineered_ties_with_diversity_take_the_lowest_position():
    """Identical beams with diversity_rate > 0: each row ranks tokens 3, 7, 9 (equal scores, lower id first); the
    diversified scores of rank 1 are equal across the beams, so the lower (beam, rank) position comes first."""
    B, nb, V = 2, 4, 1000
    g = torch.Generator().manual_seed(3)
    row = -5 + torch.rand(V, generator=g)
    row[[9, 3, 7]] = 5.0
    s = _searcher(torch.zeros(B, 1, dtype=torch.long), V, nb, 2, diversity_rate=0.5)
    s.t["beam_scores"].zero_()
    logits = row.repeat(B * nb, 1)
    s(logits.cuda())
    # diversified list: rank 1 of beams 0..3 (token 3), then rank 2 of beams 0..3 (token 7); the first four fill
    assert s.t["tokens"][0].tolist() == [3, 3, 3, 3] * B and s.t["parents"][0].tolist() == [0, 1, 2, 3] * B
    sc, tk, bm, _ = G.beam_step(logits.numpy(), np.zeros(B * nb, np.float32), None, nb, diversity_rate=0.5)
    assert tk[:, :nb].tolist() == [[3] * nb] * B and bm[:, :nb].tolist() == [list(range(nb))] * B
    assert tk[:, nb:].tolist() == [[7] * nb] * B


def test_step_zero_never_picks_the_initial_minus_1e6_beams():
    B, nb, V = 4, 8, 32001
    g = torch.Generator().manual_seed(2)
    logits = (torch.randn(B, V, generator=g) * 3).repeat_interleave(nb, 0)
    s = _searcher(torch.zeros(B, 1, dtype=torch.long), V, nb, 2)
    s(logits.cuda())
    assert (s.t["parents"][0] == 0).all()
    want = torch.sort(logits[::nb], dim=1, descending=True, stable=True).indices[:, :nb]
    assert torch.equal(s.t["tokens"][0].cpu().view(B, nb), want)
    assert (s.t["beam_scores"].cpu() > -1e5).all()


@pytest.mark.parametrize("early", [False, True])
def test_scripted_multi_step_run_equals_oracle_loop(early):
    """Scripted logits (independent of the beams) with eos at various ranks: items finish at different steps. The
    device's tables, hypothesis store and finalize output equal the oracle loop's; the steps after every item is done
    change nothing."""
    B, nb, V, S, max_new, eos, pad = 5, 3, 300, 6, 14, 5, 7
    g = torch.Generator().manual_seed(10 + early)
    prompt = torch.randint(0, V, (B, S), generator=g)
    L = []
    for t in range(max_new):
        l = torch.randn(B * nb, V, generator=g) * 2
        l[:, eos] += torch.rand(B * nb, generator=g) * 2 + 0.5 * t  # eos climbs the ranks as the steps go on
        L.append(l.numpy())
    kw = dict(num_return_sequences=2, early_stopping=early, eos_token_id=eos, pad_token_id=pad, repetition_penalty=1.1)
    s = _searcher(prompt, V, nb, max_new, length_penalty=0.8, **kw)
    for t in range(max_new):
        s(torch.from_numpy(L[t]).cuda())
    want, want_s, excused, info = G.beam_search(lambda t, tok, rows: L[t], prompt.numpy(), max_new, V, nb, penalty=1.1,
                                                length_penalty=0.8, early_stopping=early, num_return_sequences=2,
                                                eos_token_id=eos, pad_token_id=pad)
    assert not excused.any()
    done = info["done"]
    assert 0 < done.sum()
    assert np.array_equal(s.t["done"].cpu().numpy().astype(bool), done)
    assert int(s.t["state"][0]) == info["steps"] and int(s.t["state"][1]) == 0
    assert int(s.t["state"][2]) == int(done.all())
    for b, h in enumerate(info["hyps"]):
        if done[b]:
            assert int(s.t["hyp_count"][b]) == len(h.beams)
    got, got_s = s.finalize()
    assert np.array_equal(got.numpy(), want), (got, want)
    np.testing.assert_allclose(got_s.numpy(), want_s, rtol=1e-5)


@pytest.mark.parametrize("nb,n_kv,hd,max_new", [
    (4, 2, 64, 9),     # 32 positions per CTA: one position block
    (4, 4, 128, 40),   # the Qwen2-VL-7B row (512 bf16): 8 positions per CTA, 5 blocks
    (16, 4, 128, 40),  # 2 positions per CTA, 19 blocks
])
def test_kv_reorder_equals_index_select(nb, n_kv, hd, max_new):
    from paddlemix_b200 import ops
    B, S, t = 4, 5, 4
    n = max_new - 3
    cache = _cache(B * nb, S + max_new, n_layers=3, n_kv=n_kv, hd=hd, seed=3)
    before_k = [k.clone() for k in cache.k]
    before_v = [v.clone() for v in cache.v]
    layer_kv = torch.tensor([t.data_ptr() for kv in zip(cache.k, cache.v) for t in kv], dtype=torch.int64,
                            device="cuda")
    g = torch.Generator().manual_seed(nb + hd)
    perm = [torch.randint(0, nb, (nb,), generator=g) for _ in range(B)]
    for b in (0, 2):  # moved items, each with a duplicated (and so a dropped) parent
        perm[b][0] = perm[b][1] = (perm[b][1] + 1) % nb
    perm[3] = torch.arange(nb)  # identity
    parents = torch.zeros(max_new, B * nb, dtype=torch.int32)
    parents[t] = torch.cat(perm).to(torch.int32)
    state = torch.tensor([t + 1, 0, 0, n], dtype=torch.int64, device="cuda")
    done = torch.tensor([0, 1, 0, 0], dtype=torch.int32, device="cuda")  # item 1 is done: left alone
    ops.kv_reorder(layer_kv, cache.k[0], nb, S, parents.cuda(), state, done)
    idx = torch.arange(B * nb)
    for b in (0, 2):
        idx[b * nb:(b + 1) * nb] = perm[b] + b * nb
    for before, after in ((before_k, cache.k), (before_v, cache.v)):
        for li in range(3):
            want = before[li].clone()
            want[:, S:S + n] = torch.index_select(before[li][:, S:S + n], 0, idx.cuda())
            assert torch.equal(after[li], want), li
            assert torch.equal(after[li][:, :S], before[li][:, :S])  # prompt rows bitwise unchanged
    # the identity permutation and a zero length write nothing
    parents[t] = torch.arange(nb, dtype=torch.int32).repeat(B)
    snap = [k.clone() for k in cache.k]
    ops.kv_reorder(layer_kv, cache.k[0], nb, S, parents.cuda(), state, torch.zeros(B, dtype=torch.int32, device="cuda"))
    state[3] = 0
    parents[t] = torch.full((B * nb,), nb - 1, dtype=torch.int32)
    ops.kv_reorder(layer_kv, cache.k[0], nb, S, parents.cuda(), state, torch.zeros(B, dtype=torch.int32, device="cuda"))
    assert all(torch.equal(a, b) for a, b in zip(cache.k, snap))


def test_graph_replays_equal_eager_launches():
    B, nb, V, S, n = 3, 4, 32001, 5, 7
    g = torch.Generator().manual_seed(6)
    logits = (torch.randn(B * nb, V, generator=g) * 2).cuda()
    prompt = torch.randint(0, V, (B, S), generator=g)
    kw = dict(repetition_penalty=1.5, eos_token_id=11, length_penalty=1.2)
    eager = _searcher(prompt, V, nb, n, **kw)
    for _ in range(n):
        eager(logits)
    graphed = _searcher(prompt, V, nb, n, **kw)  # same seeded cache contents as `eager`
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        graphed(logits)
    assert int(graphed.t["state"][0]) == 0  # capture does not run the kernels
    for _ in range(n):
        graph.replay()
    assert torch.equal(graphed.arena, eager.arena) and torch.equal(graphed.presence, eager.presence)
    assert all(torch.equal(a, b) for a, b in zip(graphed.cache.k + graphed.cache.v, eager.cache.k + eager.cache.v))
    assert len(set(eager.t["tokens"][:, 0].tolist())) > 1


def test_c_abi_rejects_bad_arguments():
    """Only invalid arguments: every call returns before anything is launched."""
    from paddlemix_b200 import _lib
    from paddlemix_b200._lib import lib
    INVALID = -1
    B, nb, V, max_new = 2, 4, 64, 3
    s = _searcher(torch.zeros(B, 1, dtype=torch.long), V, nb, max_new, repetition_penalty=1.2)
    logits = torch.zeros(B * nb, V, device="cuda")
    t = s.t

    def state(**over):
        f = {k: t[k].data_ptr() for k in ("state", "ids", "beam_scores", "tokens", "parents", "hyp_score", "hyp_step",
                                          "hyp_slot", "hyp_count", "hyp_worst", "done")}
        f["next_ids"] = f.pop("ids")
        f["presence"] = s.presence.data_ptr()
        f.update(over)
        return _lib.BeamState(**f)

    def step(ptr=logits.data_ptr(), ld=V, b=B, n=nb, v=V, st=None, ws=s.workspace.numel(), eos=-1, pad=0, pen=1.2,
             div=0.0, lp=1.0):
        return lib.b200mix_beam_search_step(ctypes.c_void_p(ptr), ld, b, n, v, ctypes.byref(st or state()),
                                            ctypes.c_void_p(s.workspace.data_ptr()), ws, max_new, eos, pad, pen, div,
                                            lp, 0, None)

    for kw in (dict(n=1), dict(n=17), dict(v=7, ld=7), dict(ld=V - 1), dict(pen=0.0), dict(pen=-1.0),
               dict(div=-0.5), dict(div=float("inf")), dict(lp=float("nan")), dict(pad=V), dict(eos=V), dict(eos=-2),
               dict(ws=8), dict(ptr=logits.data_ptr() + 2), dict(st=state(presence=None)),
               dict(st=state(done=None)), dict(st=state(hyp_score=t["hyp_score"].data_ptr() + 4)), dict(b=0),
               dict(b=70000)):
        assert step(**kw) == INVALID, kw
    cache = s.cache
    kvt = s.layer_kv

    def reorder(n_layers=1, b=B, n=nb, max_len=cache.max_len, row=8, S=1, mn=max_new):
        return lib.b200mix_kv_reorder(ctypes.c_void_p(kvt.data_ptr()), n_layers, b, n, max_len, row, S, mn,
                                      ctypes.c_void_p(t["parents"].data_ptr()), ctypes.c_void_p(t["state"].data_ptr()),
                                      ctypes.c_void_p(t["done"].data_ptr()), None)

    for kw in (dict(n=1), dict(n=17), dict(row=12), dict(row=8192), dict(max_len=2), dict(n_layers=0), dict(b=0)):
        assert reorder(**kw) == INVALID, kw
    with pytest.raises(_lib.B200MixError):
        from paddlemix_b200 import ops
        ops.beam_search_workspace_bytes(1, 1, 64)


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


def test_qwen2vl_generate_beam_search_matches_host_loop():
    """generate(decode_strategy="beam_search") equals a host loop in the reference's structure: eager forward() decode
    calls, the cache reordered with index_select after every step, selection by the oracle's scorer."""
    from paddlemix_b200.beam_search import expand_cache
    from paddlemix_b200.qwen2_vl import Qwen2VLForConditionalGeneration
    cfg = O.QWEN2VL_CONFIGS["tiny"]
    model = Qwen2VLForConditionalGeneration(cfg).load_state_dict(O.init_qwen2vl_params(cfg, seed=5), device=0)
    grid = [[1, 8, 8], [1, 4, 8], [1, 8, 8]]
    ids, am, pv = _padded(cfg, grid, [20, 9, 14])
    V, nb, max_new, pen = cfg["vocab_size"], 4, 10, 1.05

    def host_loop(eos, nrs):
        model.cache_headroom = max_new
        out = model(input_ids=ids, attention_mask=am, pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid),
                    use_cache=True)
        cache = expand_cache(out.past_key_values, nb)
        deltas = out.rope_deltas.repeat_interleave(nb, 0)
        first = out.logits[:, -1].repeat_interleave(nb, 0).cpu().numpy()

        def logits_fn(step, tokens, rows):
            if step == 0:
                return first
            idx = torch.from_numpy(rows).cuda()
            cache.k = [torch.index_select(k, 0, idx) for k in cache.k]  # reorder_cache
            cache.v = [torch.index_select(v, 0, idx) for v in cache.v]
            o = model(input_ids=torch.from_numpy(tokens)[:, None], past_key_values=cache, rope_deltas=deltas,
                      use_cache=True)
            return o.logits[:, 0].cpu().numpy()
        return G.beam_search(logits_fn, ids.numpy(), max_new, V, nb, penalty=pen, num_return_sequences=nrs,
                             eos_token_id=eos, pad_token_id=0 if eos is None else eos)

    free, _, excused, _ = host_loop(None, 1)
    assert not excused.any()
    S = ids.shape[1]
    eos = int(free[0, S + 3])  # the best hypothesis of prompt 0 would produce it at step 3

    def run():
        return model.generate(ids, pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid), attention_mask=am,
                              max_new_tokens=max_new, decode_strategy="beam_search", num_beams=nb,
                              repetition_penalty=pen, eos_token_id=eos, num_return_sequences=2, return_scores=True)
    want, want_s, excused, info = host_loop(eos, 2)
    assert not excused.any()
    gen, scores = run()
    assert (gen[:, S:] == eos).any()
    assert torch.equal(gen, torch.from_numpy(want)), (gen[:, S:], want[:, S:])
    np.testing.assert_allclose(scores.numpy(), want_s, rtol=1e-4, atol=1e-4)
    gen2, scores2 = run()
    assert torch.equal(gen, gen2) and torch.equal(scores, scores2)
    # without eos, the loop runs max_new_tokens steps and returns the prompt plus max_new_tokens tokens per row
    free_gen = model.generate(ids, pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid), attention_mask=am,
                              max_new_tokens=max_new, decode_strategy="beam_search", num_beams=nb,
                              repetition_penalty=pen)
    assert torch.equal(free_gen, torch.from_numpy(free))
    with pytest.raises(ValueError):
        model.generate(ids, attention_mask=am, max_new_tokens=2, num_beams=4)  # num_beams needs beam_search
    with pytest.raises(ValueError):
        model.generate(ids, attention_mask=am, max_new_tokens=2, return_scores=True)
