"""Beam search on the CPU: the argument checks of generate()'s beam branch, the oracle (oracle/beam_search.py) on
hand-computed cases, and BeamSearcher's host finalize (backtracking through the token / parent tables) against the
oracle's finalize on a scripted run."""
import numpy as np
import pytest
import torch

from oracle import beam_search as G


def _args(**kw):
    from paddlemix_b200.beam_search import resolve_beam_search_args
    return resolve_beam_search_args(**{"num_beams": 2, **kw})


def test_beam_search_args():
    from paddlemix_b200.beam_search import resolve_beam_search_args as R
    from paddlemix_b200.sampling import resolve_generation_args
    a = R(num_beams=4, eos_token_id=7)
    assert (a.num_beams, a.num_return_sequences, a.length_penalty, a.early_stopping, a.diversity_rate) == (4, 1, 1.0,
                                                                                                         False, 0.0)
    assert a.pad_token_id == 7 and R(num_beams=4).pad_token_id == 0 and R(num_beams=4, eos_token_id=7,
                                                                          pad_token_id=3).pad_token_id == 3
    for bad in (dict(num_beams=1), dict(num_beams=0), dict(num_beams=2.0), dict(num_beams=True),
                dict(num_beams=4, num_return_sequences=5), dict(num_beams=4, num_return_sequences=0),
                dict(num_beams=4, length_penalty=float("nan")), dict(num_beams=4, length_penalty=float("inf")),
                dict(num_beams=4, diversity_rate=-0.1), dict(num_beams=4, diversity_rate=float("inf")),
                dict(num_beams=4, early_stopping=1), dict(num_beams=4, repetition_penalty=0.0)):
        with pytest.raises(ValueError):
            R(**bad)
    for bad in (dict(num_beams=17), dict(num_beams=4, num_beam_groups=2), dict(num_beams=4, eos_token_id=[1, 2]),
                dict(num_beams=4, early_stopping="never")):
        with pytest.raises(NotImplementedError):
            R(**bad)
    with pytest.raises(NotImplementedError):  # the sampling resolver still refuses beam search
        resolve_generation_args(decode_strategy="beam_search")


def test_gnmt_length_penalty():
    h = G.BeamHypotheses(2, 2.0, False)
    h.add("x", -3.0, 7)
    assert h.beams[0][0] == -3.0 / ((12 / 6) ** 2.0) == -0.75  # ((len + 5) / 6) ** lp, not len ** lp
    from paddlemix_b200.beam_search import BeamHypotheses
    p = BeamHypotheses(2, 2.0)
    p.add(-3.0, 7, None)
    assert p.entries[0][0] == -0.75


def test_worst_score_replacement_rule():
    h = G.BeamHypotheses(2, 0.0, False)
    assert h.worst_score == 1e6
    h.add("a", -3.0, 1)
    assert h.worst_score == -3.0
    h.add("b", -1.0, 1)
    assert h.worst_score == -3.0
    h.add("c", -2.0, 1)  # overflow: the lowest goes, worst = the second lowest of the three
    assert [x for _, x in h.beams] == ["b", "c"] and h.worst_score == -2.0
    h.add("d", -2.0, 1)  # not better than the worst: ignored
    h.add("e", -5.0, 1)
    assert [x for _, x in h.beams] == ["b", "c"]


def test_host_n_best_list_replacement_and_order():
    from paddlemix_b200.beam_search import BeamHypotheses
    p = BeamHypotheses(2, 0.0)
    for ref, sc in (("a", -3.0), ("b", -1.0), ("c", -2.0), ("d", -2.0), ("e", -5.0)):
        p.add(sc, 1, ref)
    assert [r for _, r in p.entries] == ["b", "c"] and p.worst_score == -2.0
    p = BeamHypotheses(3, 0.0)
    for ref, sc in (("a", -3.0), ("b", -3.0), ("c", -3.0), ("d", -1.0)):  # equal lowest scores: the earliest goes
        p.add(sc, 1, ref)
    assert [r for _, r in p.entries] == ["b", "c", "d"] and p.worst_score == -3.0
    assert [r for _, r in p.best(3)] == ["d", "c", "b"]  # among equal scores the later insertion first


def test_early_stopping_modes():
    for early, want in ((True, True), (False, False)):
        h = G.BeamHypotheses(2, 1.0, early)
        assert not h.is_done(-0.1, 3)  # fewer than nb hypotheses
        h.add("a", -6.0, 1)
        h.add("b", -12.0, 1)  # worst = -12 / 1 = -12
        # best running -1.0 at 7 generated tokens: -1 / 2 = -0.5 > -12
        assert h.is_done(-1.0, 7) == want
    h = G.BeamHypotheses(2, 1.0, False)
    h.add("a", -6.0, 1)
    h.add("b", -12.0, 1)
    assert h.is_done(-30.0, 7)  # -30 / 2 = -15 <= -12


def test_process_skips_eos_at_rank_ge_nb_and_pads_done_items():
    eos, pad, nb = 9, 0, 2
    hyps = [G.BeamHypotheses(nb, 1.0, False) for _ in range(2)]
    done = np.array([False, True])
    ids = np.arange(4 * 3).reshape(4, 3)
    scores = np.array([[-1.0, -2.0, -3.0, -4.0], [-1, -2, -3, -4]], np.float32)
    tokens = np.array([[eos, 5, eos, 6], [1, 2, 3, 4]])
    beams = np.array([[1, 0, 0, 1], [0, 1, 0, 1]])
    ns, nt, ni = G.beam_process(hyps, done, ids, scores, tokens, beams, 0, eos, pad)
    assert len(hyps[0].beams) == 1 and np.array_equal(hyps[0].beams[0][1], ids[1])  # rank 0 eos: hypothesis of beam 1
    assert hyps[0].beams[0][0] == -1.0 / ((0 + 5) / 6)
    assert nt[:2].tolist() == [5, 6] and ns[:2].tolist() == [-2.0, -4.0] and ni[:2].tolist() == [0, 1]  # rank-2 eos
    assert nt[2:].tolist() == [pad, pad] and ns[2:].tolist() == [0, 0] and ni[2:].tolist() == [0, 0]


def test_finalize_width_eos_pad_and_return_order():
    S, max_new, eos, pad = 2, 5, 9, 7
    h = G.BeamHypotheses(3, 1.0, False)
    for hyp, s in (([1, 2, 3], -1.0), ([1, 2, 3, 4], -1.0), ([1, 2, 5, 6, 4, 4, 4], -0.5)):
        h.beams.append((s, np.array(hyp)))
    dec, sc = G.beam_finalize([h], np.array([True]), np.zeros((3, 7), np.int64), np.zeros(3, np.float32), S, S + max_new,
                              3, pad, eos)
    # best first; among the equal scores the later insertion first; width = min(7 + 1, 7); pad fill (lengths differ)
    assert sc.tolist() == [-0.5, -1.0, -1.0]
    assert dec.tolist() == [[1, 2, 5, 6, 4, 4, 4], [1, 2, 3, 4, eos, pad, pad], [1, 2, 3, eos, pad, pad, pad]]
    h = G.BeamHypotheses(2, 1.0, False)
    for hyp in ([1, 2, 3], [1, 2, 4]):
        h.beams.append((-1.0, np.array(hyp)))
    dec, _ = G.beam_finalize([h], np.array([True]), np.zeros((2, 3), np.int64), np.zeros(2, np.float32), S, S + max_new,
                             2, pad, eos)
    assert dec.tolist() == [[1, 2, 4, eos], [1, 2, 3, eos]]  # equal lengths: zero fill, all overwritten


def test_diversity_sibling_ranks():
    g = np.random.default_rng(0)
    V, nb = 16, 2
    logits = g.standard_normal((nb, V)).astype(np.float32)
    bs = np.array([0.0, -0.3], np.float32)
    sc, tk, bm, _ = G.beam_step(logits, bs, None, nb, diversity_rate=10.0)
    s = G.beam_step_scores(logits, bs, None)
    order = [np.lexsort((np.arange(V), -s[j])) for j in range(nb)]
    # rank r costs r * 10: both rows' best come first (higher score first), then both rows' second best
    first = sorted(range(nb), key=lambda j: (-s[j, order[j][0]], j))
    second = sorted(range(nb), key=lambda j: (-s[j, order[j][1]], j))
    want = [(j, order[j][0]) for j in first] + [(j, order[j][1]) for j in second]
    assert list(zip(bm[0].tolist(), tk[0].tolist())) == want
    assert sc[0].tolist() == [s[j, t] for j, t in want]  # the scorer gets the undiversified scores
    sc0, tk0, bm0, _ = G.beam_step(logits, bs, None, nb)
    flat = s.reshape(-1)
    top = np.lexsort((np.arange(nb * V), -flat))[:2 * nb]
    assert tk0[0].tolist() == (top % V).tolist() and bm0[0].tolist() == (top // V).tolist()


def _scripted_run(B, nb, V, S, max_new, eos, pad, early, lp, seed):
    """The oracle's loop, also recording the device-format tables (tokens, local parents)."""
    g = np.random.default_rng(seed)
    prompt = g.integers(0, V, (B, S))
    ids = np.repeat(prompt, nb, 0)
    beam_scores = np.zeros((B, nb), np.float32)
    beam_scores[:, 1:] = G.BEAM_INIT
    beam_scores = beam_scores.reshape(-1)
    hyps = [G.BeamHypotheses(nb, lp, early) for _ in range(B)]
    done = np.zeros(B, bool)
    tokens = np.zeros((max_new, B * nb), np.int64)
    parents = np.zeros((max_new, B * nb), np.int32)
    steps = 0
    for t in range(max_new):
        logits = g.standard_normal((B * nb, V)).astype(np.float32) * 2
        logits[:, eos] += g.uniform(0, 3, B * nb).astype(np.float32)  # eos shows up often
        was_done = done.copy()
        sc, tk, bm, _ = G.beam_step(logits, beam_scores, None, nb)
        beam_scores, nt, ni = G.beam_process(hyps, done, ids, sc, tk, bm, t, eos, pad)
        ids = np.concatenate([ids[ni], nt[:, None]], 1)
        tokens[t] = nt
        parents[t] = np.where(np.repeat(was_done, nb), 0, ni - np.repeat(np.arange(B), nb) * nb)
        steps += 1
        if done.all():
            break
    return prompt, ids, beam_scores, hyps, done, tokens, parents, steps


@pytest.mark.parametrize("early,lp,seed", [(False, 1.0, 0), (True, 1.0, 1), (False, 0.6, 2), (False, 2.0, 3)])
def test_host_finalize_matches_oracle(early, lp, seed):
    from paddlemix_b200.beam_search import finalize_tables
    B, nb, V, S, max_new, eos, pad = 3, 3, 12, 4, 9, 5, 11
    prompt, ids, beam_scores, hyps, done, tokens, parents, steps = _scripted_run(B, nb, V, S, max_new, eos, pad, early,
                                                                                 lp, seed)
    assert any(len(h.beams) for h in hyps)
    # the device's hypothesis store: (score, generated length, the slot whose history it is) in insertion order
    hs, hst, hsl = np.zeros((B, nb)), np.zeros((B, nb), np.int32), np.zeros((B, nb), np.int32)

    def backtrack(b, length, slot):
        seq = []
        for s in range(length - 1, -1, -1):
            seq.append(tokens[s, b * nb + slot])
            slot = parents[s, b * nb + slot]
        return seq[::-1]

    for b, h in enumerate(hyps):
        for i, (score, hyp) in enumerate(h.beams):
            length = len(hyp) - S
            slot = next(j for j in range(nb) if backtrack(b, length, j) == hyp[S:].tolist())
            hs[b, i], hst[b, i], hsl[b, i] = score, length, slot
    from paddlemix_b200.beam_search import resolve_beam_search_args
    args = resolve_beam_search_args(num_beams=nb, num_return_sequences=2, length_penalty=lp, early_stopping=early,
                                    eos_token_id=eos, pad_token_id=pad)
    got, got_s = finalize_tables(torch.from_numpy(prompt), torch.from_numpy(tokens), torch.from_numpy(parents),
                                 torch.from_numpy(beam_scores), torch.from_numpy(hs), torch.from_numpy(hst),
                                 torch.from_numpy(hsl), torch.tensor([len(h.beams) for h in hyps], dtype=torch.int32),
                                 torch.tensor([h.worst_score for h in hyps], dtype=torch.float64),
                                 torch.from_numpy(done.astype(np.int32)), steps, max_new, args)
    want, want_s = G.beam_finalize(hyps, done, ids, beam_scores, S, S + max_new, 2, pad, eos)
    assert np.array_equal(got.numpy(), want), (got, want)
    assert np.array_equal(got_s.numpy(), want_s)
