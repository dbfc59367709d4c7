"""Decoding on the CPU: the oracle's Philox and logits processors on hand-built rows, and generate()'s argument checks
(paddlemix_b200.sampling.resolve_generation_args, which needs no device)."""
import numpy as np
import pytest
import torch

from oracle import generation as G


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox4x32_10_known_answers(ctr, key, want):
    """Random123's kat_vectors for philox4x32-10."""
    assert tuple(int(x) for x in G.philox4x32_10(ctr, key)) == want


def test_uniform_is_per_row_and_step():
    u = G.uniform(1234, 0, np.arange(4))
    assert ((u >= 0) & (u < 1)).all() and len(set(u.tolist())) == 4
    assert not np.array_equal(u, G.uniform(1234, 1, np.arange(4)))
    assert np.array_equal(u, G.uniform(1234, 0, np.arange(4)))


def test_repetition_penalty_sign_rule():
    logits = np.array([[2.0, -2.0, 3.0, -1.0]], dtype=np.float32)
    seen = np.array([[True, True, False, False]])
    out = G.repetition_penalty(logits, seen, 2.0)
    assert out.tolist() == [[1.0, -4.0, 3.0, -1.0]]  # positive / p, negative * p, unseen ids unchanged


def test_top_k_keeps_ties():
    probs = np.array([[0.3, 0.2, 0.2, 0.2, 0.1]], dtype=np.float32)
    assert (G.top_k_process(probs, 2) > 0).tolist() == [[True, True, True, True, False]]
    assert np.array_equal(G.top_k_process(probs, 0), probs)  # top_k = 0 disables it
    assert (G.top_k_process(probs, 99) > 0).all()


def test_top_p_keeps_first_token_and_ranks_ties_by_id():
    probs = np.array([[0.9, 0.05, 0.05], [0.25, 0.25, 0.25]], dtype=np.float32)
    keep = G.top_p_keep(probs, 0.01)
    assert keep[0].tolist() == [True, False, False]  # the first token is kept even though it exceeds top_p
    keep = G.top_p_keep(np.array([[0.25, 0.25, 0.25, 0.25]], dtype=np.float32), 0.5)
    assert keep[0].tolist() == [True, True, True, False]  # masses above: 0, .25, .5 <= .5, .75; lower ids first


def test_top_p_works_on_top_k_output_without_renormalising():
    probs = np.array([[0.4, 0.3, 0.2, 0.1]], dtype=np.float32)
    topk = G.top_k_process(probs, 2)  # [0.4, 0.3, 0, 0]
    assert G.top_p_keep(topk, 0.5)[0, :2].tolist() == [True, True]  # mass above id 1 is 0.4 <= 0.5
    renorm = topk / topk.sum()  # [0.571, 0.429]: renormalising would drop id 1
    assert G.top_p_keep(renorm, 0.5)[0, :2].tolist() == [True, False]


def test_draw_is_inverse_cdf_over_kept_mass():
    probs = np.array([[0.5, 0.25, 0.25]] * 3, dtype=np.float32)
    keep = np.array([[True, True, False]] * 3)  # kept mass 0.75
    tok, near = G.draw(probs, keep, np.array([0.0, 0.5, 0.99]))
    assert tok.tolist() == [0, 0, 1]  # targets 0, 0.375, 0.7425 against prefixes 0.5, 0.75
    assert not near.any()
    _, near = G.draw(probs, keep, np.array([2.0 / 3.0]))  # target 0.5: on the boundary
    assert near.all()


def test_eos_any_of_and_pad_filling():
    unfinished = np.array([True, True, True, False])
    out = G.get_unfinished_flag(np.array([7, 9, 3, 5]), unfinished, [7, 9])
    assert out.tolist() == [False, False, True, False]
    # a loop: row 0 emits 7 at step 0, row 1 emits 9 at step 2; finished rows continue with pad
    V = 16
    script = {0: [7, 1], 1: [2, 3], 2: [4, 9]}

    def logits_fn(step, last):
        l = np.zeros((2, V), dtype=np.float32)
        for b, t in enumerate(script.get(step, [0, 0])):
            l[b, t] = 10.0
        return l

    ids, presence, finished, _ = G.generate(logits_fn, np.array([[1, 2], [3, 4]]), 10, V, eos_token_id=[7, 9],
                                            pad_token_id=0)
    assert ids.tolist() == [[1, 2, 7, 0, 0], [3, 4, 1, 3, 9]]  # stops at the step where the last row finished
    assert finished.all() and presence[0, 0] and presence[1, 9]


def test_generation_args():
    from paddlemix_b200.sampling import presence_bitmap, resolve_generation_args as R
    a = R()
    assert not a.on_device and not a.do_sample and a.top_k == 50
    assert not R(eos_token_id=5).on_device and R(eos_token_id=5).pad_token_id == 5
    assert R(do_sample=True).do_sample and R(decode_strategy="sampling").do_sample
    assert R(repetition_penalty=1.05).on_device and R(eos_token_id=[1, 2], pad_token_id=0).on_device
    assert R(eos_token_id=5, pad_token_id=3).on_device
    with pytest.raises(NotImplementedError):
        R(decode_strategy="beam_search")
    for bad in (dict(top_p=0.0), dict(top_p=1.5), dict(temperature=0.0), dict(temperature=-1.0),
                dict(repetition_penalty=0.0), dict(top_k=-1), dict(eos_token_id=[1, 2]), dict(decode_strategy="x")):
        with pytest.raises(ValueError):
            R(**bad)
    bm = presence_bitmap(torch.tensor([[0, 33, 33, 63], [31, 5, 5, 5]]), 64)
    assert bm.dtype == torch.int32 and bm.shape == (2, 2)
    assert bm[0].tolist() == [1, (1 << 1) | -(1 << 31)] and bm[1].tolist() == [-(1 << 31) | (1 << 5), 0]
