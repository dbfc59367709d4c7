"""The shared decoder stack (paddlemix_b200/decoder.py) as Qwen2-VL runs it: eager forward() decode and the CUDA-graph
decode step are the same kernels on the same inputs, so they agree bit for bit; greedy generate() (graph replays) equals a
host loop of eager decode steps, with and without an eos."""
import pytest
import torch

from oracle import qwen2vl as O

pytestmark = pytest.mark.gpu


def _tiny_model(seed):
    from paddlemix_b200.qwen2_vl import Qwen2VLForConditionalGeneration
    cfg = O.QWEN2VL_CONFIGS["tiny"]
    return cfg, Qwen2VLForConditionalGeneration(cfg).load_state_dict(O.init_qwen2vl_params(cfg, seed=seed), device=0)


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


def test_eager_decode_equals_graphed_step():
    from paddlemix_b200 import ops
    from paddlemix_b200.qwen2_vl import GraphedDecodeStep
    cfg, model = _tiny_model(10)
    grid = [[1, 8, 8], [1, 4, 8], [1, 8, 8]]
    ids, am, pv = _padded(cfg, grid, [20, 9, 14])
    B, S = ids.shape
    model.cache_headroom = 8
    kw = dict(input_ids=ids, attention_mask=am, pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid), use_cache=True)
    a, b = model(**kw), model(**kw)
    assert torch.equal(a.logits, b.logits)
    stepper = GraphedDecodeStep(model, b.past_key_values, b.rope_deltas)
    g = torch.Generator().manual_seed(11)
    for step in range(4):
        new = torch.randint(0, 1000, (B, 1), generator=g)
        n0 = ops.launches()
        eager = model(input_ids=new, past_key_values=a.past_key_values, rope_deltas=a.rope_deltas, use_cache=True).logits
        assert ops.launches() - n0 == stepper.launches_per_step  # the same kernel sequence
        graphed = stepper.step(new.reshape(-1))
        assert eager.shape == (B, 1, cfg["vocab_size"]) and torch.equal(eager[:, 0], graphed), step
        for ca, cb in ((a.past_key_values.k, b.past_key_values.k), (a.past_key_values.v, b.past_key_values.v)):
            assert all(torch.equal(x[:, :S + step + 1], y[:, :S + step + 1]) for x, y in zip(ca, cb)), step
    assert a.past_key_values.length == b.past_key_values.length == S + 4


def _greedy_host_loop(model, kw, max_new, eos):
    """Prefill, then eager forward() decode steps with the argmax; finished rows are not padded; stops once every row
    has produced `eos`."""
    model.cache_headroom = max_new
    out = model(**kw, use_cache=True)
    toks = [out.logits[:, -1].argmax(-1).cpu()]
    done = toks[0] == eos
    while len(toks) < max_new and not bool(done.all()):
        o = model(input_ids=toks[-1][:, None], past_key_values=out.past_key_values, rope_deltas=out.rope_deltas,
                  use_cache=True)
        toks.append(o.logits[:, 0].argmax(-1).cpu())
        done |= toks[-1] == eos
    return torch.cat([kw["input_ids"], torch.stack(toks, 1)], 1)


def test_greedy_generate_with_eos_equals_host_loop():
    cfg, model = _tiny_model(11)
    grid = [[1, 8, 8], [1, 4, 8]]
    ids, am, pv = _padded(cfg, grid, [20, 9])
    S, max_new = ids.shape[1], 32
    kw = dict(input_ids=ids, attention_mask=am, pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid))

    def generate(eos):
        return model.generate(ids, pixel_values=kw["pixel_values"], image_grid_thw=kw["image_grid_thw"], attention_mask=am,
                              max_new_tokens=max_new, eos_token_id=eos)
    free = generate(None)
    assert torch.equal(generate(-1), free) and torch.equal(_greedy_host_loop(model, kw, max_new, -1), free)
    new = free[:, S:]
    # tokens both rows produce, first at different steps: the result ends at the later one (before max_new_tokens)
    both = [t for t in new.unique().tolist() if bool((new == t).any(1).all())]
    ends = {t: [int((row == t).int().argmax()) for row in new] for t in both}
    ends = {t: e for t, e in ends.items() if e[0] != e[1]}
    assert ends, new
    for eos in [int(new[0, 2])] + sorted(ends, key=lambda t: max(ends[t]))[:3]:
        want = _greedy_host_loop(model, kw, max_new, eos)
        got = generate(eos)
        assert torch.equal(got, want), (eos, got[:, S:], want[:, S:])
        assert torch.equal(got, free[:, :got.shape[1]])


def test_generate_one_or_zero_new_tokens_builds_no_decode_step(monkeypatch):
    from paddlemix_b200.qwen2_vl import modeling_qwen2_vl as M
    cfg, model = _tiny_model(12)
    grid = [[1, 8, 8], [1, 4, 8]]
    ids, am, pv = _padded(cfg, grid, [12, 9])
    first = model(input_ids=ids, attention_mask=am, pixel_values=pv.cuda(),
                  image_grid_thw=torch.tensor(grid)).logits[:, -1].argmax(-1).cpu()
    want = torch.cat([ids, first[:, None]], 1)

    class NoDecodeStep:
        def __init__(self, *args, **kwargs):
            raise AssertionError("generate() built a decode step it has no token for")
    monkeypatch.setattr(M, "GraphedDecodeStep", NoDecodeStep)
    for n in (1, 0):
        for eos in (None, -1, int(first[0])):
            got = model.generate(ids, pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid), attention_mask=am,
                                 max_new_tokens=n, eos_token_id=eos)
            assert torch.equal(got, want), (n, eos)
