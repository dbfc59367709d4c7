"""Qwen2-VL prefill parity on the GPU: paddlemix_b200.qwen2_vl against the CPU fp32 oracle (itself cross-checked
against HF transformers in tests/test_oracle_qwen2vl_vs_hf.py). Stated tolerance (bf16 pipeline vs fp32): cosine
>= 0.999 on the logits and max |err| <= 4 % of the logit range."""
import pytest
import torch

from oracle import qwen2vl as O

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


def _inputs(cfg, grid, n_text, seed=0):
    g = torch.Generator().manual_seed(seed)
    m2 = cfg["vision"]["spatial_merge_size"] ** 2
    T = sum(t * h * w for t, h, w in grid)
    pv = torch.randn(T, 3 * 2 * 14 * 14, generator=g).to(bf16).float()
    rows = []
    for (t, h, w), nt in zip(grid, n_text):
        rows.append([cfg["vision_start_token_id"]] + [cfg["image_token_id"]] * (t * h * w // m2) +
                    [cfg["vision_end_token_id"]] + torch.randint(0, 1000, (nt,), generator=g).tolist())
    return torch.tensor(rows), pv


@pytest.mark.parametrize("grid,n_text", [([[1, 8, 8], [1, 4, 8]], [20, 28]), ([[1, 16, 16]], [62])])
def test_qwen2vl_tiny_prefill_parity(grid, n_text):
    from paddlemix_b200.qwen2_vl import Qwen2VLForConditionalGeneration
    cfg = O.QWEN2VL_CONFIGS["tiny"]
    P = O.init_qwen2vl_params(cfg, seed=1)
    model = Qwen2VLForConditionalGeneration(cfg).load_state_dict(P, device=0)
    assert model.state_dict_shapes() == O.qwen2vl_param_shapes(cfg)
    input_ids, pv = _inputs(cfg, grid, n_text)
    ref = O.qwen2vl_prefill(cfg, P, input_ids, pv, grid)
    out = model(input_ids=input_ids, attention_mask=torch.ones_like(input_ids), pixel_values=pv.cuda(),
                image_grid_thw=torch.tensor(grid))
    assert out.logits.shape == ref.shape and out.logits.dtype == torch.float32
    o = out.logits.cpu()
    cos = torch.nn.functional.cosine_similarity(o.flatten(), ref.flatten(), dim=0).item()
    err = (o - ref).abs().max().item() / ref.abs().max().item()
    assert cos >= 0.999 and err <= 0.04, (cos, err)
    pos_o, d_o = O.get_rope_index(cfg, input_ids, grid)
    pos_m, d_m = model.get_rope_index(input_ids, torch.tensor(grid))
    assert torch.equal(pos_o, pos_m) and torch.equal(d_o, d_m)  # integer index math: bit-exact
    # text-only prefill (no image): 1-D RoPE degenerates from M-RoPE
    ids2 = input_ids[:, -16:].contiguous()
    ref2 = O.qwen2vl_prefill(cfg, P, ids2, None, None, position_ids=torch.arange(16).reshape(1, 1, -1).expand(3, ids2.shape[0], -1))
    out2 = model(input_ids=ids2).logits.cpu()
    assert torch.nn.functional.cosine_similarity(out2.flatten(), ref2.flatten(), dim=0).item() >= 0.999


def test_qwen2vl_kv_cache_decode_matches_full_recompute():
    """Decode phase (SURVEY.md §8(f) rank 4): prefill with use_cache, then single-token steps against the KV cache
    (M-RoPE position = past length + rope_delta, modeling_qwen2_vl.py:1413-1441). A cached step is algebraically the
    last row of a full causal forward over the extended sequence, so each step's logits are compared with the fp32
    oracle's prefill of the extended ids; greedy generate() must reproduce the argmax chain."""
    from paddlemix_b200.qwen2_vl import Qwen2VLForConditionalGeneration
    cfg = O.QWEN2VL_CONFIGS["tiny"]
    P = O.init_qwen2vl_params(cfg, seed=2)
    model = Qwen2VLForConditionalGeneration(cfg).load_state_dict(P, device=0)
    grid = [[1, 8, 8], [1, 8, 8]]
    input_ids, pv = _inputs(cfg, grid, [14, 14], seed=3)
    B, S = input_ids.shape
    out = model(input_ids=input_ids, pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid), use_cache=True)
    cache, deltas = out.past_key_values, out.rope_deltas
    assert cache.get_seq_length() == S
    ref = O.qwen2vl_prefill(cfg, P, input_ids, pv, grid)
    assert torch.nn.functional.cosine_similarity(out.logits.cpu().flatten(), ref.flatten(), dim=0).item() >= 0.999
    g = torch.Generator().manual_seed(5)
    ids = input_ids
    for step in range(4):
        new = torch.randint(0, 1000, (B, 1), generator=g)  # teacher-forced continuation
        ids = torch.cat([ids, new], 1)
        step_out = model(input_ids=new, past_key_values=cache, rope_deltas=deltas, use_cache=True)
        assert step_out.logits.shape == (B, 1, cfg["vocab_size"]) and cache.get_seq_length() == S + step + 1
        ref = O.qwen2vl_prefill(cfg, P, ids, pv, grid)[:, -1]
        o = step_out.logits[:, 0].cpu()
        cos = torch.nn.functional.cosine_similarity(o.flatten(), ref.flatten(), dim=0).item()
        err = (o - ref).abs().max().item() / ref.abs().max().item()
        assert cos >= 0.999 and err <= 0.04, (step, cos, err)
    # greedy generate: the first new token is the prefill argmax, the next ones follow the model's own decode steps
    gen = model.generate(input_ids, pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid), max_new_tokens=3)
    assert gen.shape == (B, S + 3) and torch.equal(gen[:, :S], input_ids)
    first = model(input_ids=input_ids, pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid)).logits[:, -1].argmax(-1).cpu()
    assert torch.equal(gen[:, S], first)
    with pytest.raises(NotImplementedError):
        model(input_ids=input_ids[:, :2], past_key_values=cache, rope_deltas=deltas)  # decode takes one token per sequence


def test_graphed_decode_step_matches_eager_and_oracle():
    """GraphedDecodeStep (CUDA graph, device-side cache positions, GQA rows folded into one attention tile, skinny-M
    weight-streaming GEMMs) must reproduce the eager decode steps and the oracle's full recompute."""
    from paddlemix_b200.qwen2_vl import GraphedDecodeStep, Qwen2VLForConditionalGeneration
    cfg = O.QWEN2VL_CONFIGS["tiny"]
    P = O.init_qwen2vl_params(cfg, seed=6)
    model = Qwen2VLForConditionalGeneration(cfg).load_state_dict(P, device=0)
    grid = [[1, 8, 8], [1, 8, 8], [1, 8, 8]]
    input_ids, pv = _inputs(cfg, grid, [10, 10, 10], seed=7)
    B, S = input_ids.shape
    model.cache_headroom = 16
    out_a = model(input_ids=input_ids, pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid), use_cache=True)
    out_b = model(input_ids=input_ids, pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid), use_cache=True)
    stepper = GraphedDecodeStep(model, out_b.past_key_values, out_b.rope_deltas)
    g = torch.Generator().manual_seed(8)
    ids = input_ids
    for step in range(5):
        new = torch.randint(0, 1000, (B, 1), generator=g)
        ids = torch.cat([ids, new], 1)
        eager = model(input_ids=new, past_key_values=out_a.past_key_values, rope_deltas=out_a.rope_deltas, use_cache=True).logits[:, 0]
        graphed = stepper.step(new.reshape(-1)).clone()
        assert out_b.past_key_values.get_seq_length() == S + step + 1
        assert torch.equal(graphed, eager), step  # one decode body: the same kernels on the same inputs
        ref = O.qwen2vl_prefill(cfg, P, ids, pv, grid)[:, -1]
        o = graphed.cpu()
        cos = torch.nn.functional.cosine_similarity(o.flatten(), ref.flatten(), dim=0).item()
        assert cos >= 0.999 and (o - ref).abs().max().item() <= 0.04 * ref.abs().max().item(), (step, cos)
    # greedy generate (no eos): the graphed continuation equals a host loop of eager decode steps token for token
    gen = model.generate(input_ids, pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid), max_new_tokens=6)
    out = model(input_ids=input_ids, pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid), use_cache=True)
    toks = [out.logits[:, -1].argmax(-1).cpu()]
    for _ in range(5):
        toks.append(model(input_ids=toks[-1][:, None], past_key_values=out.past_key_values, rope_deltas=out.rope_deltas,
                          use_cache=True).logits[:, 0].argmax(-1).cpu())
    assert gen.shape == (B, S + 6) and torch.equal(gen, torch.cat([input_ids, torch.stack(toks, 1)], 1))


def _padded(cfg, grid, n_text, side, seed=7):
    """Sequences of different lengths padded to one length: ids [B, S], attention_mask [B, S], pixel values."""
    g = torch.Generator().manual_seed(seed)
    m2 = cfg["vision"]["spatial_merge_size"] ** 2
    T = sum(t * h * w for t, h, w in grid)
    pv = torch.randn(T, 3 * 2 * 14 * 14, generator=g)
    seqs = [[cfg["vision_start_token_id"]] + [cfg["image_token_id"]] * (t * h * w // m2) + [cfg["vision_end_token_id"]] +
            torch.randint(0, 1000, (nt,), generator=g).tolist() for (t, h, w), nt in zip(grid, n_text)]
    S = max(len(x) for x in seqs)
    ids, am = torch.zeros(len(seqs), S, dtype=torch.long), torch.zeros(len(seqs), S, dtype=torch.long)
    for i, x in enumerate(seqs):
        sl = slice(S - len(x), S) if side == "left" else slice(0, len(x))
        ids[i, sl], am[i, sl] = torch.tensor(x), 1
    return ids, am, pv


@pytest.mark.parametrize("side", ["left", "right"])
def test_qwen2vl_padded_batch_prefill_parity(side):
    """attention_mask with zeros (modeling_qwen2_vl.py:403-444,604-607): causal + key-padding additive mask through
    b200mix_sdpa and mask-aware M-RoPE indices; the rows of real tokens match the oracle (itself checked against HF
    transformers on padded batches)."""
    from paddlemix_b200.qwen2_vl import Qwen2VLForConditionalGeneration
    cfg = O.QWEN2VL_CONFIGS["tiny"]
    P = O.init_qwen2vl_params(cfg, seed=1)
    model = Qwen2VLForConditionalGeneration(cfg).load_state_dict(P, device=0)
    grid = [[1, 8, 8], [1, 4, 8], [1, 8, 8]]
    ids, am, pv = _padded(cfg, grid, [40, 9, 150], side)
    ref = O.qwen2vl_prefill(cfg, P, ids, pv, grid, attention_mask=am)
    out = model(input_ids=ids, attention_mask=am, pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid)).logits.cpu()
    keep = am.bool()
    o, r = out[keep], ref[keep]
    cos = torch.nn.functional.cosine_similarity(o.flatten(), r.flatten(), dim=0).item()
    err = (o - r).abs().max().item() / r.abs().max().item()
    assert cos >= 0.999 and err <= 0.04, (cos, err)
    pos_o, d_o = O.get_rope_index(cfg, ids, grid, am)
    pos_m, d_m = model.get_rope_index(ids, torch.tensor(grid), None, am)
    assert torch.equal(pos_o, pos_m) and torch.equal(d_o, d_m)


def test_qwen2vl_left_padded_decode_matches_full_recompute():
    """Decode after a LEFT-padded prompt batch: the cache keeps the padding, every step masks it (eager step and the
    CUDA-graph step), logits = the oracle's full recompute of the extended, still padded, batch."""
    from paddlemix_b200.qwen2_vl import GraphedDecodeStep, Qwen2VLForConditionalGeneration
    cfg = O.QWEN2VL_CONFIGS["tiny"]
    P = O.init_qwen2vl_params(cfg, seed=2)
    model = Qwen2VLForConditionalGeneration(cfg).load_state_dict(P, device=0)
    grid = [[1, 8, 8], [1, 4, 8]]
    ids, am, pv = _padded(cfg, grid, [30, 12], "left")
    B, S = ids.shape

    def check(o, ids_ext, am_ext, what):
        ref = O.qwen2vl_prefill(cfg, P, ids_ext, pv, grid, attention_mask=am_ext)[:, -1]
        cos = torch.nn.functional.cosine_similarity(o.flatten(), ref.flatten(), dim=0).item()
        err = (o - ref).abs().max().item() / ref.abs().max().item()
        assert cos >= 0.999 and err <= 0.04, (what, cos, err)

    g = torch.Generator().manual_seed(9)
    news = [torch.randint(0, 1000, (B, 1), generator=g) for _ in range(4)]
    # eager steps
    out = model(input_ids=ids, attention_mask=am, pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid), use_cache=True)
    cache, deltas = out.past_key_values, out.rope_deltas
    check(out.logits[:, -1].cpu(), ids, am, "prefill")
    ids_e, am_e = ids, am
    for i, new in enumerate(news[:2]):
        ids_e, am_e = torch.cat([ids_e, new], 1), torch.cat([am_e, torch.ones(B, 1, dtype=torch.long)], 1)
        o = model(input_ids=new, attention_mask=am_e, past_key_values=cache, rope_deltas=deltas, use_cache=True).logits[:, 0].cpu()
        check(o, ids_e, am_e, f"eager step {i}")
    # graphed steps continue from the same cache
    stepper = GraphedDecodeStep(model, cache, deltas)
    for i, new in enumerate(news[2:]):
        ids_e, am_e = torch.cat([ids_e, new], 1), torch.cat([am_e, torch.ones(B, 1, dtype=torch.long)], 1)
        o = stepper.step(new.reshape(-1)).float().cpu()
        check(o, ids_e, am_e, f"graphed step {i}")
    gen = model.generate(ids, pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid), max_new_tokens=3, attention_mask=am)
    assert gen.shape == (B, S + 3) and torch.equal(gen[:, :S], ids)
    with pytest.raises(ValueError):
        model.generate(ids.flip(1), max_new_tokens=2, attention_mask=am.flip(1))  # right-padded prompts are refused
