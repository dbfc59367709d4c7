"""Whole-model parity against the CPU fp32 oracle AT THE BASELINE SHAPES (BASELINE.json configs[1..4]), not only at the
tiny configurations:

  C2  SDXL-base UNet2DConditionModel (2.57 B params), latent 128x128 (1024^2), 77 x 2048 context, B = 1 and B = 2
      (unet_2d_condition.py:809-1207)
  C3  SD3-medium MMDiT, 24 layers, 4096 image + 154 text tokens, B = 1 (transformer_sd3.py:279-365)
  C4  Qwen2-VL-7B shapes (hidden 3584, 28 / 4 heads x 128, MLP 18944, vocab 152064; ViT 1280 / 16 x 80 / MLP 5120) with
      the depth cut to 4 ViT blocks + 3 decoder layers, one 448x448 image + 512 text tokens = 768 tokens
      (modeling_qwen2_vl.py:1382-1503) -- the full 28 + 32 layers repeat the same layer 10x and would need ~35 GB of
      fp32 oracle weights
  C5  STDiT2-XL shapes (hidden 1152, 16 heads x 72), depth cut to 3 blocks, 16 frames x 32x32 patches = 16 x 1024
      tokens, 120 text tokens, B = 1 (stdit2.py:334-448)

Stated tolerance (bf16 kernels vs fp32 oracle, every activation rounded to bf16 after each fused op): cosine >= 0.999
and max |err| <= 4 % of the output's max magnitude -- the same bar as the tiny-config tests. Each test appends its
(cosine, max-rel) to a JSON record (see _record) so the numbers can be quoted.
The oracle needs 10-40 s per forward on the GPU box's host cores; marked `slow`.
"""
import json
import os

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.slow]
bf16 = torch.bfloat16
COS_MIN, ERR_MAX = 0.999, 0.04


def _record(name, cos, err, extra=None):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    path = os.path.join(root, "gpurun_out", "parity_baseline.json")
    os.makedirs(os.path.dirname(path), exist_ok=True)
    try:
        with open(path) as f:
            d = json.load(f)
    except Exception:
        d = {}
    d[name] = {"cosine": round(cos, 6), "max_rel_err": round(err, 5), "tolerance": {"cosine_min": COS_MIN, "max_rel_err": ERR_MAX},
               **(extra or {})}
    with open(path, "w") as f:
        json.dump(d, f, indent=1)


def _compare(out, ref, name, extra=None):
    o, r = out.float().cpu(), ref.float()
    assert o.shape == r.shape and torch.isfinite(o).all()
    cos = torch.nn.functional.cosine_similarity(o.flatten().double(), r.flatten().double(), dim=0).item()
    err = (o - r).abs().max().item() / r.abs().max().item()
    _record(name, cos, err, extra)
    assert cos >= COS_MIN and err <= ERR_MAX, (name, cos, err)
    return cos, err


@pytest.mark.parametrize("B", [1, 2])
def test_sdxl_c2_unet_vs_oracle(B):
    from oracle import unet as O
    from paddlemix_b200.ppdiffusers.unet_2d_condition import UNet2DConditionModel
    cfg = O.UNET_CONFIGS["sdxl"]
    P = O.init_params(O.unet_param_shapes(cfg), seed=1)
    keys = ("in_channels", "out_channels", "flip_sin_to_cos", "freq_shift", "down_block_types", "up_block_types",
            "block_out_channels", "layers_per_block", "norm_num_groups", "norm_eps", "cross_attention_dim",
            "transformer_layers_per_block", "attention_head_dim", "use_linear_projection", "addition_embed_type",
            "addition_time_embed_dim", "projection_class_embeddings_input_dim", "resnet_out_scale_factor")
    model = UNet2DConditionModel(**{k: cfg[k] for k in keys}).load_state_dict(P, device=0)
    g = torch.Generator().manual_seed(10 + B)
    H = 128
    x = torch.randn(B, 4, H, H, generator=g).to(bf16).float()
    ctx = torch.randn(B, 77, 2048, generator=g).to(bf16).float()
    added = {"text_embeds": torch.randn(B, 1280, generator=g).to(bf16).float(),
             "time_ids": torch.tensor([[1024., 1024., 0, 0, 1024., 1024.]] * B)}
    t = torch.tensor([981, 521][:B])  # per-sample timesteps: batch elements are not interchangeable
    out = model(x.cuda(), t.cuda(), ctx.cuda(), added_cond_kwargs={k: v.cuda() for k, v in added.items()}).sample
    with torch.no_grad():
        ref = O.unet_forward(cfg, P, x, t, ctx, added)
    _compare(out, ref, f"C2_sdxl_unet_1024_B{B}", {"shape": list(ref.shape)})


def test_sd3_c3_mmdit_vs_oracle():
    from oracle import sd3 as O
    from paddlemix_b200.ppdiffusers.transformer_sd3 import SD3Transformer2DModel
    cfg = O.SD3_CONFIGS["sd3_medium"]
    P = O.init_sd3_params(cfg, seed=1)
    model = SD3Transformer2DModel(**cfg).load_state_dict(P, device=0)
    g = torch.Generator().manual_seed(3)
    B, H, L = 1, 128, 154
    x = torch.randn(B, 16, H, H, generator=g).to(bf16).float()
    ctx = torch.randn(B, L, cfg["joint_attention_dim"], generator=g).to(bf16).float()
    pooled = torch.randn(B, cfg["pooled_projection_dim"], generator=g).to(bf16).float()
    t = torch.full((B,), 637.5)
    out = model(hidden_states=x.cuda(), encoder_hidden_states=ctx.cuda(), pooled_projections=pooled.cuda(),
                timestep=t.cuda(), return_dict=False)[0]
    with torch.no_grad():
        ref = O.sd3_forward(cfg, P, x, ctx, pooled, t)
    _compare(out, ref, "C3_sd3_medium_mmdit_1024_B1", {"tokens": 4096 + L})


def test_qwen2vl_c4_shapes_vs_oracle():
    from oracle import qwen2vl as O
    from paddlemix_b200.qwen2_vl import Qwen2VLForConditionalGeneration
    cfg = dict(O.QWEN2VL_CONFIGS["qwen2vl_7b"])
    cfg["num_hidden_layers"] = 3
    cfg["vision"] = dict(cfg["vision"], depth=4)
    P = O.init_qwen2vl_params(cfg, seed=1)
    model = Qwen2VLForConditionalGeneration(cfg).load_state_dict(P, device=0)
    g = torch.Generator().manual_seed(4)
    grid = [[1, 32, 32]]  # 448 x 448 -> 1024 patches -> 256 merged tokens
    pv = torch.randn(1024, 1176, generator=g).to(bf16).float()
    ids = torch.tensor([[cfg["vision_start_token_id"]] + [cfg["image_token_id"]] * 256 + [cfg["vision_end_token_id"]] +
                        torch.randint(0, 151643, (510,), generator=g).tolist()])
    assert ids.shape == (1, 768)
    out = model(input_ids=ids, pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid)).logits
    with torch.no_grad():
        ref = O.qwen2vl_prefill(cfg, P, ids, pv, grid)
    _compare(out, ref, "C4_qwen2vl_7b_shapes_768tok_3of28_layers", {"vit_depth": 4, "llm_layers": 3, "logits": list(ref.shape)})


def test_stdit2_c5_shapes_vs_oracle():
    from oracle import stdit2 as O
    from paddlemix_b200.opensora import STDiT2
    cfg = dict(O.STDIT2_CONFIGS["stdit2_xl"])
    cfg["depth"] = 3
    P = O.init_stdit2_params(cfg, seed=1)
    model = STDiT2(cfg).load_state_dict(P, device=0)
    g = torch.Generator().manual_seed(5)
    B, T, H, L = 1, 16, 64, 120
    x = torch.randn(B, 4, T, H, H, generator=g).to(bf16).float()
    y = torch.randn(B, 1, L, cfg["caption_channels"], generator=g).to(bf16).float()
    kw = dict(num_frames=torch.tensor([16.]), height=torch.tensor([512.]), width=torch.tensor([512.]),
              ar=torch.tensor([1.]), fps=torch.tensor([24.]))
    mask = torch.ones(B, L, dtype=torch.long)
    mask[0, 97:] = 0
    ts = torch.tensor([500.])
    out = model(x.cuda(), ts.cuda(), y.cuda(), mask=mask.cuda(), **kw)
    with torch.no_grad():
        ref = O.stdit2_forward(cfg, P, x, ts, y, mask, **kw)
    _compare(out, ref, "C5_stdit2_xl_shapes_16x1024tok_3of28_layers", {"tokens": T * 1024, "text_tokens": L})
