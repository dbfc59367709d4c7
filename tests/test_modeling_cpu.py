"""paddlemix_b200.modeling without a GPU or the built library: the synthetic-weight rule and each model's exceptions to
it, the attention-head padding helpers, the Paddle-layout getters, and the missing-key check every load_state_dict
runs before any device work."""
import math
import sys
import types

import numpy as np
import pytest
import torch

import paddlemix_b200
from oracle import clip as OCL
from oracle import llama as OL
from oracle import qwen2vl as OQ
from oracle import sd3 as O3
from oracle import stdit2 as OS2
from oracle import unet as OU
from oracle import vae as OV
from paddlemix_b200.clip import CLIPTextModel, CLIPTextModelWithProjection, CLIPVisionModel
from paddlemix_b200.llava import LlamaForCausalLM, LlavaLlamaForCausalLM
from paddlemix_b200.modeling import (bind, linear_weight, pad_head_cols, pad_head_rows, pad_head_vec, pad_head_width,
                                     synthetic_state_dict)
from paddlemix_b200.opensora import STDiT2
from paddlemix_b200.ppdiffusers.autoencoder_kl import AutoencoderKL
from paddlemix_b200.ppdiffusers.controlnet import ControlNetModel
from paddlemix_b200.ppdiffusers.transformer_sd3 import SD3Transformer2DModel
from paddlemix_b200.ppdiffusers.unet_2d_condition import UNet2DConditionModel
from paddlemix_b200.qwen2_vl import Qwen2VLForConditionalGeneration

UNET_KEYS = ("in_channels", "out_channels", "down_block_types", "up_block_types", "block_out_channels",
             "layers_per_block", "cross_attention_dim", "transformer_layers_per_block", "attention_head_dim",
             "use_linear_projection", "addition_embed_type", "addition_time_embed_dim",
             "projection_class_embeddings_input_dim")
VAE_KEYS = ("latent_channels", "out_channels", "block_out_channels", "layers_per_block", "norm_num_groups",
            "scaling_factor")
BF16_ULP = 2.0 ** -7  # relative rounding of a bf16 value


def check_rule(name, shp, t):
    """t follows the synthetic rule: U(+-1/sqrt(fan_in)) matrices, 1 + 0.1 N norm scales, 0.05 N biases."""
    assert t.dtype == torch.bfloat16 and tuple(t.shape) == tuple(shp), name
    t = t.float()
    if name.endswith(".weight") and len(shp) >= 2:
        bound = 1.0 / math.sqrt(shp[0] if len(shp) == 2 else math.prod(shp[1:]))
        assert t.abs().max() <= bound * (1 + BF16_ULP), name
        if t.numel() >= 100:
            assert t.abs().max() > 0.8 * bound, name  # the bound is the one of this fan_in, not a smaller one
    elif name.endswith(".weight"):
        assert (t - 1).abs().max() < 0.6 and (t.numel() < 100 or abs(t.std() - 0.1) < 0.02), name
    else:
        assert t.abs().max() < 0.3 and (t.numel() < 100 or abs(t.std() - 0.05) < 0.01), name


def test_synthetic_rule_per_category_and_fan_in():
    shapes = {"lin.weight": (64, 48),                # Paddle Linear [in, out]: fan_in = 64
              "conv.weight": (8, 4, 3, 3),           # conv filter [out, in, kh, kw]: fan_in = 36
              "patch.weight": (16, 3, 2, 4, 4),      # Conv3D patch embed [out, in, kt, kh, kw]: fan_in = 96
              "norm.weight": (512,), "lin.bias": (512,), "table": (4, 128)}
    P = synthetic_state_dict(shapes, 7, "cpu")
    assert list(P) == sorted(shapes)
    for name, shp in shapes.items():
        check_rule(name, shp, P[name])


def test_synthetic_draw_order_and_seed():
    shapes = {"b.bias": (5,), "a.weight": (3, 2), "c.weight": (4,)}
    P = synthetic_state_dict(shapes, 11, "cpu")
    g = torch.Generator().manual_seed(11)  # one generator, names in sorted order
    a = ((torch.rand(3, 2, generator=g) * 2 - 1) / 3 ** 0.5).to(torch.bfloat16)
    b = (0.05 * torch.randn(5, generator=g)).to(torch.bfloat16)
    c = (1.0 + 0.1 * torch.randn(4, generator=g)).to(torch.bfloat16)
    assert torch.equal(P["a.weight"], a) and torch.equal(P["b.bias"], b) and torch.equal(P["c.weight"], c)
    again = synthetic_state_dict(shapes, 11, "cpu")
    assert all(torch.equal(P[k], again[k]) for k in shapes)
    assert not torch.equal(P["b.bias"], synthetic_state_dict(shapes, 12, "cpu")["b.bias"])


def test_synthetic_special_replaces_the_rule_with_the_same_generator():
    shapes = {"a.bias": (6,), "emb": (6,), "z.bias": (6,)}
    P = synthetic_state_dict(shapes, 3, "cpu", special=lambda n, s, randn: 2.0 * randn(s) if n == "emb" else None)
    g = torch.Generator().manual_seed(3)
    want = [0.05 * torch.randn(6, generator=g), 2.0 * torch.randn(6, generator=g), 0.05 * torch.randn(6, generator=g)]
    assert all(torch.equal(P[k], w.to(torch.bfloat16)) for k, w in zip(("a.bias", "emb", "z.bias"), want))


def _stdit2_tiny():
    return STDiT2(OS2.STDIT2_CONFIGS["tiny"])


# (model, seed, which tensors the model draws differently, their expected standard deviation)
SPECIAL_CASES = {
    "unet": (lambda: UNet2DConditionModel(**{k: OU.UNET_CONFIGS["tiny_sd"][k] for k in UNET_KEYS}), 1, None, None),
    "sd3": (lambda: SD3Transformer2DModel(**O3.SD3_CONFIGS["tiny"]), 3, lambda n: n == "pos_embed.pos_embed", 0.5),
    "stdit2": (_stdit2_tiny, 5, lambda n: "scale_shift_table" in n,
               1 / math.sqrt(OS2.STDIT2_CONFIGS["tiny"]["hidden_size"])),
    "clip_text": (lambda: CLIPTextModelWithProjection(OCL.CLIP_TEXT_CONFIGS["tiny"]), 1, lambda n: "embedding" in n, 0.3),
    "clip_vision": (lambda: CLIPVisionModel(OCL.CLIP_VISION_CONFIGS["tiny"]), 1, lambda n: "embedding" in n, 0.3),
    "qwen2vl": (lambda: Qwen2VLForConditionalGeneration(OQ.QWEN2VL_CONFIGS["tiny"]), 4,
                lambda n: n == "model.embed_tokens.weight", 0.5),
}


@pytest.mark.parametrize("case", sorted(SPECIAL_CASES))
def test_init_synthetic_weights_rule_and_model_exceptions(case, monkeypatch):
    make, seed, special, std = SPECIAL_CASES[case]
    model = make()
    monkeypatch.setattr(type(model), "load_state_dict", lambda self, P, device=0: P)
    P = model.init_synthetic_weights(seed=seed, device="cpu")
    shapes = model.state_dict_shapes()
    assert P.keys() == shapes.keys()
    n_special = 0
    for name, t in P.items():
        if special is not None and special(name):  # e.g. CLIP's patch filter: the embedding rule wins over the matrix one
            n_special += 1
            assert t.dtype == torch.bfloat16 and tuple(t.shape) == tuple(shapes[name]), name
            t = t.float()
            assert abs(t.std().item() / std - 1) < 0.2 and abs(t.mean().item()) < std / 2, name
        else:
            check_rule(name, shapes[name], t)
    assert n_special > 0 or special is None


def test_pad_head_width_boundaries():
    for d, p in ((1, 64), (40, 64), (64, 64), (65, 128), (72, 128), (80, 128), (128, 128), (129, 192), (160, 192),
                 (192, 192)):
        assert pad_head_width(d) == p, d
    with pytest.raises(ValueError, match="193"):
        pad_head_width(193)


@pytest.mark.parametrize("d,dp", [(40, 64), (80, 128), (64, 64)])
def test_pad_heads_keep_values_and_zero_the_padding(d, dp):
    H, K = 3, 5
    w = torch.arange(H * d * K, dtype=torch.float32).reshape(H * d, K) + 1
    rows = pad_head_rows(w, H, d, dp).reshape(H, dp, K)
    assert torch.equal(rows[:, :d], w.reshape(H, d, K)) and not rows[:, d:].any()
    cols = pad_head_cols(w.t().contiguous(), H, d, dp).reshape(K, H, dp)
    assert torch.equal(cols[:, :, :d], w.t().reshape(K, H, d)) and not cols[:, :, d:].any()
    b = torch.arange(H * d, dtype=torch.float32) + 1
    vec = pad_head_vec(b, H, d, dp).reshape(H, dp)
    assert torch.equal(vec[:, :d], b.reshape(H, d)) and not vec[:, d:].any()


def test_linear_weight_transposes_paddle_layout():
    P = {"fc.weight": np.arange(6, dtype=np.float16).reshape(2, 3)}  # Paddle Linear [in, out]
    w = linear_weight(P, "fc")
    assert w.dtype == torch.float32 and w.is_contiguous() and torch.equal(w, torch.tensor([[0., 3.], [1., 4.], [2., 5.]]))


@pytest.fixture
def fake_ops(monkeypatch):
    """Stands in for paddlemix_b200.ops (which loads the built library): records the devices init() is called with."""
    ops = types.SimpleNamespace(inits=[])
    ops.init = ops.inits.append
    monkeypatch.setitem(sys.modules, "paddlemix_b200.ops", ops)
    monkeypatch.setattr(paddlemix_b200, "ops", ops, raising=False)
    return ops


def _controlnet_tiny():
    cfg = OU.UNET_CONFIGS["tiny_sd"]
    keys = [k for k in UNET_KEYS if k not in ("out_channels", "up_block_types")]
    return ControlNetModel(**{k: cfg[k] for k in keys}, conditioning_embedding_out_channels=(16, 32))


LLM, VIS = OL.LLAMA_CONFIGS["tiny"], OCL.CLIP_VISION_CONFIGS["tiny"]
# (model, prefix of the key to remove)
MODELS = {
    "unet": (lambda: UNet2DConditionModel(**{k: OU.UNET_CONFIGS["tiny_sd"][k] for k in UNET_KEYS}), "mid_block."),
    "controlnet": (_controlnet_tiny, "controlnet_mid_block."),
    "vae": (lambda: AutoencoderKL(**{k: OV.VAE_CONFIGS["tiny"][k] for k in VAE_KEYS}), "decoder.mid_block."),
    "sd3": (lambda: SD3Transformer2DModel(**O3.SD3_CONFIGS["tiny"]), "norm_out."),
    "stdit2": (_stdit2_tiny, "blocks.1."),
    "clip_text": (lambda: CLIPTextModel(OCL.CLIP_TEXT_CONFIGS["tiny"]), "text_model.final_layer_norm."),
    "clip_vision": (lambda: CLIPVisionModel(VIS), "vision_model.post_layernorm."),
    "qwen2vl": (lambda: Qwen2VLForConditionalGeneration(OQ.QWEN2VL_CONFIGS["tiny"]), "visual.blocks.1."),
    "llama": (lambda: LlamaForCausalLM(LLM), "lm_head."),
    "llava": (lambda: LlavaLlamaForCausalLM(LLM, vision_config=VIS), LlavaLlamaForCausalLM.VT),
}


@pytest.mark.parametrize("case", sorted(MODELS))
def test_load_state_dict_names_a_missing_key_before_device_work(case, fake_ops):
    make, prefix = MODELS[case]
    model = make()
    shapes = model.state_dict_shapes()
    key = sorted(k for k in shapes if k.startswith(prefix))[-1]
    P = {k: None for k in shapes if k != key}  # the check looks at names only
    with pytest.raises(KeyError, match=key.replace(".", r"\.")):
        model.load_state_dict(P, device=0)
    assert fake_ops.inits == [] and model.device is None


def test_bind_resolves_the_device(fake_ops):
    model = _stdit2_tiny()
    P = dict.fromkeys(model.state_dict_shapes())
    assert bind(model, P, 3) == torch.device("cuda", 3) and model.device == torch.device("cuda", 3)
    assert bind(model, P, "cuda:2") == torch.device("cuda", 2)
    assert bind(model, P, "cpu") == torch.device("cpu") and model.device == torch.device("cpu")
    assert fake_ops.inits == [3, 2, 0]
