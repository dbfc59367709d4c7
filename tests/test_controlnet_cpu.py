"""ControlNet host logic without a GPU: parameter names / shapes against the oracle, from_unet's weight mapping, the
pipeline's keep table and guess-mode scales, constructor checks, and an oracle property (zero convs at zero give
residuals of exactly 0, which leave the UNet's output unchanged)."""
import pytest
import torch

from oracle import controlnet as OC
from oracle import unet as O
from paddlemix_b200.ppdiffusers.controlnet import (ControlNetModel, controlnet_keep, guess_mode_scales,
                                                  map_unet_state_dict)
from paddlemix_b200.ppdiffusers.unet_2d_condition import UNet2DConditionModel

UNET_KEYS = ("in_channels", "out_channels", "flip_sin_to_cos", "freq_shift", "down_block_types", "up_block_types",
             "block_out_channels", "layers_per_block", "norm_num_groups", "norm_eps", "cross_attention_dim",
             "transformer_layers_per_block", "attention_head_dim", "use_linear_projection", "addition_embed_type",
             "addition_time_embed_dim", "projection_class_embeddings_input_dim", "resnet_out_scale_factor")
CN_KEYS = tuple(k for k in UNET_KEYS if k not in ("out_channels", "up_block_types", "resnet_out_scale_factor"))
TINY_COND = (16, 32)  # a 2x conditioning embedding for the small test configs


def cn_cfg(name, **kw):
    return {**O.UNET_CONFIGS[name], **kw}


def controlnet(cfg):
    extra = {k: cfg[k] for k in ("conditioning_channels", "conditioning_embedding_out_channels",
                                 "controlnet_conditioning_channel_order") if k in cfg}
    return ControlNetModel(**{k: cfg[k] for k in CN_KEYS}, **extra)


@pytest.mark.parametrize("name,kw", [("sd15", {}), ("sdxl", {}), ("tiny_sd", {}), ("tiny_xl", {}),
                                     ("tiny_sd", dict(conditioning_embedding_out_channels=TINY_COND,
                                                      conditioning_channels=1))])
def test_state_dict_shapes_match_oracle(name, kw):
    cfg = cn_cfg(name, **kw)
    shapes = controlnet(cfg).state_dict_shapes()
    assert shapes == OC.controlnet_param_shapes(cfg)
    assert controlnet(cfg).num_residuals == len(OC.zero_conv_channels(cfg)) + 1


def test_residual_shapes_follow_the_encoder():
    cfg = cn_cfg("sdxl")
    m = controlnet(cfg)
    shapes = m.residual_shapes(128, 128)
    assert [c for _, _, c in shapes[:-1]] == OC.zero_conv_channels(cfg)
    assert shapes[0] == (128, 128, 320) and shapes[-1] == (32, 32, 1280)


def test_from_unet_name_mapping():
    cfg = O.UNET_CONFIGS["tiny_xl"]
    unet = UNet2DConditionModel(**{k: cfg[k] for k in UNET_KEYS})
    unet_P = O.init_params(O.unet_param_shapes(cfg), seed=3)
    cn = ControlNetModel.from_unet(unet, conditioning_embedding_out_channels=(16, 32, 96, 256), unet_state_dict=unet_P)
    assert cn.device is None  # a host-only UNet: nothing to load onto
    ref_cfg = {**cfg, "conditioning_embedding_out_channels": (16, 32, 96, 256)}
    shapes = cn.state_dict_shapes()
    assert shapes == OC.controlnet_param_shapes(ref_cfg)
    assert cn.config.addition_embed_type == "text_time" and cn.config.block_out_channels == cfg["block_out_channels"]
    cn_P = O.init_params(shapes, seed=4)
    mapped = {**cn_P, **map_unet_state_dict(shapes, unet_P)}
    ref = OC.from_unet_params(ref_cfg, unet_P, cn_P)
    assert mapped.keys() == ref.keys()
    assert all(torch.equal(mapped[k], ref[k]) for k in ref)
    copied = set(map_unet_state_dict(shapes, unet_P))
    assert "down_blocks.1.attentions.0.transformer_blocks.0.attn2.to_k.weight" in copied
    assert "mid_block.resnets.1.conv2.weight" in copied and "time_embedding.linear_2.bias" in copied
    assert not any(k.startswith(("add_embedding.", "controlnet_")) for k in copied)
    with pytest.raises(ValueError):
        ControlNetModel.from_unet(unet, device=0)  # load_weights_from_unet without the UNet's state dict


@pytest.mark.parametrize("n,start,end", [(10, [0.0], [1.0]), (7, [0.2], [0.6]), (9, [0.0, 0.3], [0.5, 1.0]),
                                         (4, [0.0], [0.0])])
def test_keep_table_matches_oracle(n, start, end):
    multi = len(start) > 1
    assert controlnet_keep(n, start, end, multi) == OC.controlnet_keep(n, start, end, multi)
    if end == [0.0]:
        assert controlnet_keep(n, start, end, multi) == [0.0] * n


@pytest.mark.parametrize("scale", [1.0, 0.5, 0.35])
def test_guess_mode_scales_match_oracle(scale):
    m = controlnet(cn_cfg("sdxl"))
    s = m.residual_scales(scale, guess_mode=True)
    assert s.dtype == torch.float32 and s.numel() == m.num_residuals
    assert torch.equal(s, OC.guess_mode_scales(m.num_residuals - 1, scale))
    assert torch.equal(guess_mode_scales(9, scale), OC.guess_mode_scales(9, scale))
    assert abs(s[0].item() - 0.1 * scale) < 1e-7 and abs(s[-1].item() - scale) < 1e-7
    assert torch.equal(m.residual_scales(scale), torch.full((m.num_residuals,), scale))
    lst = [0.1 * k for k in range(m.num_residuals)]
    assert torch.equal(m.residual_scales(lst), torch.tensor(lst, dtype=torch.float32))
    with pytest.raises(ValueError):
        m.residual_scales(lst[:-1])


def test_constructor_checks():
    cfg = cn_cfg("tiny_sd")
    with pytest.raises(NotImplementedError):
        ControlNetModel(**{k: cfg[k] for k in CN_KEYS}, global_pool_conditions=True)
    with pytest.raises(NotImplementedError):
        ControlNetModel(**{k: cfg[k] for k in CN_KEYS}, class_embed_type="timestep")
    with pytest.raises(NotImplementedError):
        ControlNetModel(**{k: cfg[k] for k in CN_KEYS}, not_an_option=1)
    with pytest.raises(ValueError):
        ControlNetModel(**{k: cfg[k] for k in CN_KEYS}, controlnet_conditioning_channel_order="rbg")
    with pytest.raises(NotImplementedError):  # a 200-channel conditioning conv fits neither conv kernel
        ControlNetModel(**{k: cfg[k] for k in CN_KEYS}, conditioning_embedding_out_channels=(16, 200, 256))
    # reference defaults pass, and the reference's config keys are kept
    m = ControlNetModel(**{k: cfg[k] for k in CN_KEYS}, upcast_attention=False, encoder_hid_dim=None,
                        controlnet_conditioning_channel_order="bgr")
    assert m.config.controlnet_conditioning_channel_order == "bgr"
    assert m.config.conditioning_embedding_out_channels == (16, 32, 96, 256)


def test_oracle_zero_convs_give_zero_residuals():
    """ControlNetModel.from_unet zero-initialises every zero conv (and the conditioning embedding's conv_out): its
    residuals are exactly 0, so the UNet's output with them equals its output without them."""
    cfg = cn_cfg("tiny_sd", conditioning_embedding_out_channels=TINY_COND)
    unet_P = O.init_params(O.unet_param_shapes(cfg), seed=1)
    P = O.init_params(OC.controlnet_param_shapes(cfg), seed=2)
    for k in OC.zero_module_names(cfg):
        P[k] = torch.zeros_like(P[k])
    P = OC.from_unet_params(cfg, unet_P, P)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 4, 8, 8, generator=g)
    ctx = torch.randn(2, 7, cfg["cross_attention_dim"], generator=g)
    img = torch.rand(2, 3, 16, 16, generator=g)
    down, mid = OC.controlnet_forward(cfg, P, x, 500, ctx, img, conditioning_scale=0.7)
    assert all(torch.count_nonzero(d) == 0 for d in down) and torch.count_nonzero(mid) == 0
    with_cn = O.unet_forward(cfg, unet_P, x, 500, ctx, down_block_additional_residuals=down,
                             mid_block_additional_residual=mid)
    assert torch.equal(with_cn, O.unet_forward(cfg, unet_P, x, 500, ctx))
    # and the residual shapes are the UNet's skip shapes
    m = controlnet(cfg)
    assert [(d.shape[2], d.shape[3], d.shape[1]) for d in (*down, mid)] == m.residual_shapes(8, 8)
