"""LoRA host logic without a GPU: key formats, where every layer lands in the device layout, the adapter state
machine and ops.lora_apply's refusals."""
import pytest
import torch

from oracle import unet as O

bf16 = torch.bfloat16
KEYS = ("in_channels", "out_channels", "down_block_types", "up_block_types", "block_out_channels", "layers_per_block",
        "cross_attention_dim", "transformer_layers_per_block", "attention_head_dim", "use_linear_projection",
        "addition_embed_type", "addition_time_embed_dim", "projection_class_embeddings_input_dim")


def new_unet(name):
    from paddlemix_b200.ppdiffusers.unet_2d_condition import UNet2DConditionModel
    cfg = O.UNET_CONFIGS[name]
    return UNet2DConditionModel(**{k: cfg[k] for k in KEYS})


def factors(shape, r, g, lo=-2, hi=3):
    """Small-integer torch-layout factors (every product below is exact in bf16 and fp32)."""
    n_out, n_in = shape[:2]
    up = torch.randint(lo, hi, (n_out, r), generator=g).float()
    down = torch.randint(lo, hi, (r, n_in) + tuple(shape[2:]), generator=g).float()
    return up, down


def lora_sd(unet, r, g, fmt="paddle", alpha=None):
    """A LoRA on every LoRA-compatible layer in one of the accepted key formats / layouts; returns (state dict,
    network_alphas, from_diffusers, {layer: (up, down)} in torch layout)."""
    from paddlemix_b200.ppdiffusers.lora import lora_layer_shapes
    sd, alphas, truth = {}, {}, {}
    for layer, shape in lora_layer_shapes(unet.state_dict_shapes()).items():
        if fmt == "kohya" and layer.startswith(("time_embedding.", "add_embedding.")):
            continue  # kohya names cannot spell these (the reference's conversion turns them into unknown names)
        up, down = factors(shape, r, g)
        truth[layer] = (up, down)
        if len(shape) == 4:
            up_s, down_s = up.reshape(*up.shape, 1, 1), down
        elif fmt == "paddle" or fmt == "legacy":
            up_s, down_s = up.t(), down.t()
        else:
            up_s, down_s = up, down
        if fmt == "kohya":
            name = "lora_unet_" + layer.replace(".", "_")
            sd[name + ".lora_down.weight"], sd[name + ".lora_up.weight"] = down_s, up_s
            if alpha is not None:
                sd[name + ".alpha"] = torch.tensor(alpha)
            continue
        key = layer
        if fmt == "legacy" and ".attn" in layer:
            a, p = layer.rsplit(".", 1) if not layer.endswith("to_out.0") else (layer[:-len(".to_out.0")], "to_out")
            key = f"{a}.processor.{p}_lora"
            sd[f"{key}.down.weight"], sd[f"{key}.up.weight"] = down_s, up_s
        else:
            sd[f"unet.{key}.lora.down.weight"], sd[f"unet.{key}.lora.up.weight"] = down_s, up_s
        if alpha is not None:
            alphas[f"unet.{layer}.alpha"] = alpha
    return sd, (alphas or None), fmt in ("torch", "kohya"), truth


# ---- key formats --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["sd15", "sdxl"])
@pytest.mark.parametrize("fmt", ["paddle", "torch", "legacy", "kohya"])
def test_every_format_maps_every_layer(name, fmt):
    from paddlemix_b200.ppdiffusers import lora as L
    unet = new_unet(name)
    g = torch.Generator().manual_seed(0)
    sd, alphas, torch_layout, truth = lora_sd(unet, 1, g, fmt, alpha=2.0)
    # a dict carries no format metadata: torch layout is named explicitly, except for kohya keys (a torch format)
    sd2, alphas2, from_diffusers = L.lora_state_dict(sd, unet.config, True if fmt == "torch" else None)
    assert from_diffusers == torch_layout
    if alphas is not None:
        alphas2 = {**(alphas2 or {}), **alphas}
    sd2, te = L.split_text_encoder(sd2)
    parsed = L.parse_lora(sd2, alphas2, from_diffusers, L.lora_layer_shapes(unet.state_dict_shapes()))
    assert set(parsed) == set(truth)
    assert set(truth) == set(L.targets(unet)) or fmt == "kohya"
    for layer, (up, down, s) in parsed.items():
        assert torch.equal(up, truth[layer][0]) and torch.equal(down, truth[layer][1]), layer
        assert s == 2.0, layer


def test_kohya_sgm_names_and_text_encoder_split():
    from paddlemix_b200.ppdiffusers import lora as L
    unet = new_unet("sdxl")
    shapes = L.lora_layer_shapes(unet.state_dict_shapes())
    want = {"input_blocks_4_1_transformer_blocks_0_attn1_to_q": "down_blocks.1.attentions.0.transformer_blocks.0.attn1.to_q",
            "input_blocks_3_0_op": "down_blocks.0.downsamplers.0.conv",
            "input_blocks_1_0_emb_layers_1": "down_blocks.0.resnets.0.time_emb_proj",
            "input_blocks_1_0_in_layers_2": "down_blocks.0.resnets.0.conv1",
            "input_blocks_1_0_out_layers_3": "down_blocks.0.resnets.0.conv2",
            "middle_block_1_transformer_blocks_3_attn2_to_out_0": "mid_block.attentions.0.transformer_blocks.3.attn2.to_out.0",
            "middle_block_2_in_layers_2": "mid_block.resnets.1.conv1",
            "output_blocks_0_0_skip_connection": "up_blocks.0.resnets.0.conv_shortcut",
            "output_blocks_2_2_conv": "up_blocks.0.upsamplers.0.conv",
            "output_blocks_5_1_proj_in": "up_blocks.1.attentions.2.proj_in",
            "output_blocks_4_1_transformer_blocks_1_ff_net_0_proj": "up_blocks.1.attentions.1.transformer_blocks.1.ff.net.0.proj"}
    g = torch.Generator().manual_seed(1)
    sd = {}
    for k, layer in want.items():
        up, down = factors(shapes[layer], 4, g)
        sd[f"lora_unet_{k}.lora_down.weight"] = down
        sd[f"lora_unet_{k}.lora_up.weight"] = up.reshape(*up.shape, *((1, 1) if down.dim() == 4 else ()))
        sd[f"lora_unet_{k}.alpha"] = torch.tensor(8.0)
    sd["lora_te1_text_model_encoder_layers_0_self_attn_q_proj.lora_down.weight"] = torch.zeros(4, 768)
    sd["lora_te1_text_model_encoder_layers_0_self_attn_q_proj.lora_up.weight"] = torch.zeros(768, 4)
    sd2, alphas, from_diffusers = L.lora_state_dict(sd, unet.config)
    assert from_diffusers
    unet_sd, te = L.split_text_encoder(sd2)
    assert len(te) == 2 and all(k.startswith("text_encoder.") for k in te)
    parsed = L.parse_lora(unet_sd, alphas, True, shapes)
    assert set(parsed) == set(want.values())
    assert all(s == 2.0 for _, _, s in parsed.values())


def test_refusals_happen_on_the_host():
    from paddlemix_b200.ppdiffusers import lora as L
    unet = new_unet("tiny_sd")
    shapes = L.lora_layer_shapes(unet.state_dict_shapes())
    cases = [({"conv_in.lora.down.weight": torch.zeros(4, 4, 3, 3), "conv_in.lora.up.weight": torch.zeros(64, 4, 1, 1)},
              "LoRACompatible"),
             ({"lora_unet_down_blocks_0_resnets_0_conv1.hada_w1_a": torch.zeros(1)}, "hada_w1_a"),
             ({"x.lokr_w1": torch.zeros(1)}, "lokr_w1"),
             ({"down_blocks.0.resnets.0.conv1.dora_scale": torch.zeros(1)}, "dora_scale"),
             ({"down_blocks.9.resnets.0.conv1.lora.down.weight": torch.zeros(4, 64, 3, 3),
               "down_blocks.9.resnets.0.conv1.lora.up.weight": torch.zeros(64, 4, 1, 1)}, "no LoRA-compatible layer"),
             ({"time_embedding.linear_1.lora.down.weight": torch.zeros(4, 64),  # torch layout read as Paddle
               "time_embedding.linear_1.lora.up.weight": torch.zeros(256, 4)}, "do not fit")]
    for sd, msg in cases:
        with pytest.raises(ValueError, match=msg):
            s2, a2, fd = L.lora_state_dict(sd, unet.config)
            L.parse_lora(L.split_text_encoder(s2)[0], a2, fd, shapes)
    with pytest.raises(ValueError, match="matches no LoRA layer"):
        L.parse_lora({"time_embedding.linear_1.lora.down.weight": torch.zeros(64, 4),
                      "time_embedding.linear_1.lora.up.weight": torch.zeros(4, 256)},
                     {"unet.time_embedding.linear_2.alpha": 1.0}, False, shapes)
    with pytest.raises(ValueError, match="no UNet entries"):
        unet.load_attn_procs({"text_encoder.x.lora.down.weight": torch.zeros(1)})


# ---- device order ---------------------------------------------------------------------------------------------------
def cpu_loaded(name, g, gamma_beta=True):
    """The model's device layout built on the CPU from all-zero weights plus one integer dW per layer, with integer
    LayerNorm gammas / betas: every transform of the load path is then exact, and each tensor region holds the load
    path's own image of that layer's dW."""
    from paddlemix_b200.ppdiffusers import lora as L
    unet = new_unet(name)
    P, truth = {}, {}
    lshapes = L.lora_layer_shapes(unet.state_dict_shapes())
    for k, s in unet.state_dict_shapes().items():
        P[k] = torch.zeros(s)
        if k.endswith(".weight") and len(s) == 1:
            P[k] = torch.randint(1, 4, s, generator=g).float() if gamma_beta else torch.ones(s)
        elif ".norm" in k and k.endswith(".bias"):
            P[k] = torch.randint(-2, 3, s, generator=g).float()
    for layer, shape in lshapes.items():
        up, down = factors(shape, 3, g, -1, 2)
        truth[layer] = (up, down)
        dw = (up @ down.reshape(down.shape[0], -1)).reshape((shape[0],) + tuple(shape[1:]))
        P[layer + ".weight"] = dw.t().contiguous() if len(shape) == 2 else dw
    unet.device = torch.device("cpu")
    unet._load_tensors(P, unet.device)
    return unet, truth


@pytest.mark.parametrize("name", ["tiny_sd", "tiny_xl", "ref_tiny"])
def test_device_order_factors_match_the_load_path(name):
    from paddlemix_b200.ppdiffusers import lora as L
    g = torch.Generator().manual_seed(3)
    unet, truth = cpu_loaded(name, g)
    kinds = set()
    for layer, places in L.targets(unet).items():
        up, down = truth[layer]
        for p in places:
            U, D = p.rows(up).double(), p.cols(down).double()
            dev = U @ D
            r0 = p.r0()
            w = p.tensor()[r0: r0 + U.shape[0]].double()
            if p.ln is not None:
                gamma, beta, colsum, bias = p.ln()
                dev = dev * gamma.double()[None, :]
                assert torch.equal(colsum[r0: r0 + U.shape[0]].double(), dev.sum(1)), layer
                assert torch.equal(bias[r0: r0 + U.shape[0]].double(), U @ (D @ beta.double())), layer
            assert torch.equal(w, dev), f"{layer}: device-order U @ D differs from the load path's tensor"
            kinds.add((p.rows.__name__ if hasattr(p.rows, "__name__") else "", D.shape[1] // max(1, down.shape[1]),
                       p.ln is not None))
    assert len(kinds) >= 4


# ---- adapter state machine ------------------------------------------------------------------------------------------
def test_adapter_state_machine(monkeypatch):
    from paddlemix_b200.ppdiffusers import lora as L
    g = torch.Generator().manual_seed(4)
    unet, _ = cpu_loaded("tiny_sd", g)
    calls = []
    monkeypatch.setattr(L.LoraState, "realise", lambda self: calls.append(self.coefficients()))
    sdA, _, _, _ = lora_sd(unet, 2, g)
    sdB, _, _, _ = lora_sd(unet, 3, g)
    assert unet.load_attn_procs(sdA) == "default_0"
    assert calls[-1] == {"default_0": 1.0}
    unet.load_attn_procs(sdB, adapter_name="B")
    assert calls[-1] == {"B": 1.0}, "a new adapter becomes the only active one"
    with pytest.raises(ValueError, match="already in use"):
        unet.load_attn_procs(sdB, adapter_name="B")
    unet.set_adapters(["default_0", "B"], [0.5, 2.0])
    assert calls[-1] == {"default_0": 0.5, "B": 2.0}
    n = len(calls)
    unet._set_lora_scale(1.0)
    assert len(calls) == n, "an unchanged scale launches nothing"
    unet._set_lora_scale(0.5)
    assert calls[-1] == {"default_0": 0.25, "B": 1.0}
    unet.fuse_lora(0.5)
    assert calls[-1] == {"default_0": 0.25, "B": 1.0}
    n = len(calls)
    unet._set_lora_scale(3.0)
    assert len(calls) == n, "fused adapters ignore the call scale"
    with pytest.raises(ValueError, match="fused"):
        unet.set_adapters("B")
    unet.unload_lora_weights()
    assert set(unet._lora.adapters) == {"default_0", "B"}, "fused adapters survive unload"
    unet.unfuse_lora()
    assert calls[-1] == {"default_0": 1.5, "B": 6.0}
    unet.set_adapters("B", 0.0)
    assert calls[-1] == {}
    unet.unload_lora_weights()
    assert not unet._lora.adapters
    with pytest.raises(ValueError, match="not loaded"):
        unet.set_adapters("B")


# ---- ops.lora_apply refusals ------------------------------------------------------------------------------------------
def test_lora_apply_refuses_before_launch():
    from paddlemix_b200 import ops
    from paddlemix_b200._lib import B200MixError

    def item(**kw):
        it = dict(out=torch.zeros(16, 32, dtype=bf16), base=torch.zeros(16, 32, dtype=bf16), U=torch.zeros(16, 8),
                  D=torch.zeros(8, 32))
        it.update(kw)
        return {k: v for k, v in it.items() if v is not None}

    big = torch.zeros(64, 32, dtype=bf16)
    cases = [(item(out=torch.zeros(16, 32)), TypeError, "out must be"),
             (item(U=torch.zeros(16, 8, dtype=torch.float64)), TypeError, "U must be"),
             (item(U=torch.zeros(16, 7), D=torch.zeros(7, 32)), ValueError, "multiple of 8"),
             (item(U=torch.zeros(16, 520), D=torch.zeros(520, 32)), ValueError, "up to 512"),
             (item(out=torch.zeros(16, 12, dtype=bf16), base=torch.zeros(16, 12, dtype=bf16), D=torch.zeros(8, 12)),
              ValueError, "multiple"),
             (item(D=torch.zeros(8, 40)), ValueError, "D must be"),
             (item(out=torch.zeros(16, 64, dtype=bf16)[:, ::2]), ValueError, "contiguous last dimension"),
             (item(out=torch.zeros(16, 36, dtype=bf16)[:, :32]), ValueError, "multiples of 8"),
             (item(colsum=torch.zeros(16)), ValueError, "go together"),
             (item(col_scale=torch.zeros(16)), ValueError, "col_scale must be"),
             (item(out=big[:16], base=big[8:24]), ValueError, "overlaps"),
             (dict(item(), extra=1), ValueError, "unknown fields")]
    for it, exc, msg in cases:
        with pytest.raises(exc, match=msg):
            ops.lora_apply([it])
    with pytest.raises(ValueError, match="overlap"):
        ops.lora_apply([item(out=big[:16]), item(out=big[8:24])])
    with pytest.raises(ValueError, match="no items"):
        ops.lora_apply([])
    with pytest.raises(B200MixError, match="CUDA tensor"):
        ops.lora_apply([item()])
