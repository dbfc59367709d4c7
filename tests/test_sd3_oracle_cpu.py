"""The SD3 oracle split into sd3_embed / joint_block / sd3_final (the pieces the GPU tests compare block by block)
gives exactly what the single-function restatement of SD3Transformer2DModel.forward gives."""
import torch
import torch.nn.functional as F

from oracle import sd3 as O

bf16 = torch.bfloat16


def forward_in_one_piece(cfg, P, hidden_states, encoder_hidden_states, pooled_projections, timestep):
    """transformer_sd3.py:279-365 written out in one function, as the oracle stated it before the split."""
    ps, heads = cfg["patch_size"], cfg["num_attention_heads"]
    B, _, H, W = hidden_states.shape
    x = F.conv2d(hidden_states, P["pos_embed.proj.weight"], P["pos_embed.proj.bias"], stride=ps)
    x = x.flatten(2).transpose(1, 2)
    h, w, mx = H // ps, W // ps, cfg["pos_embed_max_size"]
    top, left = (mx - h) // 2, (mx - w) // 2
    pe = P["pos_embed.pos_embed"].reshape(1, mx, mx, -1)[:, top:top + h, left:left + w, :].reshape(1, h * w, -1)
    x = x + pe
    t = torch.as_tensor(timestep, dtype=torch.float32).reshape(-1).expand(B)
    t_proj = O.get_timestep_embedding(t, 256, flip_sin_to_cos=True, downscale_freq_shift=0)
    t_emb = O.linear(F.silu(O.linear(t_proj, P, "time_text_embed.timestep_embedder.linear_1")), P,
                     "time_text_embed.timestep_embedder.linear_2")
    p_emb = O.linear(F.silu(O.linear(pooled_projections, P, "time_text_embed.text_embedder.linear_1")), P,
                     "time_text_embed.text_embedder.linear_2")
    temb = t_emb + p_emb
    c = O.linear(encoder_hidden_states, P, "context_embedder")
    for i in range(cfg["num_layers"]):
        c, x = O.joint_block(x, c, temb, P, f"transformer_blocks.{i}", heads, i == cfg["num_layers"] - 1)
    e = O.linear(F.silu(temb), P, "norm_out.linear")
    scale, shift = e.chunk(2, dim=1)
    x = (O._ln(x) + P["norm_out.norm.bias"]) * (1 + scale)[:, None, :] + shift[:, None, :]
    x = O.linear(x, P, "proj_out")
    oc = cfg["out_channels"]
    x = x.reshape(B, h, w, ps, ps, oc).permute(0, 5, 1, 3, 2, 4)
    return x.reshape(B, oc, h * ps, w * ps)


def test_sd3_oracle_split_equals_forward():
    """tiny config, non-square 24 x 16 latent, three samples with their own timestep, pooled embedding and context."""
    cfg = O.SD3_CONFIGS["tiny"]
    P = O.init_sd3_params(cfg, seed=3)
    g = torch.Generator().manual_seed(11)
    B, H, W, L = 3, 24, 16, 13
    x = torch.randn(B, cfg["in_channels"], H, W, generator=g).to(bf16).float()
    ctx = torch.randn(B, L, cfg["joint_attention_dim"], generator=g).to(bf16).float()
    pooled = torch.randn(B, cfg["pooled_projection_dim"], generator=g).to(bf16).float()
    ts = torch.tensor([999.0, 512.25, 3.5])
    ps = cfg["patch_size"]
    h, w = H // ps, W // ps
    xe, c, temb = O.sd3_embed(cfg, P, x, ctx, pooled, ts)
    assert xe.shape == (B, h * w, 128) and c.shape == (B, L, 128) and temb.shape == (B, 128)
    for i in range(cfg["num_layers"]):
        last = i == cfg["num_layers"] - 1
        c, xe = O.joint_block(xe, c, temb, P, f"transformer_blocks.{i}", cfg["num_attention_heads"], last)
        assert (c is None) == last
    split = O.sd3_final(cfg, P, xe, temb, h, w)
    whole = O.sd3_forward(cfg, P, x, ctx, pooled, ts)
    ref = forward_in_one_piece(cfg, P, x, ctx, pooled, ts)
    assert split.shape == (B, cfg["out_channels"], H, W)
    assert torch.equal(split, ref) and torch.equal(whole, ref)
    # the samples really differ, and a non-square crop of the position table is not its transpose
    assert (ref[1] - ref[0]).abs().max() > 0.1 * ref.abs().max()
    pe = O.sd3_pos_embed(cfg, P, h, w)
    assert pe.shape == (1, h * w, 128) and not torch.equal(pe, O.sd3_pos_embed(cfg, P, w, h).reshape(1, w, h, -1)
                                                           .transpose(1, 2).reshape(1, h * w, -1))
