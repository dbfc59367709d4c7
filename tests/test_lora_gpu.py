"""LoRA on the device: b200mix_lora_apply against an fp64 host reference, and the UNet / pipelines with LoRAs
against the fp32 oracle on the merged weights (oracle/lora.py + oracle/unet.py).

Kernel bound (tf32 operands rounded with rna, fp32 accumulation, one bf16 rounding):
    |out - bf16(exact)| <= ulp_bf16(exact) + 2^-10 * sum_j |col_scale[k] * U[n, j] * D[j, k]|
Model tolerances are test_unet_gpu.py's (cosine >= 0.999, max |err| <= 4 % of the output's max magnitude), and the
LoRA-free output must fail them, so each comparison proves the LoRA is applied."""
import pytest
import torch

from oracle import lora as OL
from oracle import unet as O

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
UNET_KEYS = ("in_channels", "out_channels", "flip_sin_to_cos", "freq_shift", "down_block_types", "up_block_types",
             "block_out_channels", "layers_per_block", "norm_num_groups", "norm_eps", "cross_attention_dim",
             "transformer_layers_per_block", "attention_head_dim", "use_linear_projection", "addition_embed_type",
             "addition_time_embed_dim", "projection_class_embeddings_input_dim", "resnet_out_scale_factor")


# ---- kernel ------------------------------------------------------------------------------------------------------
def ulp_bf16(x):
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


def make_item(N, K, R, g, ld=None, col_scale=False, colsum=False, zero=False):
    dev = "cuda"
    ld = ld or K
    parent = (torch.randn(N + 3, ld, generator=g) * 0.05).to(bf16).to(dev)
    out = parent[2: 2 + N, :K]  # a row slice with a row stride
    R8 = (R + 7) // 8 * 8
    U = torch.zeros(N, R8)
    D = torch.zeros(R8, K)
    if not zero:
        U[:, :R] = torch.randn(N, R, generator=g) * 0.02
        D[:R] = torch.randn(R, K, generator=g) * 0.5
    it = dict(out=out, base=out.clone(), U=U.to(dev), D=D.to(dev))
    if col_scale:
        it["col_scale"] = (1 + 0.3 * torch.randn(K, generator=g)).to(dev)
    if colsum:
        it["colsum_base"] = out.float().sum(1).contiguous()
        it["colsum"] = torch.full((N,), float("nan"), device=dev)
    return it, parent


def check_item(it, what):
    U, D = it["U"].double().cpu(), it["D"].double().cpu()
    cs = it["col_scale"].double().cpu() if "col_scale" in it else torch.ones(D.shape[1], dtype=torch.float64)
    base = it["base"].double().cpu()
    exact = base + (U @ D) * cs[None, :]
    absum = (U.abs() @ D.abs()) * cs.abs()[None, :]
    out = it["out"].double().cpu()
    bound = ulp_bf16(exact) + 2.0 ** -10 * absum
    err = (out - exact.to(bf16).double()).abs()
    assert (err <= bound).all(), f"{what}: worst excess {(err - bound).max().item()}"
    if "colsum" in it:
        want = it["colsum_base"].double().cpu() + (out - base).sum(1)
        got = it["colsum"].double().cpu()
        assert torch.allclose(got, want, rtol=1e-5, atol=1e-5 * base.abs().sum(1).max().item()), what


@pytest.mark.parametrize("R", [1, 4, 7, 64, 128, 256])
def test_lora_apply_matches_fp64(R):
    from paddlemix_b200 import ops
    g = torch.Generator().manual_seed(R)
    items = [make_item(200, 328, R, g, ld=520, col_scale=True, colsum=True)[0],
             make_item(64, 64, R, g)[0], make_item(1, 8, R, g, col_scale=True)[0], make_item(333, 2880, R, g)[0]]
    ops.lora_apply(items)
    for i, it in enumerate(items):
        check_item(it, f"R={R} item {i}")


def test_lora_apply_many_items_one_launch_deterministic():
    from paddlemix_b200 import ops
    g = torch.Generator().manual_seed(5)
    items = []
    for i in range(300):
        N = int(torch.randint(1, 140, (1,), generator=g))
        K = 8 * int(torch.randint(1, 40, (1,), generator=g))
        R = int(torch.randint(1, 40, (1,), generator=g))
        items.append(make_item(N, K, R, g, ld=K + 8 * (i % 3), col_scale=i % 2 == 0, colsum=i % 4 == 0)[0])
    n0 = ops.launches()
    ops.lora_apply(items)
    assert ops.launches() - n0 == 1
    first = [(it["out"].clone(), it.get("colsum", torch.zeros(1)).clone()) for it in items]
    for it in items:
        check_item(it, "many items")
    ops.lora_apply(items)
    for it, (o, c) in zip(items, first):
        assert torch.equal(it["out"], o) and torch.equal(it.get("colsum", torch.zeros(1)), c), "not deterministic"


def test_lora_apply_zero_update_is_bit_exact():
    from paddlemix_b200 import ops
    g = torch.Generator().manual_seed(9)
    items, parents = [], []
    for R in (8, 64):
        it, parent = make_item(130, 200 - 200 % 8, R, g, ld=256, col_scale=True, colsum=True, zero=True)
        it["base"].view(torch.int16)[0, :4] = torch.tensor([-32768, 0, -32768, 1], dtype=torch.int16)  # -0, +0
        items.append(it), parents.append(parent)
    before = [p.clone() for p in parents]
    for it in items:
        it["out"].copy_(torch.randn_like(it["out"], dtype=torch.float32).to(bf16))
    ops.lora_apply(items)
    for it, p, b in zip(items, parents, before):
        assert torch.equal(it["out"].view(torch.int16), it["base"].view(torch.int16))
        assert torch.equal(it["colsum"].view(torch.int32), it["colsum_base"].view(torch.int32))
        rest = torch.ones_like(p, dtype=torch.bool)
        rest[2: 2 + it["out"].shape[0], : it["out"].shape[1]] = False
        assert torch.equal(p[rest], b[rest]), "wrote outside the target"


# ---- UNet ---------------------------------------------------------------------------------------------------------
def make_unet(name, seed=1):
    from paddlemix_b200.ppdiffusers.unet_2d_condition import UNet2DConditionModel
    cfg = O.UNET_CONFIGS[name]
    P = O.init_params(O.unet_param_shapes(cfg), seed=seed)
    return cfg, P, UNet2DConditionModel(**{k: cfg[k] for k in UNET_KEYS}).load_state_dict(P, device=0)


def synthetic_lora(unet, seed, rank=4, strength=0.5, alpha=None, layers=None):
    """A ppdiffusers-format (Paddle layout) LoRA on every LoRA-compatible layer (or `layers`): dW elements of about
    `strength` times the weight's own spread."""
    from paddlemix_b200.ppdiffusers.lora import lora_layer_shapes
    g = torch.Generator().manual_seed(seed)
    sd, alphas = {}, {}
    for layer, shape in lora_layer_shapes(unet.state_dict_shapes()).items():
        if layers is not None and layer not in layers:
            continue
        n_out, n_in = shape[:2]
        fan = n_in * (shape[2] * shape[3] if len(shape) == 4 else 1)
        down = torch.randn(rank, fan, generator=g) / fan ** 0.5
        up = torch.randn(n_out, rank, generator=g) * strength / (3 * rank) ** 0.5
        if alpha is not None:
            up = up * rank / alpha
            alphas[f"unet.{layer}.alpha"] = alpha
        if len(shape) == 2:  # Paddle Linear: down [in, r], up [r, out]
            sd[f"unet.{layer}.lora.down.weight"], sd[f"unet.{layer}.lora.up.weight"] = down.t().contiguous(), up.t().contiguous()
        else:
            sd[f"unet.{layer}.lora.down.weight"] = down.reshape(rank, n_in, shape[2], shape[3])
            sd[f"unet.{layer}.lora.up.weight"] = up.reshape(n_out, rank, 1, 1)
    return sd, (alphas or None)


def inputs(cfg, B, H, L, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, cfg["in_channels"], H, H, generator=g).to(bf16).float()
    ctx = torch.randn(B, L, cfg["cross_attention_dim"], generator=g).to(bf16).float()
    added = None
    if cfg["addition_embed_type"] == "text_time":
        n_text = cfg["projection_class_embeddings_input_dim"] - 6 * cfg["addition_time_embed_dim"]
        added = {"text_embeds": torch.randn(B, n_text, generator=g).to(bf16).float(),
                 "time_ids": torch.tensor([[H * 8., H * 8., 0, 0, H * 8., H * 8.]] * B)}
    return x, ctx, added


def cuda(d):
    return None if d is None else {k: v.cuda() for k, v in d.items()}


def stats(out, ref):
    out, ref = out.float().cpu(), ref.float().cpu()
    cos = torch.nn.functional.cosine_similarity(out.flatten(), ref.flatten(), dim=0).item()
    return cos, (out - ref).abs().max().item() / ref.abs().max().item()


def check_vs_oracle(cfg, P, unet, loras, x, ctx, added, t, what, **kw):
    """unet (LoRA applied) against the oracle on the merged weights, which the LoRA-free oracle must not pass."""
    dev = "cuda"
    Pd = {k: v.to(dev) for k, v in P.items()}
    merged = OL.merge(Pd, loras)
    tt = torch.tensor([float(t)], device=dev)  # the oracle builds its embedding on the timestep's device
    ref = O.unet_forward(cfg, merged, x.to(dev), tt, ctx.to(dev), cuda(added))
    plain = O.unet_forward(cfg, Pd, x.to(dev), tt, ctx.to(dev), cuda(added))
    out = unet(x.cuda(), t, ctx.cuda(), added_cond_kwargs=cuda(added), return_dict=False, **kw)[0]
    cos, rel = stats(out, ref)
    assert cos >= 0.999 and rel <= 0.04, f"{what}: cosine {cos}, max rel err {rel}"
    pc, pr = stats(plain, ref)
    assert pc < 0.999 or pr > 0.04, f"{what}: the LoRA-free output passes too (cosine {pc}, rel {pr})"
    print(f"{what}: cosine {cos:.6f}, max rel err {rel:.4f} (LoRA-free: {pc:.4f}, {pr:.3f})")


@pytest.mark.slow
@pytest.mark.parametrize("name,H", [("sd15", 32), ("sdxl", 64)])
def test_full_size_full_coverage_lora_vs_oracle(name, H):
    cfg, P, unet = make_unet(name)
    sd, alphas = synthetic_lora(unet, 3, rank=8, alpha=4.0)
    unet.load_attn_procs(sd, network_alphas=alphas)
    x, ctx, added = inputs(cfg, 1, H, 77)
    check_vs_oracle(cfg, P, unet, [(sd, alphas, 1.0)], x, ctx, added, 701, f"{name} full-coverage LoRA")
    # two adapters mixed with set_adapters weights
    sd2, _ = synthetic_lora(unet, 4, rank=16)
    unet.load_attn_procs(sd2, adapter_name="b")
    unet.set_adapters(["default_0", "b"], [0.6, -0.8])
    check_vs_oracle(cfg, P, unet, [(sd, alphas, 0.6), (sd2, None, -0.8)], x, ctx, added, 301,
                    f"{name} two adapters")


def device_tensors(unet):
    from paddlemix_b200.ppdiffusers.lora import targets
    out = {}
    for layer, places in targets(unet).items():
        for i, p in enumerate(places):
            out[f"{layer}[{i}]"] = p.tensor().clone()
            if p.ln is not None:
                _, _, colsum, bias = p.ln()
                out[f"{layer}[{i}].colsum"], out[f"{layer}[{i}].bias"] = colsum.clone(), bias.clone()
    return out


def same_bits(a, b):
    return a.keys() == b.keys() and all(torch.equal(a[k].view(torch.uint8), b[k].view(torch.uint8)) for k in a)


@pytest.mark.parametrize("name", ["tiny_sd", "tiny_xl"])
def test_exactness(name):
    cfg, P, unet = make_unet(name)
    x, ctx, added = inputs(cfg, 2, 16, 20)
    run = lambda **kw: unet(x.cuda(), 501, ctx.cuda(), added_cond_kwargs=cuda(added), return_dict=False, **kw)[0].clone()  # noqa: E731
    fresh_t, fresh_y = device_tensors(unet), run()
    A, aA = synthetic_lora(unet, 10, rank=7, alpha=3.0, strength=1.0)
    B, _ = synthetic_lora(unet, 11, rank=5)
    unet.load_attn_procs(A, network_alphas=aA, adapter_name="A")
    with_a_t, with_a = device_tensors(unet), run()
    assert not torch.equal(with_a, fresh_y)
    assert torch.equal(run(cross_attention_kwargs={"scale": 0.0}), fresh_y), "scale 0 must equal no LoRA"
    assert same_bits(device_tensors(unet), fresh_t)
    check_vs_oracle(cfg, P, unet, [(A, aA, 0.5)], x, ctx, added, 501, f"{name} scale 0.5",
                    cross_attention_kwargs={"scale": 0.5})
    assert torch.equal(run(), with_a), "scale back to 1.0"
    unet.load_attn_procs(B, adapter_name="B")
    unet.set_adapters("A")
    assert same_bits(device_tensors(unet), with_a_t), "A -> B -> A must equal A"
    unet.fuse_lora(0.7)
    fused = run(cross_attention_kwargs={"scale": 0.0})
    assert torch.equal(fused, run()), "a fused adapter ignores the call scale"
    unet.unfuse_lora()
    assert same_bits(device_tensors(unet), with_a_t)
    unet.unload_lora_weights()
    assert same_bits(device_tensors(unet), fresh_t) and torch.equal(run(), fresh_y)
    assert unet._lora.snap == {}, "snapshots are freed with the last adapter"


# ---- pipelines ----------------------------------------------------------------------------------------------------
SD = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False, set_alpha_to_one=False,
          steps_offset=1)


def test_pipeline_graphs_see_lora_and_call_scale():
    from oracle.schedulers import DDIMScheduler as ODDIM
    from paddlemix_b200.ppdiffusers.pipelines import StableDiffusionPipeline
    from paddlemix_b200.ppdiffusers.schedulers import DDIMScheduler
    cfg, P, unet = make_unet("tiny_xl")
    x, ctx, added = inputs(cfg, 2, 16, 20)
    neg = torch.zeros_like(ctx)
    steps, gs = 4, 5.0
    run = dict(prompt_embeds=ctx, negative_prompt_embeds=neg, latents=x, num_inference_steps=steps, guidance_scale=gs,
               added_cond_kwargs=added)
    graphed = StableDiffusionPipeline(unet, DDIMScheduler(**SD))
    plain = graphed(**run).cpu()
    g0 = dict(graphed._graphed)
    sd, alphas = synthetic_lora(unet, 21, rank=8)
    graphed.load_lora_weights(sd)
    eager = StableDiffusionPipeline(unet, DDIMScheduler(**SD), use_cuda_graph=False)
    for s in (1.0, 0.5):
        kw = {"cross_attention_kwargs": {"scale": s}}
        lat = graphed(**run, **kw).cpu()
        assert graphed._graphed == g0, "no new graph may be captured"
        assert torch.equal(lat, eager(**run, **kw).cpu()), f"graphed != eager at scale {s}"
        assert not torch.equal(lat, plain)
        sch = ODDIM(**SD)
        sch.set_timesteps(steps)
        merged = OL.merge(P, [(sd, alphas, s)])
        cur = x.clone()
        add2 = {k: torch.cat([v, v], 0) for k, v in added.items()}
        for t in sch.timesteps:
            eps = O.unet_forward(cfg, merged, torch.cat([cur, cur]), int(t), torch.cat([neg, ctx]), add2)
            eu, ec = eps.chunk(2)
            cur = sch.step(eu + gs * (ec - eu), t, cur)
        cos, rel = stats(lat, cur)
        assert cos >= 0.999 and rel <= 0.04, f"scale {s}: cosine {cos}, rel {rel}"
    with pytest.raises(NotImplementedError):
        graphed(**run, cross_attention_kwargs={"foo": 1})
    graphed.unload_lora_weights()
    assert torch.equal(graphed(**run).cpu(), plain)
