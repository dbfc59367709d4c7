"""Open-Sora IDDPM sampling without a GPU: respacing, the fp32 step scalars against oracle/iddpm.py, the proof that the
B-row loop the pipeline runs equals the reference's 2B-row loop bit for bit, the null-caption key through the
checkpoint loader, and the pipeline's argument checks."""
import numpy as np
import pytest
import torch

from oracle import iddpm as O
from paddlemix_b200.opensora.iddpm import IDDPM, space_timesteps


# ---- respacing -------------------------------------------------------------------------------------------------------
def test_space_timesteps_100_of_1000():
    """One section of 1000 steps, stride 999/99 = 111/11: step k is round(111 k / 11), so k = 6 is round(60.55) = 61
    and k = 11 is exactly 111."""
    s = sorted(space_timesteps(1000, "100"))
    assert len(s) == 100 and s[:6] == [0, 10, 20, 30, 40, 50] and s[6] == 61 and s[11] == 111 and s[-1] == 999
    assert s == sorted({round(111 * k / 11) for k in range(100)})


def test_space_timesteps_ddim_and_sections():
    assert space_timesteps(1000, "ddim50") == set(range(0, 1000, 20))
    s = sorted(space_timesteps(300, [10, 15, 20]))
    assert len(s) == 45
    assert s[:10] == list(range(0, 100, 11))                 # stride 99 / 9 = 11
    assert s[10] == 100 and s[24] == 199 and s[11] == 107     # stride 99 / 14: round(7.07) = 7
    assert s[25] == 200 and s[-1] == 299 and s[26] == 205     # stride 99 / 19: round(5.21) = 5
    assert space_timesteps(300, "10,15,20") == set(s)
    # Python's round: half to even (4.5 -> 4)
    assert space_timesteps(10, "3") == {0, 4, 9}


def test_space_timesteps_errors():
    with pytest.raises(ValueError, match="cannot divide section of 10 steps into 11"):
        space_timesteps(10, [11])
    with pytest.raises(ValueError, match="integer stride"):
        space_timesteps(1000, "ddim999")
    for args in ((10, [11]), (1000, "ddim999")):
        with pytest.raises(ValueError):
            O.space_timesteps(*args)


@pytest.mark.parametrize("resp", ["100", "ddim50", "10,15,20", "250"])
def test_respacing_matches_oracle(resp):
    s = IDDPM(timestep_respacing=resp)
    assert space_timesteps(1000, resp) == O.space_timesteps(1000, resp)
    assert s.timestep_map == O.Diffusion(1000, resp).timestep_map == sorted(space_timesteps(1000, resp))
    # the respaced alphas_cumprod are the base ones at the kept steps
    np.testing.assert_allclose(s.alphas_cumprod, s.base_alphas_cumprod[s.timestep_map], rtol=1e-13, atol=0)


def test_base_schedule_is_linear():
    s = IDDPM()
    assert s.num_timesteps == 1000 and s.timestep_map == list(range(1000))
    betas = 1 - s.base_alphas_cumprod / np.concatenate([[1.0], s.base_alphas_cumprod[:-1]])
    np.testing.assert_allclose(betas, np.linspace(1e-4, 0.02, 1000), rtol=1e-9)
    from paddlemix_b200.opensora.iddpm import linear_betas
    b = linear_betas(1000)
    assert b[0] == 1e-4 and b[-1] == 0.02 and np.array_equal(b, O.linspace_paddle(1e-4, 0.02, 1000).numpy())


@pytest.mark.parametrize("resp", ["100", "ddim50", "10,15,20"])
def test_step_scalars_bit_exact_vs_oracle(resp):
    s, d = IDDPM(timestep_respacing=resp), O.Diffusion(1000, resp)
    tabs = (d.sqrt_recip_alphas_cumprod, d.sqrt_recipm1_alphas_cumprod, d.posterior_mean_coef1, d.posterior_mean_coef2,
            d.log_betas, d.posterior_log_variance_clipped)
    for i in range(s.num_timesteps):
        want = tuple(float(d.extract(t, i)) for t in tabs)
        got = s.step_scalars(i)
        assert np.array(got, dtype=np.float32).tobytes() == np.array(want, dtype=np.float32).tobytes(), i
    # posterior_log_variance_clipped[0] is log(posterior_variance[1])
    assert s.posterior_log_variance_clipped[0] == np.log(s.posterior_variance[1])


def test_constructor_options():
    assert IDDPM(num_sampling_steps=100).timestep_map == IDDPM(timestep_respacing="100").timestep_map
    with pytest.raises(ValueError):
        IDDPM(num_sampling_steps=100, timestep_respacing="100")
    for kw in (dict(use_kl=True), dict(sigma_small=True), dict(predict_xstart=True), dict(learn_sigma=False),
               dict(noise_schedule="squaredcos_cap_v2")):
        with pytest.raises(NotImplementedError):
            IDDPM(**kw)


# ---- the B-row loop is the 2B-row loop -------------------------------------------------------------------------------
def toy_model(x, t, y, **kw):
    """Per-row elementwise model: 2C output channels from the state, the timestep and one caption value per row."""
    C = x.shape[1]
    yv = y[:, 0, 0, :1].float().reshape(-1, 1, 1, 1, 1)
    tv = (t.float() / 1000).reshape(-1, 1, 1, 1, 1)
    eps = torch.tanh(x * 0.7 + yv) * (1 - tv) + 0.1 * x
    var = torch.tanh(x[:, :C] * yv - tv)
    return torch.cat([eps, var], 1)


@pytest.mark.parametrize("noise", ["randn", "philox"])
@pytest.mark.parametrize("cfg_channel", [3, 4, None])
def test_b_rows_equal_reference_2b_rows(cfg_channel, noise):
    d = O.Diffusion(1000, "20")
    B, C = 2, 4
    g = torch.Generator().manual_seed(3)
    z = torch.randn(B, C, 3, 4, 6, generator=g)
    y_cond, y_null = torch.randn(B, 1, 5, 8, generator=g), torch.randn(B, 1, 5, 8, generator=g)
    if noise == "randn":
        table = {i: torch.randn(2 * B, C, 3, 4, 6, generator=g) for i in range(d.num_timesteps)}
        fn2 = lambda i, shape: table[i]               # the second half differs: it never feeds back
        fn1 = lambda i, shape: table[i][:B]
    else:
        fn1 = fn2 = O.philox_noise_fn(1234567890123)  # the first B rows of a 2B draw are the B-row draw
    ref = O.sample_2b(d, toy_model, z, y_cond, y_null, 7.0, cfg_channel, fn2)
    got = O.sample_b(d, toy_model, z, y_cond, y_null, 7.0, cfg_channel, fn1)
    assert torch.equal(ref, got) and bool(torch.isfinite(got).all())
    # guidance and noise both matter
    other = O.sample_b(d, toy_model, z, y_cond, y_null, 1.0, cfg_channel, fn1)
    assert not torch.equal(other, got)


def test_philox_normal_oracle_statistics():
    z = O.philox_normal(42, 7, 1 << 18).double()
    assert abs(z.mean().item()) < 5 / 512 and abs(z.std().item() - 1) < 5 * 2 ** 0.5 / 512
    assert torch.equal(z.float(), O.philox_normal(42, 7, 1 << 18))
    assert not torch.equal(O.philox_normal(42, 8, 16), O.philox_normal(42, 7, 16))
    assert torch.equal(O.philox_normal(42, 7, 10), O.philox_normal(42, 7, 16)[:10])


# ---- null caption through the checkpoint loader ----------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["torch", "paddle"])
def test_null_caption_key_passes_untransposed(layout):
    from oracle import stdit2 as OS
    from paddlemix_b200.opensora import STDiT2
    from paddlemix_b200.weights import check_against_model, linear_weight_keys, torch_to_paddle_layout
    cfg = OS.STDIT2_CONFIGS["tiny"]
    model = STDiT2(cfg)
    assert "y_embedder.y_embedding" not in model.state_dict_shapes()
    lin = linear_weight_keys(model) if layout == "torch" else set()
    sd = {k: torch.zeros(v[::-1] if k in lin else v) for k, v in model.state_dict_shapes().items()}
    ye = torch.randn(cfg["model_max_length"], cfg["caption_channels"])
    sd["y_embedder.y_embedding"] = ye
    if layout == "torch":
        sd = torch_to_paddle_layout(model, sd)
    assert torch.equal(sd["y_embedder.y_embedding"], ye)
    rep = check_against_model(model, sd, strict=True)
    assert rep["unexpected"] == ["y_embedder.y_embedding"] and not rep["missing"]
    assert model.null_caption(2) is None  # nothing loaded yet


# ---- pipeline argument checks (no device work happens before them) ---------------------------------------------------
class _Stop(Exception):
    pass


class StubTransformer:
    """Records the first call and stops the loop there."""

    def __init__(self, null=None):
        self.device = torch.device("cpu")
        self._null = null
        self.calls = []

    def null_caption(self, n):
        return None if self._null is None else self._null[None, None].repeat(n, 1, 1, 1)

    def __call__(self, x, t, y, mask=None, **kw):
        self.calls.append((x.clone(), t.clone(), y.clone(), mask, kw))
        raise _Stop


def test_pipeline_argument_checks():
    from paddlemix_b200.opensora import OpenSoraPipeline
    emb = torch.randn(2, 1, 6, 8)
    pipe = OpenSoraPipeline(StubTransformer(), IDDPM(num_sampling_steps=5))
    with pytest.raises(ValueError, match="no null caption"):
        pipe(emb, num_frames=2, height=32, width=32)
    pipe = OpenSoraPipeline(StubTransformer(null=torch.randn(7, 8)), IDDPM(num_sampling_steps=5))
    with pytest.raises(ValueError, match="caption length"):
        pipe(emb, num_frames=2, height=32, width=32)
    with pytest.raises(ValueError, match="caption length"):
        pipe(emb, negative_prompt_embeds=torch.randn(2, 1, 5, 8), num_frames=2, height=32, width=32)
    for h, w in ((24, 32), (32, 40), (33, 32)):
        with pytest.raises(ValueError, match="multiples of 16"):
            pipe(emb, negative_prompt_embeds=emb, num_frames=2, height=h, width=w)
    with pytest.raises(ValueError, match="latents must be"):
        pipe(emb, negative_prompt_embeds=emb, num_frames=2, height=32, width=32, latents=torch.randn(2, 4, 2, 4, 2))
    with pytest.raises(ValueError, match="prompt_attention_mask"):
        pipe(emb, prompt_attention_mask=torch.ones(2, 5), negative_prompt_embeds=emb, num_frames=2, height=32, width=32)
    with pytest.raises(ValueError, match="vae"):
        pipe(emb, negative_prompt_embeds=emb, num_frames=2, height=32, width=32, output_type="pt")


@pytest.mark.parametrize("num_frames,fps,want", [(1, 24, 120.0), (16, 24, 24.0), (4, 8, 8.0)])
def test_pipeline_first_call(num_frames, fps, want):
    """The first transformer call: 2B rows with the conditional rows and the caption first, the null caption after,
    the mask at B rows, the size tensors at 2B rows, the first respaced timestep, fps 120 for a single frame."""
    from paddlemix_b200.opensora import OpenSoraPipeline
    null = torch.randn(6, 8)
    tr = StubTransformer(null=null)
    pipe = OpenSoraPipeline(tr, IDDPM(num_sampling_steps=10))
    emb = torch.randn(2, 1, 6, 8)
    mask = torch.tensor([[1, 1, 1, 1, 1, 1], [1, 1, 1, 0, 0, 0]])
    lat = torch.randn(2, 4, num_frames, 6, 4)
    with pytest.raises(_Stop):
        pipe(emb, prompt_attention_mask=mask, num_frames=num_frames, height=48, width=32, fps=fps, latents=lat)
    x, t, y, m, kw = tr.calls[0]
    assert torch.equal(x, torch.cat([lat, lat])) and torch.equal(t, torch.full((4,), 999.0))
    assert torch.equal(y[:2], emb.to(torch.bfloat16).float()) and torch.equal(y[2:], null[None, None].repeat(2, 1, 1, 1).to(torch.bfloat16).float())
    assert torch.equal(m, mask)
    for k, v in dict(num_frames=num_frames, height=48.0, width=32.0, ar=1.5, fps=want).items():
        assert torch.equal(kw[k], torch.full((4,), float(v))), k
