"""Stochastic DDIM (eta > 0) and DPM-Solver++ 2M SDE without a GPU: the host schedulers' scalars bit for bit against
the oracle, the kernels' documented arithmetic (restated here on the host scalars) against the oracle steps, the
deterministic limit of zero noise, the options outside the device step, the seed and step index each step hands its
kernel, the wrappers' input checks and the pipelines' rule for passing the generator."""
import numpy as np
import pytest
import torch

from oracle import schedulers as OS
from oracle import stochastic as OSa
from paddlemix_b200 import _lib, ops
from paddlemix_b200.ppdiffusers import schedulers as S
from paddlemix_b200.sampling import seed_from

SD = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")


# ---- DDIM, eta > 0 -----------------------------------------------------------------------------------------------------
DDIM_GRID = [dict(timestep_spacing=s, steps_offset=o, set_alpha_to_one=a)
             for s in ("linspace", "leading", "trailing") for o in (0, 1) for a in (True, False)]
DDIM_GRID += [dict(SD, timestep_spacing="leading", steps_offset=1, set_alpha_to_one=False),
              dict(beta_schedule="squaredcos_cap_v2")]


@pytest.mark.parametrize("cfg", DDIM_GRID, ids=lambda c: "-".join(str(v) for v in c.values()))
@pytest.mark.parametrize("eta", [0.3, 0.5, 1.0])
@pytest.mark.parametrize("steps", [1, 2, 10, 50])
def test_ddim_eta_host_scalars_are_the_oracles(cfg, eta, steps):
    h, o = S.DDIMScheduler(**cfg), OSa.DDIMScheduler(**cfg)
    h.set_timesteps(steps), o.set_timesteps(steps)
    assert np.array_equal(h.timesteps, o.timesteps.numpy())
    for t in h.timesteps:
        got, want = h.eta_step_scalars(int(t), eta), o.eta_step_scalars(int(t), eta)
        assert got == want, (int(t), got, want)
        assert got[4] > 0.0 or int(t) - 1000 // steps < 0


def test_ddim_step_scalars_are_the_eta_zero_case():
    h = S.DDIMScheduler(**SD)
    h.set_timesteps(30)
    for t in h.timesteps:
        sc = h.eta_step_scalars(int(t), 0.0)
        assert h.step_scalars(int(t)) == sc[:4] and sc[4] == 0.0


def kernel_ddim_eta(m, x, z, sc, pred, clip, clipped_eps):
    """b200mix_ddim_eta_step as include/b200mix.h documents it, on fp32 tensors."""
    sa_t, sb_t, sa_p, sb_p, std = (torch.tensor(v, dtype=torch.float32) for v in sc)
    if pred == "epsilon":
        x0, e = (x - sb_t * m) / sa_t, m
    elif pred == "sample":
        x0 = m
        e = (x - sa_t * x0) / sb_t
    else:
        x0, e = sa_t * x - sb_t * m, sa_t * m + sb_t * x
    if clip > 0:
        x0 = x0.clamp(-clip, clip)
    if clipped_eps:
        e = (x - sa_t * x0) / sb_t
    return (sa_p * x0 + sb_p * e) + std * z


@pytest.mark.parametrize("pred", ["epsilon", "sample", "v_prediction"])
@pytest.mark.parametrize("clip_sample", [False, True])
@pytest.mark.parametrize("use_clipped", [False, True])
@pytest.mark.parametrize("eta", [0.3, 1.0])
def test_ddim_eta_kernel_arithmetic_is_the_oracle_step(pred, clip_sample, use_clipped, eta):
    kw = dict(SD, prediction_type=pred, clip_sample=clip_sample, set_alpha_to_one=False, steps_offset=1)
    h, o = S.DDIMScheduler(**kw), OSa.DDIMScheduler(**kw)
    h.set_timesteps(12), o.set_timesteps(12)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 4, 8, 8, generator=g)
    for t in h.timesteps:
        m, z = torch.randn(x.shape, generator=g) * 1.5, torch.randn(x.shape, generator=g)
        want = o.step(m, t, x, eta=eta, use_clipped_model_output=use_clipped, variance_noise=z)
        got = kernel_ddim_eta(m, x, z, h.eta_step_scalars(int(t), eta), pred, h.clip_sample_range if clip_sample else 0,
                              use_clipped)
        assert torch.equal(got, want), int(t)
        x = want


def test_ddim_oracle_seed_is_the_philox_stream_at_the_call_index():
    from oracle.iddpm import philox_normal
    a, b = OSa.DDIMScheduler(**SD), OSa.DDIMScheduler(**SD)
    a.set_timesteps(5), b.set_timesteps(5)
    x = torch.randn(1, 4, 4, 3, generator=torch.Generator().manual_seed(2))
    for i, t in enumerate(a.timesteps):
        m = x * 0.5
        z = philox_normal(77, i, x.numel()).reshape(x.shape)
        xa = a.step(m, t, x, eta=0.5, seed=77)
        assert torch.equal(xa, b.step(m, t, x, eta=0.5, variance_noise=z))
        x = xa


# ---- DPM-Solver++ 2M SDE -------------------------------------------------------------------------------------------------
SDE_GRID = [dict(timestep_spacing=s, steps_offset=o, use_karras_sigmas=k, use_lu_lambdas=lu)
            for s in ("linspace", "leading", "trailing") for o in (0, 1)
            for k, lu in ((False, False), (True, False), (False, True))]
SDE_GRID += [dict(solver_order=n, lower_order_final=lo, euler_at_final=e, use_karras_sigmas=k)
             for n in (1, 2) for lo in (True, False) for e in (False, True) for k in (False, True)]
SDE_GRID += [dict(SD, use_karras_sigmas=True), dict(lambda_min_clipped=-5.1), dict(beta_schedule="squaredcos_cap_v2")]


def sde_pair(**kw):
    kw = dict(kw, algorithm_type="sde-dpmsolver++")
    return S.DPMSolverMultistepScheduler(**kw), OSa.DPMSolverSDEScheduler(**kw)


@pytest.mark.parametrize("cfg", SDE_GRID, ids=lambda c: "-".join(str(v) for v in c.values()))
@pytest.mark.parametrize("steps", [1, 2, 7, 20, 50])
def test_dpm_sde_host_scalars_are_the_oracles(cfg, steps):
    h, o = sde_pair(**cfg)
    h.set_timesteps(steps), o.set_timesteps(steps)
    assert np.array_equal(h.timesteps, o.timesteps.numpy()) and np.array_equal(h.sigmas, o.sigmas.numpy())
    for t in h.timesteps:
        got, want = h.sde_step_scalars(t), o.step_scalars(torch.tensor(t))
        assert got == want, (t, got, want)
    assert h._step_index == o._step_index == len(h.timesteps)


def kernel_sde(eps, x, m_prev, z, sc):
    """b200mix_dpmpp_2m_sde_step as include/b200mix.h documents it, on fp32 tensors; returns (x_next, x0)."""
    order, sigma_cur, alpha_cur, A, B, halfB, inv_r0, N = sc
    A, B, halfB, inv_r0, N, sigma_cur, alpha_cur = (torch.tensor(v, dtype=torch.float32)
                                                    for v in (A, B, halfB, inv_r0, N, sigma_cur, alpha_cur))
    m0 = (x - sigma_cur * eps) / alpha_cur
    r = A * x + B * m0
    if order == 2:
        r = r + halfB * (inv_r0 * (m0 - m_prev))
    return r + N * z, m0


@pytest.mark.parametrize("cfg", [dict(), dict(use_karras_sigmas=True), dict(use_lu_lambdas=True),
                                 dict(solver_order=1), dict(euler_at_final=True, use_karras_sigmas=True)],
                         ids=["default", "karras", "lu", "order1", "euler_at_final"])
@pytest.mark.parametrize("steps", [5, 20])
def test_dpm_sde_kernel_arithmetic_is_the_oracle_step(cfg, steps):
    h, o = sde_pair(**SD, **cfg)
    h.set_timesteps(steps), o.set_timesteps(steps)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 4, 8, 8, generator=g)
    m_prev = None
    for t in h.timesteps:
        eps, z = torch.randn(x.shape, generator=g), torch.randn(x.shape, generator=g)
        want = o.step(eps, torch.tensor(t), x, noise=z)
        got, m_prev = kernel_sde(eps, x, m_prev, z, h.sde_step_scalars(t))
        assert torch.equal(got, want), t
        x = want


def test_dpm_sde_zero_noise_is_the_reference_formula_with_that_noise():
    """With z = 0 the order-1 SDE update is (sigma_t/sigma_s*exp(-h))*x + (alpha_t*(1 - exp(-2h)))*x0 + 0, which is
    neither the ODE update nor the input."""
    h, o = sde_pair(**SD, solver_order=1)
    ode = OS.DPMSolverMultistepScheduler(**SD, solver_order=1)
    h.set_timesteps(10), o.set_timesteps(10), ode.set_timesteps(10)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(1, 4, 8, 8, generator=g)
    for t in h.timesteps[:5]:
        eps = torch.randn(x.shape, generator=g)
        zero = torch.zeros_like(x)
        want = o.step(eps, torch.tensor(t), x, noise=zero)
        a_t, s_t, lam_t = [v for v in o._lambdas(o._step_index)[0]]
        a_s, s_s, lam_s = [v for v in o._lambdas(o._step_index - 1)[0]]
        hh = lam_t - lam_s
        x0 = (x - s_s * eps) / a_s
        ref = (s_t / s_s * OS.exp_f32(-hh)) * x + (a_t * (1 - OS.exp_f32(-2.0 * hh))) * x0
        ref = ref + s_t * OS.pow_half(1.0 - OS.exp_f32(-2 * hh)) * zero
        assert torch.equal(want, ref)
        assert torch.equal(kernel_sde(eps, x, None, zero, h.sde_step_scalars(t))[0], want)
        assert not torch.equal(want, ode.step(eps, torch.tensor(t), x)) and not torch.equal(want, x)
        x = want


@pytest.mark.parametrize("kw", [dict(algorithm_type="sde-dpmsolver"), dict(algorithm_type="sde-dpmsolver++", solver_type="heun"),
                                dict(algorithm_type="sde-dpmsolver++", solver_order=3),
                                dict(algorithm_type="sde-dpmsolver++", prediction_type="v_prediction")])
def test_dpm_sde_out_of_scope_options_raise(kw):
    with pytest.raises(NotImplementedError):
        S.DPMSolverMultistepScheduler(**kw)


# ---- what each step hands its kernel -------------------------------------------------------------------------------------
class _Recorder:
    def __init__(self):
        self.calls = []

    def __call__(self, name):
        def rec(*args, **kw):
            self.calls.append((name, args, kw))
            return kw.get("out")
        return rec


@pytest.fixture
def recorded(monkeypatch):
    r = _Recorder()
    for name in ("ddim_step", "ddim_eta_step", "dpmpp_2m_step", "dpmpp_2m_sde_step"):
        monkeypatch.setattr(ops, name, r(name))
    return r


def test_ddim_eta_zero_keeps_the_deterministic_call(recorded):
    s = S.DDIMScheduler(**SD)
    s.set_timesteps(4)
    x = torch.zeros(4)
    for t in s.timesteps:
        s.step(x, t, x, eta=0.0, generator=torch.Generator().manual_seed(1))
    assert [c[0] for c in recorded.calls] == ["ddim_step"] * 4
    assert all(c[1][4:8] == s.step_scalars(int(t)) for c, t in zip(recorded.calls, s.timesteps))


def test_ddim_eta_steps_key_philox_by_seed_and_call_index(recorded):
    s = S.DDIMScheduler(**SD)
    for _ in range(2):  # set_timesteps restarts the count and draws a fresh seed from the next generator
        s.set_timesteps(4)
        for t in s.timesteps:
            s.step(torch.zeros(4), t, torch.zeros(4), eta=0.5, generator=torch.Generator().manual_seed(9))
    seed = seed_from(torch.Generator().manual_seed(9))
    assert [(c[2]["seed"], c[2]["step"]) for c in recorded.calls] == [(seed, i) for i in range(4)] * 2
    noise = torch.zeros(4)
    s.set_timesteps(4)
    s.step(torch.zeros(4), s.timesteps[0], torch.zeros(4), eta=0.5, variance_noise=noise)
    assert recorded.calls[-1][1][4] is noise and s._seed is None, "given noise draws no seed"


def test_ddim_refuses_generator_and_variance_noise_together():
    s = S.DDIMScheduler(**SD)
    s.set_timesteps(4)
    x = torch.zeros(4)
    with pytest.raises(ValueError, match="Cannot pass both generator and variance_noise"):
        s.step(x, s.timesteps[0], x, eta=0.5, generator=torch.Generator(), variance_noise=x)
    with pytest.raises(ValueError, match="eta must be"):
        s.step(x, s.timesteps[0], x, eta=-0.1)


def test_dpm_sde_steps_key_philox_by_seed_and_step_index(recorded):
    s = S.DPMSolverMultistepScheduler(**SD, algorithm_type="sde-dpmsolver++")
    s.set_timesteps(6)
    x = torch.zeros(4)
    for t in s.timesteps:
        s.step(x, t, x, generator=torch.Generator().manual_seed(5))
    seed = seed_from(torch.Generator().manual_seed(5))
    assert [(c[2]["seed"], c[2]["step"]) for c in recorded.calls] == [(seed, i) for i in range(6)]
    assert [c[1][5] is None for c in recorded.calls] == [True] + [False] * 4 + [True], "orders 1, 2, 2, 2, 2, 1"
    ode = S.DPMSolverMultistepScheduler(**SD)
    ode.set_timesteps(6)
    ode.step(x, ode.timesteps[0], x, generator=torch.Generator())
    assert recorded.calls[-1][0] == "dpmpp_2m_step"
    with pytest.raises(ValueError, match="takes noise"):
        ode.step(x, ode.timesteps[1], x, noise=x)


def test_schedulers_that_draw_noise_take_the_generator():
    """The pipelines pass their call's generator to exactly these schedulers' steps."""
    takes = {c.__name__ for c in (S.DDIMScheduler, S.LCMScheduler, S.FlowMatchEulerDiscreteScheduler,
                                  S.EulerDiscreteScheduler, S.EulerAncestralDiscreteScheduler,
                                  S.DPMSolverMultistepScheduler, S.UniPCMultistepScheduler)
             if getattr(c, "takes_generator", False)}
    assert takes == {"DDIMScheduler", "EulerAncestralDiscreteScheduler", "DPMSolverMultistepScheduler"}


# ---- the wrappers refuse malformed tensors before any kernel is reached -------------------------------------------------
bf16 = torch.bfloat16
SHAPE = (2, 4, 8, 7)


def _t(dtype=torch.float32, shape=SHAPE):
    return torch.zeros(shape, dtype=dtype)


class _NoKernels:
    def __getattr__(self, name):
        raise AssertionError(f"{name} was reached with invalid inputs")


def _ddim(m_u=None, m_c=None, out=None, noise=None, x=None, m_out=None):
    return ops.ddim_eta_step(_t(bf16) if m_u is None else m_u, _t(bf16) if m_c is None else m_c, 7.5,
                             _t() if x is None else x, noise, 0.9, 0.4, 0.95, 0.2, 0.1, out=out)


def _sde(m_u=None, m_c=None, out=None, noise=None, x=None, m_out=None):
    return ops.dpmpp_2m_sde_step(_t(bf16) if m_u is None else m_u, _t(bf16) if m_c is None else m_c, 7.5,
                                 _t() if x is None else x, noise, _t(), _t() if m_out is None else m_out, 0.9, 0.6, 0.8,
                                 0.1, 0.05, 0.7, 0.3, out=out)


BAD = {
    "short model output": (dict(m_u=_t(bf16, (2, 4, 8, 6))), ValueError, "elements"),
    "strided model output": (dict(m_u=_t(bf16, (2, 4, 7, 8)).transpose(2, 3)), ValueError, "contiguous"),
    "bf16 / fp32 CFG pair": (dict(m_c=_t()), TypeError, "model_output_cond must be"),
    "bf16 out": (dict(out=_t(bf16)), TypeError, "out must be"),
    "strided state": (dict(x=_t(shape=(2, 4, 7, 8)).transpose(2, 3)), ValueError, "contiguous"),
    "short noise": (dict(noise=_t(shape=(2, 4, 8, 6))), ValueError, "noise has"),
    "bf16 noise": (dict(noise=_t(bf16)), TypeError, "noise must be"),
}


@pytest.mark.parametrize("case", list(BAD))
@pytest.mark.parametrize("op", ["ddim_eta_step", "dpmpp_2m_sde_step"])
def test_new_steps_refuse_malformed_inputs_before_launch(op, case, monkeypatch):
    monkeypatch.setattr(ops, "lib", _NoKernels())
    kw, err, pattern = BAD[case]
    with pytest.raises(err, match=pattern):
        (_ddim if op == "ddim_eta_step" else _sde)(**kw)


@pytest.mark.parametrize("bad", [_t(shape=(2, 4, 8, 6)), _t(bf16), None], ids=["short", "bf16", "missing"])
def test_dpm_sde_refuses_a_malformed_history_entry(bad, monkeypatch):
    monkeypatch.setattr(ops, "lib", _NoKernels())
    with pytest.raises((ValueError, TypeError)):
        ops.dpmpp_2m_sde_step(_t(bf16), None, 0.0, _t(), None, None, bad, 0.9, 0.6, 0.8, 0.1, 0.05, 0.7, 0.3)


@pytest.mark.parametrize("op", ["ddim_eta_step", "dpmpp_2m_sde_step"])
@pytest.mark.parametrize("noise", [False, True], ids=["philox", "noise"])
def test_new_steps_pass_well_formed_inputs_to_the_device_check(op, noise, monkeypatch):
    monkeypatch.setattr(ops, "lib", _NoKernels())
    with pytest.raises(_lib.B200MixError, match="CUDA tensor"):
        (_ddim if op == "ddim_eta_step" else _sde)(noise=_t() if noise else None)
