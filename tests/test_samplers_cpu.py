"""Euler-ancestral and UniPC without a GPU: the oracle against the reference's goldens and the pinned Euler oracle,
the host schedulers' scalars bit for bit against the oracle, the options outside the device step, the wrappers'
input checks, the seed drawn from a generator, and DPM-Solver's schedule under the shared schedule helper."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import samplers as OSa
from oracle import schedulers as OS
from paddlemix_b200 import _lib, ops
from paddlemix_b200.ppdiffusers import EulerAncestralDiscreteScheduler, UniPCMultistepScheduler
from paddlemix_b200.ppdiffusers import schedulers as S
from paddlemix_b200.sampling import seed_from

GOLD = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "unipc_goldens.json")))


def deter(kind, flip=False):  # test_schedulers.py:261-290 (4d), test_scheduler_unipc.py:299-325 (1d)
    shape = (3, 8, 8, 4) if kind == "4d" else (3, 8, 4)
    n = int(np.prod(shape))
    s = torch.arange(n)
    s = (s.flip(-1) if flip else s).reshape(shape) / n
    return s.permute(3, 0, 1, 2) if kind == "4d" else s.permute(2, 0, 1)


def model(sample, t):  # test_schedulers.py:295-303
    return sample * t / (t + 1)


@pytest.mark.parametrize("kind", ["4d", "1d"])
def test_oracle_unipc_matches_reference_goldens(kind):
    fx = GOLD["fixtures"][kind]
    for case in fx["full_loop"]:
        sch = OSa.UniPCMultistepScheduler(**{**GOLD["config"], **case["config"]})
        sch.set_timesteps(GOLD["num_inference_steps"])
        x = deter(kind)
        for t in sch.timesteps:
            x = sch.step(model(x, t), t, x)
        assert abs(x.abs().mean().item() - case["mean"]) < GOLD["mean_atol"], (case, x.abs().mean().item())
    g = fx["full_loop_with_noise"]
    sch = OSa.UniPCMultistepScheduler(**GOLD["config"])
    sch.set_timesteps(GOLD["num_inference_steps"])
    timesteps = sch.timesteps[g["t_start"]:]
    x = sch.add_noise(deter(kind), deter(kind, flip=True), timesteps[:1])
    for t in timesteps:
        x = sch.step(model(x, t), t, x)
    assert abs(x.abs().sum().item() - g["sum"]) < GOLD["sum_atol"]
    assert abs(x.abs().mean().item() - g["mean"]) < GOLD["mean_atol"]


@pytest.mark.parametrize("prediction_type", ["epsilon", "v_prediction"])
def test_oracle_euler_ancestral_without_noise_is_the_euler_step_to_sigma_down(prediction_type):
    kw = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", prediction_type=prediction_type)
    a, e = OSa.EulerAncestralDiscreteScheduler(**kw), OS.EulerDiscreteScheduler(**kw)
    a.set_timesteps(8), e.set_timesteps(8)
    x = deter("4d") * 10
    for t in a.timesteps:
        if a._step_index is None:
            a._init_step_index(t)
        _, sigma_down = a.sigmas_up_down()
        i = a._step_index
        e._step_index = i
        e.sigmas = a.sigmas.clone()
        e.sigmas[i + 1] = sigma_down
        m = model(x, t) - 0.3
        want = e.step(m, t, x)
        got = a.step(m, t, x, torch.zeros_like(x))
        assert torch.equal(got, want)
        x = got


EA_GRID = [dict(timestep_spacing=s, steps_offset=o, beta_schedule=b, prediction_type=p)
           for s in ("linspace", "leading", "trailing") for o in (0, 1)
           for b in ("linear", "scaled_linear", "squaredcos_cap_v2") for p in ("epsilon", "v_prediction")]


@pytest.mark.parametrize("cfg", EA_GRID, ids=lambda c: "-".join(str(v) for v in c.values()))
@pytest.mark.parametrize("steps", [1, 2, 25])
def test_euler_ancestral_host_scalars_are_the_oracles(cfg, steps):
    if cfg["beta_schedule"] == "scaled_linear":
        cfg = dict(cfg, beta_start=0.00085, beta_end=0.012)
    h, o = EulerAncestralDiscreteScheduler(**cfg), OSa.EulerAncestralDiscreteScheduler(**cfg)
    h.set_timesteps(steps), o.set_timesteps(steps)
    assert np.array_equal(h.timesteps, o.timesteps.numpy()) and np.array_equal(h.sigmas, o.sigmas.numpy())
    assert h.init_noise_sigma == float(o.init_noise_sigma)
    for t in h.timesteps:
        if o._step_index is None:
            o._init_step_index(torch.tensor(t))
        want = o.step_scalars()
        o._step_index += 1
        assert h.step_scalars(t) == want


UNIPC_GRID = ([dict(timestep_spacing=s, steps_offset=o, use_karras_sigmas=k)
               for s in ("linspace", "leading", "trailing") for o in (0, 1) for k in (False, True)] +
              [dict(solver_order=n, solver_type=b, lower_order_final=lo, use_karras_sigmas=k)
               for n in (1, 2, 3) for b in ("bh1", "bh2") for lo in (True, False) for k in (False, True)] +
              [dict(solver_order=3, disable_corrector=[0, 2, 5]), dict(solver_order=2, disable_corrector=[1]),
               dict(prediction_type="sample", solver_order=3), dict(prediction_type="v_prediction", solver_order=3),
               dict(beta_schedule="scaled_linear", beta_start=0.00085, beta_end=0.012, solver_order=3),
               dict(beta_schedule="squaredcos_cap_v2", solver_order=3, solver_type="bh1")])


def _same(a, b):
    """Equal as floats, with nan equal to nan (the Karras final step without lower_order_final)."""
    if isinstance(a, list):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if isinstance(a, float) and np.isnan(a):
        return isinstance(b, float) and np.isnan(b)
    return a == b and (not isinstance(a, float) or np.signbit(a) == np.signbit(b))


@pytest.mark.parametrize("cfg", UNIPC_GRID, ids=lambda c: "-".join(str(v) for v in c.values()))
@pytest.mark.parametrize("steps", [1, 2, 10, 20])
def test_unipc_host_scalars_are_the_oracles(cfg, steps):
    h, o = UniPCMultistepScheduler(**cfg), OSa.UniPCMultistepScheduler(**cfg)
    h.set_timesteps(steps), o.set_timesteps(steps)
    assert np.array_equal(h.timesteps, o.timesteps.numpy()) and np.array_equal(h.sigmas, o.sigmas.numpy())
    for t in h.timesteps:
        got, want = h.step_scalars(t), o.step_scalars(torch.tensor(t))
        assert got.keys() == want.keys() and all(_same(got[k], want[k]) for k in got), (t, got, want)


def test_unipc_starts_in_the_middle_of_a_schedule():
    h, o = UniPCMultistepScheduler(solver_order=3), OSa.UniPCMultistepScheduler(solver_order=3)
    h.set_timesteps(10), o.set_timesteps(10)
    for t in h.timesteps[4:]:
        got, want = h.step_scalars(t), o.step_scalars(torch.tensor(t))
        assert all(_same(got[k], want[k]) for k in got)
    assert h.step_index == 10


@pytest.mark.parametrize("kw", [dict(thresholding=True), dict(predict_x0=False), dict(solver_p=object()),
                                dict(solver_order=4), dict(trained_betas=[0.1] * 1000)])
def test_unipc_out_of_scope_options_raise(kw):
    with pytest.raises(NotImplementedError):
        UniPCMultistepScheduler(**kw)


def test_unipc_maps_dpm_solver_types_to_bh2():
    assert UniPCMultistepScheduler(solver_type="midpoint").solver_type == "bh2"
    with pytest.raises(NotImplementedError):
        UniPCMultistepScheduler(solver_type="nope")


@pytest.mark.parametrize("kw", [dict(prediction_type="sample"), dict(trained_betas=[0.1] * 1000)])
def test_euler_ancestral_out_of_scope_options_raise(kw):
    with pytest.raises(NotImplementedError):
        EulerAncestralDiscreteScheduler(**kw)


DPM_GRID = [dict(timestep_spacing=s, steps_offset=o, use_karras_sigmas=k, use_lu_lambdas=lu)
            for s in ("linspace", "leading", "trailing") for o in (0, 1) for k, lu in ((False, False), (True, False),
                                                                                        (False, True))]
DPM_GRID += [dict(lambda_min_clipped=-5.1), dict(lambda_min_clipped=-5.1, timestep_spacing="trailing")]


@pytest.mark.parametrize("cfg", DPM_GRID, ids=lambda c: "-".join(str(v) for v in c.values()))
@pytest.mark.parametrize("steps", [1, 7, 25])
def test_dpm_solver_schedule_is_unchanged_by_the_shared_helper(cfg, steps):
    h, o = S.DPMSolverMultistepScheduler(**cfg), OS.DPMSolverMultistepScheduler(**cfg)
    h.set_timesteps(steps), o.set_timesteps(steps)
    assert np.array_equal(h.timesteps, o.timesteps.numpy()) and np.array_equal(h.sigmas, o.sigmas.numpy())
    assert h.num_inference_steps == o.num_inference_steps


def test_seed_from_a_generator_is_deterministic():
    a, b = seed_from(torch.Generator().manual_seed(7)), seed_from(torch.Generator().manual_seed(7))
    assert a == b and 0 <= a < 2 ** 63 and a != seed_from(torch.Generator().manual_seed(8))
    torch.manual_seed(11)
    c = seed_from(None)
    torch.manual_seed(11)
    assert seed_from(None) == c


# ---- the wrappers refuse malformed tensors before any kernel is reached (CPU tensors show every other refusal) ------
bf16 = torch.bfloat16
SHAPE = (2, 4, 8, 8)


def _t(dtype=torch.float32, shape=SHAPE):
    return torch.zeros(shape, dtype=dtype)


class _NoKernels:
    def __getattr__(self, name):
        raise AssertionError(f"{name} was reached with invalid inputs")


COEFFS = dict(alpha_t=0.5, sigma_t=0.8, A_c=0.9, K_c=-0.1, E_c=-0.1, rc_last=0.5, rc=[0.1], rk_c=[-0.9], A_p=0.9,
              K_p=-0.1, E_p=-0.1, rp=[0.5], rk_p=[-0.9])


def _ea(m_u=None, m_c=None, out=None, noise=None, x=None):
    return ops.euler_ancestral_step(_t(bf16) if m_u is None else m_u, _t(bf16) if m_c is None else m_c, 7.5,
                                    _t() if x is None else x, noise, 0.9, -0.6, 1.8, -0.2, 0.1, out=out)


def _unipc(m_u=None, m_c=None, out=None, hist=None, last=None, m_out=None):
    return ops.unipc_step(_t(bf16) if m_u is None else m_u, _t(bf16) if m_c is None else m_c, 7.5, _t(), COEFFS,
                          _t() if m_out is None else m_out, _t(), last_sample=_t() if last is None else last,
                          m_prev=_t(), hist_c=[_t() if hist is None else hist], hist_p=[_t()], out=out)


BAD = {
    "short model output": (lambda f: f(m_u=_t(bf16, (2, 4, 8, 7))), ValueError, "elements"),
    "strided model output": (lambda f: f(m_u=_t(bf16).transpose(2, 3)), ValueError, "contiguous"),
    "bf16 / fp32 CFG pair": (lambda f: f(m_c=_t(torch.float32)), TypeError, "model_output_cond must be"),
    "bf16 out": (lambda f: f(out=_t(bf16)), TypeError, "out must be"),
    "strided state": (lambda f: f(x=_t().transpose(2, 3)) if f is _ea else f(last=_t().transpose(2, 3)), ValueError,
                      "contiguous"),
}


@pytest.mark.parametrize("case", list(BAD))
@pytest.mark.parametrize("op", ["euler_ancestral_step", "unipc_step"])
def test_new_steps_refuse_malformed_inputs_before_launch(op, case, monkeypatch):
    monkeypatch.setattr(ops, "lib", _NoKernels())
    make, err, pattern = BAD[case]
    with pytest.raises(err, match=pattern):
        make(_ea if op == "euler_ancestral_step" else _unipc)


@pytest.mark.parametrize("bad", [_t(shape=(2, 4, 8, 7)), _t(bf16), _t().transpose(2, 3)], ids=["short", "bf16", "strided"])
def test_euler_ancestral_refuses_malformed_noise(bad, monkeypatch):
    monkeypatch.setattr(ops, "lib", _NoKernels())
    with pytest.raises((ValueError, TypeError)):
        _ea(noise=bad)


@pytest.mark.parametrize("bad", [_t(shape=(2, 4, 8, 7)), _t(bf16), _t().transpose(2, 3)], ids=["short", "bf16", "strided"])
@pytest.mark.parametrize("where", ["history", "m_out"])
def test_unipc_refuses_malformed_history(bad, where, monkeypatch):
    monkeypatch.setattr(ops, "lib", _NoKernels())
    with pytest.raises((ValueError, TypeError)):
        _unipc(hist=bad) if where == "history" else _unipc(m_out=bad)


def test_unipc_refuses_corrector_history_without_the_corrector(monkeypatch):
    monkeypatch.setattr(ops, "lib", _NoKernels())
    with pytest.raises(ValueError, match="go together"):
        ops.unipc_step(_t(bf16), None, 0.0, _t(), COEFFS, _t(), _t(), hist_c=[_t()])
    with pytest.raises(ValueError, match="at most two"):
        ops.unipc_step(_t(bf16), None, 0.0, _t(), COEFFS, _t(), _t(), hist_p=[_t()] * 3)


@pytest.mark.parametrize("op", ["euler_ancestral_step", "unipc_step"])
def test_new_steps_pass_well_formed_inputs_to_the_device_check(op, monkeypatch):
    monkeypatch.setattr(ops, "lib", _NoKernels())
    with pytest.raises(_lib.B200MixError, match="CUDA tensor"):
        _ea() if op == "euler_ancestral_step" else _unipc()


def test_unipc_coeffs_mirror_the_header_layout():
    """b200mix_unipc_coeffs is 17 floats in declaration order."""
    import ctypes
    assert ctypes.sizeof(_lib.UnipcCoeffs) == 17 * 4
    assert _lib.UnipcCoeffs.A_p.offset == 10 * 4 and _lib.UnipcCoeffs.rk_p.offset == 15 * 4
