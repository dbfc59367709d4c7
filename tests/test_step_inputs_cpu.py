"""The sampler-step wrappers refuse malformed tensors before anything reaches a kernel. The kernels read every tensor
flat over the state's element count and read the CFG pair with one dtype flag, so a short, strided or mixed-dtype input
would otherwise be read out of bounds or silently misread. The checks run before the CUDA-placement check, so CPU
tensors show them here."""
import pytest
import torch

from paddlemix_b200 import _lib, ops

bf16 = torch.bfloat16
SHAPE = (2, 4, 8, 8)
OPS = ["ddim_step", "lcm_step", "euler_step", "dpmpp_2m_step", "cfg_combine"]


def _t(dtype=torch.float32, shape=SHAPE):
    return torch.zeros(shape, dtype=dtype)


def _call(op, m_u, m_c, out):
    x = _t()
    if op == "ddim_step":
        return ops.ddim_step(m_u, m_c, 7.5, x, 0.5, 0.8, 0.6, 0.7, "v_prediction", 1.0, out=out)
    if op == "lcm_step":
        return ops.lcm_step(m_u, m_c, 7.5, x, _t(), 0.5, 0.8, 0.1, 0.9, 0.6, 0.7, out=out, denoised=_t())
    if op == "euler_step":
        return ops.euler_step(m_u, m_c, 7.5, x, 0.9, -0.1, out=out)
    if op == "dpmpp_2m_step":
        return ops.dpmpp_2m_step(m_u, m_c, 7.5, x, _t(), _t(), 0.9, 0.4, 0.9, -0.1, -0.05, 1.0, out=out)
    return ops.cfg_combine(m_u, m_c, 7.5, guidance_rescale=0.7, out=out)


class _NoKernels:
    def __getattr__(self, name):
        raise AssertionError(f"{name} was reached with invalid inputs")


BAD = {  # (model output, model_output_cond, out), the error it must raise, a pattern of its message
    "short model output": (lambda: (_t(bf16, (2, 4, 8, 7)), _t(bf16), None), ValueError, "elements"),
    "strided model output": (lambda: (_t(bf16).transpose(2, 3), _t(bf16), None), ValueError, "contiguous"),
    "bf16 / fp32 CFG pair": (lambda: (_t(bf16), _t(torch.float32), None), TypeError, "model_output_cond must be"),
    "bf16 out": (lambda: (_t(bf16), _t(bf16), _t(bf16)), TypeError, "out must be"),
}


@pytest.mark.parametrize("case", list(BAD))
@pytest.mark.parametrize("op", OPS)
def test_step_refuses_malformed_inputs_before_launch(op, case, monkeypatch):
    monkeypatch.setattr(ops, "lib", _NoKernels())
    make, err, pattern = BAD[case]
    with pytest.raises(err, match=pattern):
        _call(op, *make())


@pytest.mark.parametrize("op", OPS)
def test_step_passes_well_formed_inputs_to_the_device_check(op, monkeypatch):
    monkeypatch.setattr(ops, "lib", _NoKernels())
    with pytest.raises(_lib.B200MixError, match="CUDA tensor"):
        _call(op, _t(bf16), _t(bf16), _t())
