"""Host-side parameter plumbing shared by every model class: the read-only config dict, fp32 views of reference-named
parameters in the Paddle layout, zero-padding of attention heads to the attention kernel's width, synthetic weights
and the preamble of every load_state_dict (missing-key check, device binding).

Each model keeps only what is its own: parameter names and shapes (state_dict_shapes) and the fused device layout its
load_state_dict builds from them. Nothing here touches the GPU except bind(), which initialises the library on the
model's device.
"""
import math
from typing import Any, Callable, Dict, Optional, Union

import numpy as np
import torch

bf16 = torch.bfloat16


class FrozenDict(dict):
    """Attribute-style read-only config, like ppdiffusers.configuration_utils.FrozenDict (:58)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        raise Exception(f"You cannot use ``__setattr__`` on a {self.__class__.__name__} instance.")


def to_f32(x) -> torch.Tensor:
    """fp32 view of a parameter on whatever device it already lives on (host numpy / torch, or CUDA)."""
    if isinstance(x, np.ndarray):
        x = torch.from_numpy(x)
    return x.detach().to(torch.float32)


def linear_weight(P: Dict[str, Any], name: str) -> torch.Tensor:
    """P[name + ".weight"], a Paddle Linear weight [in, out], as the fp32 contiguous [out, in] the GEMMs take."""
    return to_f32(P[name + ".weight"]).t().contiguous()


def linear_bias(P: Dict[str, Any], name: str) -> torch.Tensor:
    """P[name + ".bias"] as fp32."""
    return to_f32(P[name + ".bias"])


def device_linear(P: Dict[str, Any], name: str, dev: torch.device):
    """A Linear as ops.linear takes it: (bf16 [out, in] weight, fp32 bias) on dev."""
    return linear_weight(P, name).to(dev, bf16), device_vector(P, name + ".bias", dev)


def device_vector(P: Dict[str, Any], key: str, dev: torch.device) -> torch.Tensor:
    """P[key] (a bias, norm weight or table) as a contiguous fp32 tensor on dev."""
    return to_f32(P[key]).contiguous().to(dev)


# ---- attention heads zero-padded to the attention kernel's head width (exact: the padded lanes of q, k and v are 0,
# and the out-projection's padded input columns are 0) ------------------------------------------------------------------
def pad_head_width(d: int) -> int:
    """The head width the sm_90a attention kernel runs a head of size d at."""
    for p in (64, 128, 192):
        if d <= p:
            return p
    raise ValueError(f"attention head size {d} > 192 is not supported by the sm_90a attention kernel")


def pad_head_rows(w: torch.Tensor, heads: int, d: int, dp: int) -> torch.Tensor:
    """[heads * d, in] -> [heads * dp, in] (a q / k / v projection's output rows)."""
    if d == dp:
        return w
    out = torch.zeros(heads, dp, w.shape[-1], device=w.device)
    out[:, :d] = w.reshape(heads, d, -1)
    return out.reshape(heads * dp, -1)


def pad_head_vec(b: torch.Tensor, heads: int, d: int, dp: int) -> torch.Tensor:
    """[heads * d] -> [heads * dp] (a q / k / v projection's bias)."""
    if d == dp:
        return b
    out = torch.zeros(heads, dp, device=b.device)
    out[:, :d] = b.reshape(heads, d)
    return out.reshape(-1)


def pad_head_cols(w: torch.Tensor, heads: int, d: int, dp: int) -> torch.Tensor:
    """[out, heads * d] -> [out, heads * dp] (the out-projection's input columns)."""
    if d == dp:
        return w
    out = torch.zeros(w.shape[0], heads, dp, device=w.device)
    out[:, :, :d] = w.reshape(w.shape[0], heads, d)
    return out.reshape(w.shape[0], heads * dp)


# ---- loading ----------------------------------------------------------------------------------------------------------
def _device(device: Union[int, str, torch.device]) -> torch.device:
    return torch.device("cuda", device) if isinstance(device, int) else torch.device(device)


def synthetic_state_dict(shapes: Dict[str, tuple], seed: int, device: Union[int, str, torch.device],
                         special: Optional[Callable[[str, tuple, Callable], Optional[torch.Tensor]]] = None
                         ) -> Dict[str, torch.Tensor]:
    """Random bf16 weights for a state dict's names and shapes, drawn on `device` (there are no checkpoints offline):
    U(-1/sqrt(fan_in), 1/sqrt(fan_in)) matrices and filters (fan_in = shape[0] for a Paddle Linear [in, out], the
    product of the other axes for a conv filter [out, in, k...]), norm scales 1 + 0.1 N, biases 0.05 N. One generator
    seeded once draws every tensor in sorted name order, so a seed gives the same weights on the same device type.
    special(name, shape, randn) may return a tensor for a parameter that a model draws differently (randn(shape) draws
    from the same generator); None applies the rule."""
    dev = _device(device)
    g = torch.Generator(device=dev).manual_seed(seed)

    def randn(shp):
        return torch.randn(shp, generator=g, device=dev)

    def rule(name, shp):
        if name.endswith(".weight") and len(shp) >= 2:
            fan_in = shp[0] if len(shp) == 2 else math.prod(shp[1:])
            return (torch.rand(shp, generator=g, device=dev) * 2 - 1) / fan_in ** 0.5
        if name.endswith(".weight"):
            return 1.0 + 0.1 * randn(shp)
        return 0.05 * randn(shp)

    P = {}
    for name, shp in sorted(shapes.items()):
        t = None if special is None else special(name, shp, randn)
        P[name] = (rule(name, shp) if t is None else t).to(bf16)
    return P


def bind(model, P: Dict[str, Any], device: Union[int, str, torch.device]) -> torch.device:
    """The start of every load_state_dict: refuses a state dict that lacks any of model.state_dict_shapes() (before any
    device work), then initialises the library on `device` (an int means cuda:N) and sets model.device."""
    missing = [k for k in model.state_dict_shapes() if k not in P]
    if missing:
        raise KeyError(f"state dict is missing {len(missing)} parameters, e.g. {missing[:3]}")
    from . import ops
    dev = _device(device)
    ops.init(dev.index or 0)
    model.device = dev
    return dev
