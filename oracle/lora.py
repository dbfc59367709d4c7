"""ORACLE (test infrastructure, not product code): the reference's LoRA merge in fp32, Paddle layout.

LoRACompatibleLinear._fuse_lora (ppdiffusers/models/lora.py:117-144): W [in, out] + s * (down [in, r] @ up [r, out]),
with up scaled by network_alpha / rank (:123-130). LoRACompatibleConv._fuse_lora (:312-338):
W [out, in, kh, kw] + s * reshape(up.flatten(1) @ down.flatten(1)). The legacy attention-processor names are mapped as
UNet2DConditionLoadersMixin.convert_state_dict_legacy_attn_format does (loaders/unet.py:423-445).
oracle.unet.unet_forward then runs on the merged parameters.
"""
from typing import Dict, Optional

import torch


def legacy_to_layer(key: str) -> str:
    """'...attn1.processor.to_out_lora.up.weight' -> '...attn1.to_out.0.lora.up.weight' (loaders/unet.py:435-439)."""
    if "processor" not in key.split("."):
        return key
    return key.replace(".processor", "").replace("to_out_lora", "to_out.0.lora").replace("_lora", ".lora")


def layer_delta(P, layer: str, down: torch.Tensor, up: torch.Tensor, alpha: Optional[float]) -> torch.Tensor:
    """The reference's fp32 weight update of one layer (scale 1) in the layer's own Paddle layout."""
    down, up = down.float(), up.float()
    if alpha is not None:
        rank = down.shape[1] if P[layer + ".weight"].dim() == 2 else down.shape[0]
        up = up * alpha / rank
    w = P[layer + ".weight"]
    if w.dim() == 2:
        return down @ up
    return (up.flatten(1) @ down.flatten(1)).reshape(w.shape)


def merge(P: Dict[str, torch.Tensor], loras, device=None) -> Dict[str, torch.Tensor]:
    """P: reference-named fp32 parameters. loras: list of (state_dict, network_alphas, scale): state_dict in
    ppdiffusers naming ('<layer>.lora.down.weight', optionally legacy processor names or a 'unet.' prefix) and
    Paddle layout; network_alphas {'<layer>.alpha': a} or None. Returns P with every W replaced by
    W + sum_i scale_i * dW_i, summed in fp32."""
    out = dict(P)
    for sd, alphas, scale in loras:
        alphas = {legacy_to_layer(k.replace("unet.", "", 1))[: -len(".alpha")]: v for k, v in (alphas or {}).items()}
        groups: Dict[str, Dict[str, torch.Tensor]] = {}
        for k, v in sd.items():
            k = legacy_to_layer(k[len("unet."):] if k.startswith("unet.") else k)
            layer, kind = k.rsplit(".lora.", 1)[0], k.split(".")[-2]
            groups.setdefault(layer, {})[kind] = v
        for layer, f in groups.items():
            d = layer_delta(P, layer, f["down"], f["up"], alphas.get(layer))
            w = out[layer + ".weight"].float()
            out[layer + ".weight"] = w + scale * d.to(w.device)
    return out
