"""ORACLE (test infrastructure, not product code): CPU fp32 restatement of the reference's T2I-Adapter
(ppdiffusers/models/adapter.py: T2IAdapter :216-285, FullAdapter :290-337, FullAdapterXL :340-387, AdapterBlock /
AdapterResnetBlock :390-462, LightAdapter / LightAdapterBlock / LightAdapterResnetBlock :468-583, MultiAdapter :27-100)
and of the adapter pipelines' residual preparation (pipelines/t2i_adapter/pipeline_stable_diffusion_adapter.py:823-836,
pipeline_stable_diffusion_xl_adapter.py:1029-1032).

An adapter config is a dict with the T2IAdapter constructor's keys: in_channels, channels, num_res_blocks,
downscale_factor, adapter_type. Parameter names are the reference's state-dict keys; tensors are NCHW fp32.
"""
from typing import Dict, List, Sequence

import torch
import torch.nn.functional as F

ADAPTER_CONFIGS = {
    # TencentARC/t2iadapter_*_sd14v1 / sd15v2 (FullAdapter at SD1.x widths)
    "sd15": dict(in_channels=3, channels=(320, 640, 1280, 1280), num_res_blocks=2, downscale_factor=8,
                 adapter_type="full_adapter"),
    # TencentARC/t2i-adapter-*-sdxl-1.0 (FullAdapterXL)
    "sdxl": dict(in_channels=3, channels=(320, 640, 1280, 1280), num_res_blocks=2, downscale_factor=16,
                 adapter_type="full_adapter_xl"),
    # the reference's LightAdapter defaults (:473-479)
    "sd15_light": dict(in_channels=3, channels=(320, 640, 1280), num_res_blocks=4, downscale_factor=8,
                       adapter_type="light_adapter"),
    # small adapters whose features fit oracle.unet's tiny_sd / tiny_xl
    "tiny_sd": dict(in_channels=3, channels=(64, 128, 128), num_res_blocks=2, downscale_factor=8,
                    adapter_type="full_adapter"),
    "tiny_xl": dict(in_channels=3, channels=(64, 128, 256, 256), num_res_blocks=2, downscale_factor=16,
                    adapter_type="full_adapter_xl"),
    "tiny_sd_light": dict(in_channels=1, channels=(64, 128), num_res_blocks=2, downscale_factor=8,
                          adapter_type="light_adapter"),
}


def _blocks(cfg):
    """(in_channels, out_channels, down) of every block, as the reference constructs them."""
    ch, t = tuple(cfg["channels"]), cfg["adapter_type"]
    if t == "full_adapter":
        return [(ch[0], ch[0], False)] + [(ch[i - 1], ch[i], True) for i in range(1, len(ch))]
    if t == "full_adapter_xl":
        out = []
        for i in range(len(ch)):
            if i == 1:
                out.append((ch[0], ch[1], False))
            elif i == 2:
                out.append((ch[1], ch[2], True))
            else:
                out.append((ch[i], ch[i], False))
        return out
    if t == "light_adapter":
        cin = cfg["in_channels"] * cfg["downscale_factor"] ** 2
        return ([(cin, ch[0], False)] + [(ch[i], ch[i + 1], True) for i in range(len(ch) - 1)]
                + [(ch[-1], ch[-1], True)])
    raise ValueError(f"Unsupported adapter_type: '{t}'")


def total_downscale_factor(cfg) -> int:
    f, n, t = cfg["downscale_factor"], len(cfg["channels"]), cfg["adapter_type"]
    return {"full_adapter": f * 2 ** (n - 1), "full_adapter_xl": f * 2, "light_adapter": f * 2 ** n}[t]


def adapter_param_shapes(cfg) -> Dict[str, tuple]:
    S = {}

    def conv(name, i, o, k):
        S[name + ".weight"] = (o, i, k, k)
        S[name + ".bias"] = (o,)

    light = cfg["adapter_type"] == "light_adapter"
    if not light:
        conv("adapter.conv_in", cfg["in_channels"] * cfg["downscale_factor"] ** 2, cfg["channels"][0], 3)
    for b, (cin, cout, _) in enumerate(_blocks(cfg)):
        p = f"adapter.body.{b}"
        if light:
            mid = cout // 4
            conv(p + ".in_conv", cin, mid, 1)
            for j in range(cfg["num_res_blocks"]):
                conv(f"{p}.resnets.{j}.block1", mid, mid, 3)
                conv(f"{p}.resnets.{j}.block2", mid, mid, 3)
            conv(p + ".out_conv", mid, cout, 1)
        else:
            if cin != cout:
                conv(p + ".in_conv", cin, cout, 1)
            for j in range(cfg["num_res_blocks"]):
                conv(f"{p}.resnets.{j}.block1", cout, cout, 3)
                conv(f"{p}.resnets.{j}.block2", cout, cout, 1)
    return S


def _conv(x, P, name, k):
    return F.conv2d(x, P[name + ".weight"], P[name + ".bias"], padding=k // 2)


def adapter_forward(cfg, P, image) -> List[torch.Tensor]:
    """T2IAdapter.forward on an NCHW fp32 image: the list of features (NCHW fp32)."""
    light = cfg["adapter_type"] == "light_adapter"
    x = F.pixel_unshuffle(image.float(), cfg["downscale_factor"])
    if not light:
        x = _conv(x, P, "adapter.conv_in", 3)
    feats = []
    for b, (cin, cout, down) in enumerate(_blocks(cfg)):
        p = f"adapter.body.{b}"
        if down:  # nn.AvgPool2D(2, 2, ceil_mode=True), exclusive=True
            x = F.avg_pool2d(x, 2, 2, ceil_mode=True, count_include_pad=False)
        if light or cin != cout:
            x = _conv(x, P, p + ".in_conv", 1)
        for j in range(cfg["num_res_blocks"]):
            h = F.relu(_conv(x, P, f"{p}.resnets.{j}.block1", 3))
            x = _conv(h, P, f"{p}.resnets.{j}.block2", 3 if light else 1) + x
        if light:
            x = _conv(x, P, p + ".out_conv", 1)
        feats.append(x)
    return feats


def multi_adapter_forward(cfgs, Ps, images, adapter_weights=None) -> List[torch.Tensor]:
    """MultiAdapter.forward: sum_k w_k * features_k, default w = 1 / n."""
    n = len(cfgs)
    w = [1.0 / n] * n if adapter_weights is None else list(adapter_weights)
    out = None
    for cfg, P, img, wk in zip(cfgs, Ps, images, w):
        f = adapter_forward(cfg, P, img)
        out = [wk * t for t in f] if out is None else [a + wk * t for a, t in zip(out, f)]
    return out


def pipeline_residuals(features: Sequence[torch.Tensor], scale: float, batch: int, do_cfg: bool) -> List[torch.Tensor]:
    """The adapter state the pipelines hand the UNet (pipeline_stable_diffusion_adapter.py:827-836): features * scale
    (a MultiAdapter's weights are already applied: pass scale 1), tiled to the prompt batch, doubled for CFG."""
    out = []
    for f in features:
        v = f * scale
        if v.shape[0] != batch:
            v = v.repeat(batch // v.shape[0], 1, 1, 1)
        out.append(torch.cat([v, v], 0) if do_cfg else v)
    return out


def residual_steps(num_inference_steps: int, adapter_conditioning_factor: float) -> List[bool]:
    """Per step, whether the UNet gets the adapter residuals (pipeline_stable_diffusion_xl_adapter.py:1029-1032)."""
    return [i < int(num_inference_steps * adapter_conditioning_factor) for i in range(num_inference_steps)]


def adapter_flops(cfg, B, height, width) -> Dict[str, object]:
    """2*MAC of one adapter forward for B images of height x width, and per layer: name, flops and the bytes a bf16
    kernel reads and writes once (input + weights + output; fp32 image input for the pixel unshuffle)."""
    light = cfg["adapter_type"] == "light_adapter"
    f = cfg["downscale_factor"]
    h, w, c = height // f, width // f, cfg["in_channels"] * f * f
    layers = [dict(name="pixel_unshuffle", flops=0, bytes=B * height * width * cfg["in_channels"] * (4 + 2))]

    def conv(name, cin, cout, k):
        fl = 2 * B * h * w * k * k * cin * cout
        layers.append(dict(name=name, flops=fl, bytes=2 * (B * h * w * (cin + cout) + k * k * cin * cout)))

    if not light:
        conv("conv_in", c, cfg["channels"][0], 3)
    for b, (cin, cout, down) in enumerate(_blocks(cfg)):
        if down:
            h2, w2 = (h + 1) // 2, (w + 1) // 2
            layers.append(dict(name=f"body.{b}.pool", flops=0, bytes=2 * B * cin * (h * w + h2 * w2)))
            h, w = h2, w2
        mid = cout // 4 if light else cout
        if light or cin != cout:
            conv(f"body.{b}.in_conv", cin, mid, 1)
        for j in range(cfg["num_res_blocks"]):
            conv(f"body.{b}.resnets.{j}.block1", mid, mid, 3)
            layers.append(dict(name=f"body.{b}.resnets.{j}.relu", flops=0, bytes=2 * 2 * B * h * w * mid))
            conv(f"body.{b}.resnets.{j}.block2", mid, mid, 3 if light else 1)
        if light:
            conv(f"body.{b}.out_conv", mid, cout, 1)
    return dict(total=sum(x["flops"] for x in layers), layers=layers)
