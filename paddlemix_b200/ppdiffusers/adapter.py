"""T2IAdapter / MultiAdapter — host-side mirrors of ppdiffusers.models.adapter (ppdiffusers/models/adapter.py:27-583) on
the sm_90a kernels. An adapter turns a control image into one feature map per UNet down block; the UNet adds them as
`down_intrablock_additional_residuals`. It does not depend on the timestep, so pipelines run it once per call.

Per block (the reference's AdapterBlock :390-435 and LightAdapterBlock :515-555), on bf16 NHWC:
  * the input image goes through b200mix_pixel_unshuffle (NCHW fp32 / bf16 -> NHWC bf16, C * f^2 channels);
  * full_adapter / full_adapter_xl: conv_in on the wgmma conv3x3, then per block an optional 2x2 average pool
    (b200mix_avgpool2x2_nhwc), an optional 1x1 in_conv (ops.linear on the pixel rows) and num_res_blocks x
    [conv3x3 -> ReLU (b200mix_activation) -> 1x1 conv with the block input added in the GEMM epilogue];
  * light_adapter: pool, 1x1 in_conv to out/4 channels, num_res_blocks x [conv3x3 -> ReLU -> conv3x3 + input], 1x1
    out_conv. The mid channels (80 / 160 / 320 for the default config) are zero-padded at load to a multiple of 64, the
    wgmma conv3x3's Cin granule: the padded filters and biases are zero, so the padded channels stay zero through ReLU
    and the residual adds and the out_conv's zero columns leave the features unchanged.
"""
from typing import Any, Dict, List, Optional, Sequence, Union

import torch
import torch.nn.functional as F

from ..modeling import FrozenDict, bind, synthetic_state_dict
from .unet_2d_condition import _Conv3x3, _Linear

bf16 = torch.bfloat16
ADAPTER_TYPES = ("full_adapter", "full_adapter_xl", "light_adapter")


def _pad64(c: int) -> int:
    return -(-c // 64) * 64


class _Block:
    """One AdapterBlock / LightAdapterBlock: down (2x2 average pool first), in_conv (1x1, or None), resnets
    [(block1, block2)], out_conv (light adapter only)."""

    def __init__(self, name, cin, cout, num_res_blocks, down, light):
        self.down, self.light, self.cout = down, light, cout
        if light:
            mid = cout // 4
            self.in_conv = _Linear(f"{name}.in_conv", cin, mid, conv1x1=True)
            self.resnets = [(_Conv3x3(f"{name}.resnets.{j}.block1", mid, mid), _Conv3x3(f"{name}.resnets.{j}.block2", mid, mid))
                            for j in range(num_res_blocks)]
            self.out_conv = _Linear(f"{name}.out_conv", mid, cout, conv1x1=True)
        else:
            self.in_conv = _Linear(f"{name}.in_conv", cin, cout, conv1x1=True) if cin != cout else None
            self.resnets = [(_Conv3x3(f"{name}.resnets.{j}.block1", cout, cout),
                             _Linear(f"{name}.resnets.{j}.block2", cout, cout, conv1x1=True)) for j in range(num_res_blocks)]
            self.out_conv = None

    def leaves(self):
        out = [self.in_conv] + [m for r in self.resnets for m in r] + [self.out_conv]
        return [m for m in out if m is not None]

    def pad_mid(self):
        """Light adapter: zero-pad the mid channels of the loaded device weights to a multiple of 64 (exact)."""
        mid = self.in_conv.cout
        p = _pad64(mid) - mid
        if not p:
            return
        self.in_conv.w = F.pad(self.in_conv.w, (0, 0, 0, p)).contiguous()       # [mid + p, cin]
        self.in_conv.b = F.pad(self.in_conv.b, (0, p)).contiguous()
        for b1, b2 in self.resnets:
            for conv in (b1, b2):                                                # [O, 3, 3, I]
                conv.w = F.pad(conv.w, (0, p, 0, 0, 0, 0, 0, p)).contiguous()
                conv.b = F.pad(conv.b, (0, p)).contiguous()
        self.out_conv.w = F.pad(self.out_conv.w, (0, p)).contiguous()           # [cout, mid + p]


class T2IAdapter:
    """Drop-in for ppdiffusers.T2IAdapter (models/adapter.py:216-285) in inference."""

    def __init__(self, in_channels: int = 3, channels: Sequence[int] = (320, 640, 1280, 1280), num_res_blocks: int = 2,
                 downscale_factor: int = 8, adapter_type: str = "full_adapter"):
        if adapter_type not in ADAPTER_TYPES:
            raise ValueError(f"Unsupported adapter_type: '{adapter_type}'. Choose either 'full_adapter' or "
                             "'full_adapter_xl' or 'light_adapter'.")
        ch = tuple(int(c) for c in channels)
        self.config = FrozenDict(in_channels=in_channels, channels=ch, num_res_blocks=num_res_blocks,
                                 downscale_factor=downscale_factor, adapter_type=adapter_type)
        self.device = None
        self._check_supported()
        light = adapter_type == "light_adapter"
        cin = in_channels * downscale_factor ** 2
        self.conv_in = None if light else _Conv3x3("adapter.conv_in", cin, ch[0])
        b = "adapter.body"
        if adapter_type == "full_adapter":  # :309-319
            spec = [(ch[0], ch[0], False)] + [(ch[i - 1], ch[i], True) for i in range(1, len(ch))]
            self.total_downscale_factor = downscale_factor * 2 ** (len(ch) - 1)
        elif adapter_type == "full_adapter_xl":  # :359-371: one downsampling block, at index 2
            spec = [(ch[i - 1], ch[i], i == 2) if i in (1, 2) else (ch[i], ch[i], False) for i in range(len(ch))]
            self.total_downscale_factor = downscale_factor * 2
        else:  # :486-497
            spec = ([(cin, ch[0], False)] + [(ch[i], ch[i + 1], True) for i in range(len(ch) - 1)]
                    + [(ch[-1], ch[-1], True)])
            self.total_downscale_factor = downscale_factor * 2 ** len(ch)
        self.blocks = [_Block(f"{b}.{i}", ci, co, num_res_blocks, down, light) for i, (ci, co, down) in enumerate(spec)]

    def _check_supported(self):
        """Refuses, before any device work, configs whose channel counts no kernel takes."""
        c = self.config
        if c.downscale_factor not in (8, 16):
            raise NotImplementedError(f"T2IAdapter(b200): downscale_factor {c.downscale_factor} (b200mix_pixel_unshuffle "
                                      "takes 8 or 16)")
        if c.adapter_type == "light_adapter":
            bad = [x for x in c.channels if x % 8]
            need = "multiples of 8 (2x2 pool and 1x1 convs on 16-byte channel vectors)"
        else:
            bad = [x for x in c.channels if x % 64]
            need = "multiples of 64 (the wgmma conv3x3 takes Cin % 64 == 0)"
        if bad or not c.channels or c.num_res_blocks < 0:
            raise NotImplementedError(f"T2IAdapter(b200) {c.adapter_type}: channels {c.channels} must be {need}")
        if c.adapter_type == "full_adapter_xl" and any(c.channels[i] != c.channels[i - 1] for i in range(3, len(c.channels))):
            raise NotImplementedError(f"T2IAdapter(b200) full_adapter_xl: channels {c.channels} (blocks 3.. take channels[i] "
                                      "as their input, so they must repeat channels[2], models/adapter.py:361-367)")

    @property
    def downscale_factor(self) -> int:
        """The factor of the initial pixel unshuffle; image sides must be multiples of it."""
        return self.config.downscale_factor

    def _leaves(self):
        return ([self.conv_in] if self.conv_in is not None else []) + [m for blk in self.blocks for m in blk.leaves()]

    def state_dict_shapes(self) -> Dict[str, tuple]:
        """Names and shapes of the reference state dict (Paddle layouts)."""
        out = {}
        for m in self._leaves():
            out.update(m.shapes())
        return out

    def init_synthetic_weights(self, seed: int = 1, device: Union[int, str] = 0):
        return self.load_state_dict(synthetic_state_dict(self.state_dict_shapes(), seed, device), device)

    def load_state_dict(self, state_dict: Dict[str, Any], device: Union[int, str] = 0):
        dev = bind(self, state_dict, device)
        for m in self._leaves():
            m.load(state_dict, dev)
        for blk in self.blocks:
            if blk.light:
                blk.pad_mid()
        return self

    def feature_shapes(self, height: int, width: int) -> List[tuple]:
        """(h, w, channels) of every feature for a height x width image."""
        h, w = height // self.downscale_factor, width // self.downscale_factor
        out = []
        for blk in self.blocks:
            if blk.down:
                h, w = (h + 1) // 2, (w + 1) // 2
            out.append((h, w, blk.cout))
        return out

    def forward(self, x: torch.Tensor) -> List[torch.Tensor]:
        """x: the control image, NCHW [B, C, H, W] (fp32 or bf16, host or device; H and W multiples of
        downscale_factor). Returns the features, bf16 NHWC [B, h, w, c], one per block."""
        from .. import ops
        from .._lib import ACT_RELU
        if self.device is None:
            raise RuntimeError("load_state_dict() must be called before forward()")
        x = x.to(self.device)
        if x.dtype not in (torch.float32, bf16):
            x = x.float()
        h = ops.pixel_unshuffle(x.contiguous(), self.downscale_factor)
        if self.conv_in is not None:
            h = ops.conv3x3(h, self.conv_in.w, self.conv_in.b)
        feats = []
        for blk in self.blocks:
            if blk.down:
                h = ops.avgpool2x2_nhwc(h)
            if blk.in_conv is not None:
                h = ops.linear(h, blk.in_conv.w, blk.in_conv.b)
            for b1, b2 in blk.resnets:
                r = ops.activation(ops.conv3x3(h, b1.w, b1.b), ACT_RELU)
                if blk.light:
                    h = ops.conv3x3(r, b2.w, b2.b, residual=h)
                else:
                    h = ops.linear(r, b2.w, b2.b, residual=h)
            if blk.out_conv is not None:
                h = ops.linear(h, blk.out_conv.w, blk.out_conv.b)
            feats.append(h)
        return feats

    __call__ = forward


class MultiAdapter:
    """ppdiffusers.MultiAdapter (models/adapter.py:27-100): several adapters whose features are summed with one weight
    each (default 1 / n). The weighted sum is one b200mix_weighted_sum_rows pass per feature, rounded once."""

    def __init__(self, adapters: Sequence[T2IAdapter], adapter_weights: Optional[List[float]] = None):
        self.adapters = list(adapters)
        self.num_adapter = len(self.adapters)
        if not self.adapters:
            raise ValueError("Expecting at least one adapter")
        if len(self.adapters) == 1:
            raise ValueError("For a single adapter, please use the `T2IAdapter` class instead of `MultiAdapter`")
        a0 = self.adapters[0]
        for idx, a in enumerate(self.adapters[1:], 1):
            if (a.total_downscale_factor != a0.total_downscale_factor or a.downscale_factor != a0.downscale_factor):
                raise ValueError(
                    f"Expecting all adapters to have the same downscaling behavior, but got:\n"
                    f"adapters[0].total_downscale_factor={a0.total_downscale_factor}\n"
                    f"adapters[0].downscale_factor={a0.downscale_factor}\n"
                    f"adapter[`{idx}`].total_downscale_factor={a.total_downscale_factor}\n"
                    f"adapter[`{idx}`].downscale_factor={a.downscale_factor}")
        self.total_downscale_factor = a0.total_downscale_factor
        self.downscale_factor = a0.downscale_factor
        self.adapter_weights = [1.0 / self.num_adapter] * self.num_adapter
        self.adapter_weights = self.weights(adapter_weights)

    def weights(self, adapter_weights: Optional[List[float]] = None) -> List[float]:
        """adapter_weights as a list of floats, one per adapter (None: this MultiAdapter's default). The reference zips
        them with the adapters, which only works for a sequence, so anything else is refused."""
        if adapter_weights is None:
            return list(self.adapter_weights)
        if not isinstance(adapter_weights, (list, tuple)) or len(adapter_weights) != self.num_adapter or \
                not all(isinstance(w, (int, float)) and not isinstance(w, bool) for w in adapter_weights):
            raise ValueError(f"adapter_weights must be a list of {self.num_adapter} floats, one per adapter, got "
                             f"{adapter_weights!r}")
        return [float(w) for w in adapter_weights]

    @property
    def device(self):
        return self.adapters[0].device

    def forward(self, xs: Sequence[torch.Tensor], adapter_weights: Optional[List[float]] = None) -> List[torch.Tensor]:
        """xs: one control image per adapter (NCHW, batch 1 or the common batch). Returns sum_k w_k * features_k, bf16
        NHWC."""
        from .. import ops
        w = self.weights(adapter_weights)
        xs = list(xs)
        if len(xs) != self.num_adapter:
            raise ValueError(f"MultiAdapter requires passing the same number of images as adapters. Given {len(xs)} "
                             f"images and {self.num_adapter} adapters.")
        feats = [a.forward(x) for a, x in zip(self.adapters, xs)]
        rows = max(f[0].shape[0] for f in feats)
        out = []
        for level in zip(*feats):
            o = torch.empty((rows,) + tuple(level[0].shape[1:]), device=level[0].device, dtype=bf16)
            out.append(ops.weighted_sum_rows(level, w, out=o))
        return out

    __call__ = forward
