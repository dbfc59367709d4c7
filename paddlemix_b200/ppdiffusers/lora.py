"""LoRA for UNet2DConditionModel: the reference's key formats, named adapters, and their realisation in the device
weights with one b200mix_lora_apply launch.

Reference: LoraLoaderMixin.lora_state_dict (ppdiffusers/loaders/lora.py:169-352), the kohya / A1111 conversion
(loaders/lora_conversion_utils.py:22-283), UNet2DConditionLoadersMixin.load_attn_procs / fuse_lora / unfuse_lora
(loaders/unet.py:85-445, :594-622) and the per-layer merges of models/lora.py:117-165, :312-362.

A LoRA names reference layers; load_state_dict turned each of them into one or more device tensors (head-padded q/k/v
rows, the batched self-attention w_qkv, the batched cross-attention K/V and time_emb_proj weights, interleaved GEGLU
rows, LayerNorm-folded copies, [O, 3, 3, I] convs and the per-parity upsample taps). `targets()` records, for every
LoRA-compatible layer, where it landed: the tensor, the first row, and how the up factor's rows and the down factor's
columns map to device order. The realised weights are
    base + sum_fused s_f * dW_f + lam * sum_active w_a * dW_a,      dW = (alpha / rank) * up @ down,
where base is a device snapshot of each touched tensor taken before its first change, so every state is computed from
the snapshot with one rounding and never depends on earlier states. Writes go in place, so captured CUDA graphs replay
with the new weights.
"""
import re
import warnings
from collections import OrderedDict
from typing import Any, Dict, List, Optional, Tuple

import torch

from ..modeling import pad_head_cols, pad_head_rows, to_f32

TEXT_ENCODER_PREFIXES = ("text_encoder.", "text_encoder_2.", "lora_te_", "lora_te1_", "lora_te2_")
UNSUPPORTED_MARKERS = ("hada_", "lokr_", "dora_scale")  # LoHa, LoKr, DoRA
REFUSED_LAYERS = ("conv_in", "conv_out")  # plain nn.Conv2D in the reference (loaders/unet.py:357-358)


# ---- key formats -------------------------------------------------------------------------------------------------
def _sgm_to_diffusers(keys: List[str], layers_per_block: int) -> Dict[str, str]:
    """kohya names with SGM (SDXL original) block names -> kohya names with diffusers block names
    (lora_conversion_utils.py:22-120). keys: full kohya keys; returns {old: new} for every key (unchanged when no
    key uses SGM names)."""
    sgm = ("input_blocks", "middle_block", "output_blocks")
    if not any(p in k for k in keys for p in sgm):
        return {k: k for k in keys}
    inner = ("resnets", "attentions", "upsamplers")
    out = {}
    for k in keys:
        if "text" in k:
            out[k] = k
            continue
        parts = k.split("_")
        # lora_unet_<input|middle|output>_<blocks|block>_<block id>_<inner id>_...
        if not any(p in k for p in sgm):
            raise ValueError(f"Checkpoint not supported because layer {k} not supported.")
        bid = int(parts[4])
        if "input_blocks" in k:
            blk, layer = (bid - 1) // (layers_per_block + 1), (bid - 1) % (layers_per_block + 1)
            inner_id = int(parts[5])
            kind, idx = (inner[inner_id], str(layer)) if "op" not in k else ("downsamplers", "0")
            new = parts[:4] + [str(blk), kind, idx] + parts[6:]
        elif "middle_block" in k:
            if bid not in (0, 1, 2):
                raise ValueError(f"Invalid middle block id {bid}.")
            kind, idx = (("resnets", "0"), ("attentions", "0"), ("resnets", "1"))[bid]
            new = parts[:4] + [kind, idx] + parts[5:]
        else:
            blk, layer = bid // (layers_per_block + 1), bid % (layers_per_block + 1)
            inner_id = int(parts[5])
            new = parts[:4] + [str(blk), inner[inner_id], str(layer) if inner_id < 2 else "0"] + parts[6:]
        out[k] = "_".join(new)
    return out


def _kohya_unet_layer(lora_name: str) -> str:
    """'lora_unet_down_blocks_0_attentions_0_..._attn1_to_q' -> 'down_blocks.0.attentions.0....attn1.to_q'
    (the lora_unet_ branch of lora_conversion_utils.py:140-200)."""
    n = lora_name[len("lora_unet_"):].replace("_", ".")
    for a, b in (("input.blocks", "down_blocks"), ("down.blocks", "down_blocks"), ("middle.block", "mid_block"),
                 ("mid.block", "mid_block"), ("output.blocks", "up_blocks"), ("up.blocks", "up_blocks"),
                 ("transformer.blocks", "transformer_blocks"), ("to.q", "to_q"), ("to.k", "to_k"), ("to.v", "to_v"),
                 ("to.out.0", "to_out.0"), ("proj.in", "proj_in"), ("proj.out", "proj_out"),
                 ("emb.layers", "time_emb_proj")):
        n = n.replace(a, b)
    if "emb" in n and "time.emb.proj" not in n:  # SGM emb_layers_1 -> time_emb_proj
        n = re.sub(r"\.\d+(?=\D*$)", "", n, count=1)
    if ".in." in n:
        n = n.replace("in.layers.2", "conv1")
    if ".out." in n:
        n = n.replace("out.layers.3", "conv2")
    if "downsamplers" in n or "upsamplers" in n:
        n = n.replace("op", "conv")
    for a, b in (("skip.connection", "conv_shortcut"), ("time.emb.proj", "time_emb_proj"),
                 ("conv.shortcut", "conv_shortcut")):
        n = n.replace(a, b)
    return n


def _is_kohya(sd) -> bool:
    return len(sd) > 0 and all(k.startswith(("lora_unet_", "lora_te_", "lora_te1_", "lora_te2_")) for k in sd)


def _check_supported(sd):
    for k in sd:
        if any(m in k for m in UNSUPPORTED_MARKERS):
            raise ValueError(f"{k}: LoHa / LoKr / DoRA weights are not supported (only plain LoRA up / down factors)")


def lora_state_dict(pretrained_model_name_or_path_or_dict, unet_config=None, from_diffusers: Optional[bool] = None):
    """LoraLoaderMixin.lora_state_dict (lora.py:169-352): reads a file (safetensors / .pdparams through
    weights.read_checkpoint) or takes a dict; kohya keys are converted to diffusers names with their alphas
    (SGM block names are remapped with `unet_config`'s layers_per_block). Returns (state_dict, network_alphas,
    from_diffusers). Text-encoder entries stay in the state dict under text_encoder.* / text_encoder_2.*.
    from_diffusers=None: a file's safetensors format metadata decides ("pt" = torch layout); a kohya dict is in torch
    layout (it is a torch trainer's format); any other dict in Paddle layout."""
    if isinstance(pretrained_model_name_or_path_or_dict, dict):
        sd = dict(pretrained_model_name_or_path_or_dict)
        detected = None
    else:
        from ..weights import read_checkpoint
        sd, layout = read_checkpoint(pretrained_model_name_or_path_or_dict)
        detected = layout == "torch"
    _check_supported(sd)
    network_alphas = None
    if _is_kohya(sd):
        if detected is None:
            detected = True
        if unet_config is not None:
            ren = _sgm_to_diffusers(list(sd), unet_config["layers_per_block"])
            sd = {ren[k]: v for k, v in sd.items()}
        sd, network_alphas = _convert_kohya(sd)
    if from_diffusers is None:
        from_diffusers = bool(detected)
    return sd, network_alphas, from_diffusers


def _convert_kohya(sd):
    """kohya keys -> {'unet.<layer>.lora.down.weight', ...} and {'unet.<layer>.alpha': alpha}; text-encoder keys keep
    their names under text_encoder.* / text_encoder_2.* (they are split off, not applied)."""
    out, alphas = {}, {}
    names = sorted({k.split(".")[0] for k in sd})
    for lname in names:
        down, up = sd.get(lname + ".lora_down.weight"), sd.get(lname + ".lora_up.weight")
        extra = [k for k in sd if k.split(".")[0] == lname and
                 k not in (lname + ".lora_down.weight", lname + ".lora_up.weight", lname + ".alpha")]
        if extra or down is None or up is None:
            raise ValueError(f"kohya LoRA {lname}: expected lora_down.weight, lora_up.weight and optionally alpha, "
                             f"got {sorted(k for k in sd if k.split('.')[0] == lname)}")
        if lname.startswith("lora_unet_"):
            prefix, layer = "unet.", _kohya_unet_layer(lname)
        else:
            prefix = "text_encoder_2." if lname.startswith("lora_te2_") else "text_encoder."
            layer = lname.split("_", 2)[2]
        out[f"{prefix}{layer}.lora.down.weight"] = down
        out[f"{prefix}{layer}.lora.up.weight"] = up
        if lname + ".alpha" in sd:
            alphas[f"{prefix}{layer}.alpha"] = float(to_f32(sd[lname + ".alpha"]).reshape(-1)[0])
    return out, alphas


def _legacy_to_layer(key: str) -> str:
    """'...attn1.processor.to_out_lora.down.weight' -> '...attn1.to_out.0.lora.down.weight' (loaders/unet.py:435-445)."""
    if "processor" not in key.split("."):
        return key
    return key.replace(".processor", "").replace("to_out_lora", "to_out.0.lora").replace("_lora", ".lora")


def split_text_encoder(sd) -> Tuple[Dict[str, Any], Dict[str, Any]]:
    """(UNet entries with any 'unet.' prefix removed, text-encoder entries)."""
    unet, te = {}, {}
    for k, v in sd.items():
        if k.startswith(TEXT_ENCODER_PREFIXES):
            te[k] = v
        else:
            unet[k[len("unet."):] if k.startswith("unet.") else k] = v
    return unet, te


def lora_layer_shapes(state_dict_shapes: Dict[str, tuple]) -> Dict[str, tuple]:
    """Every LoRA-compatible layer of the model and its torch-layout weight shape [out, in] or [out, in, kh, kw]: every
    Linear and conv weight except conv_in / conv_out."""
    out = {}
    for k, s in state_dict_shapes.items():
        if not k.endswith(".weight") or len(s) not in (2, 4):
            continue
        layer = k[: -len(".weight")]
        if layer in REFUSED_LAYERS:
            continue
        out[layer] = (s[1], s[0]) if len(s) == 2 else tuple(s)  # Paddle Linear [in, out] -> [out, in]
    return out


def parse_lora(state_dict, network_alphas, from_diffusers: bool, layer_shapes: Dict[str, tuple]):
    """UNet LoRA entries (diffusers / ppdiffusers or legacy processor names, no 'unet.' prefix) -> {layer: (up, down,
    scale)} in torch layout: up fp32 [out, r], down fp32 [r, in] or [r, in, kh, kw], scale = alpha / r (1 without an
    alpha). Paddle layout (from_diffusers False) holds a Linear's down as [in, r] and up as [r, out]; convs are the
    same in both. Raises ValueError for unknown or refused layers, shapes that fit no layer, and unmatched alphas."""
    _check_supported(state_dict)
    groups: Dict[str, Dict[str, Any]] = OrderedDict()
    for k, v in state_dict.items():
        k2 = _legacy_to_layer(k)
        if k2.endswith(".alpha"):
            continue
        m = re.fullmatch(r"(.+)\.lora\.(down|up)\.weight", k2)
        if m is None:
            raise ValueError(f"{k}: not a LoRA up / down weight")
        groups.setdefault(m.group(1), {})[m.group(2)] = v
    alphas = {}
    for k, v in list((network_alphas or {}).items()) + [(k, v) for k, v in state_dict.items() if k.endswith(".alpha")]:
        if k.startswith(TEXT_ENCODER_PREFIXES):
            continue
        k = k[len("unet."):] if k.startswith("unet.") else k
        layer = _legacy_to_layer(k[: -len(".alpha")] + ".lora.down.weight")[: -len(".lora.down.weight")]
        if layer not in groups:
            raise ValueError(f"network alpha {k} matches no LoRA layer of the state dict")
        alphas[layer] = float(to_f32(v).reshape(-1)[0]) if torch.is_tensor(v) else float(v)
    out = OrderedDict()
    for layer, f in groups.items():
        if layer in REFUSED_LAYERS:
            raise ValueError(f"Module {layer} is not a LoRACompatibleConv or LoRACompatibleLinear module.")
        if layer not in layer_shapes:
            raise ValueError(f"{layer}: no LoRA-compatible layer of this UNet has that name")
        if set(f) != {"down", "up"}:
            raise ValueError(f"{layer}: needs both lora.down.weight and lora.up.weight")
        shape = layer_shapes[layer]
        down, up = to_f32(f["down"]).cpu(), to_f32(f["up"]).cpu()
        if len(shape) == 2:
            n_out, n_in = shape
            if not from_diffusers:
                down, up = down.t(), up.t()
            ok = down.dim() == 2 and up.dim() == 2 and down.shape[1] == n_in and up.shape[0] == n_out and \
                up.shape[1] == down.shape[0]
        else:
            n_out, n_in = shape[:2]
            ok = (down.dim() == 4 and up.dim() == 4 and down.shape[1] == n_in and tuple(down.shape[2:]) == shape[2:]
                  and tuple(up.shape[2:]) == (1, 1) and up.shape[0] == n_out and up.shape[1] == down.shape[0])
            up = up.reshape(up.shape[0], up.shape[1]) if ok else up
        if not ok:
            want = ((f"down [{n_in}, r] / up [r, {n_out}] (Paddle layout)" if not from_diffusers else
                     f"down [r, {n_in}] / up [{n_out}, r] (torch layout)") if len(shape) == 2 else
                    f"down [r, {n_in}, {shape[2]}, {shape[3]}] / up [{n_out}, r, 1, 1]")
            raise ValueError(f"{layer}: LoRA factors down {tuple(f['down'].shape)} / up {tuple(f['up'].shape)} do not "
                             f"fit the layer's weight {shape}: expected {want}")
        r = down.shape[0]
        out[layer] = (up.contiguous(), down.contiguous(), alphas[layer] / r if layer in alphas else 1.0)
    return out


# ---- where each layer lives on the device ---------------------------------------------------------------------------
def interleave_rows(w: torch.Tensor) -> torch.Tensor:
    """GEGLU (value, gate) halves -> interleaved rows, so both land in the same accumulator tile (the load path's
    transform of ff.net.0.proj, for weights, biases and LoRA up factors alike)."""
    half = w.shape[0] // 2
    return torch.stack([w[:half], w[half:]], 1).reshape(2 * half, *w.shape[1:]).contiguous()


def _cols_linear(d):
    return d.reshape(d.shape[0], -1)


def _cols_conv3x3(d):  # [r, I, 3, 3] -> [r, 3 * 3 * I] in the device's [ky, kx, i] order
    return d.permute(0, 2, 3, 1).reshape(d.shape[0], -1)


def _cols_up4(d):  # [r, I, 3, 3] -> [r, 16 * I]: the per-parity tap sums of fold_upsample_conv_weight
    from ..ops import fold_upsample_taps
    return fold_upsample_taps(d.permute(0, 2, 3, 1)).reshape(d.shape[0], -1)


def _ident(u):
    return u


class Place:
    """One device tensor a layer feeds: rows [r0, r0 + n) of tensor(), the up factor's rows in device order
    (rows(U)), the down factor's columns in device order (cols(D)), and for a LayerNorm-folded copy ln() =
    (gamma [K], beta [K], colsum [rows of the tensor], bias [rows of the tensor])."""
    __slots__ = ("tensor", "r0", "rows", "cols", "ln")

    def __init__(self, tensor, r0=lambda: 0, rows=_ident, cols=_cols_linear, ln=None):
        self.tensor, self.r0, self.rows, self.cols, self.ln = tensor, r0, rows, cols, ln


def targets(unet) -> Dict[str, List[Place]]:
    """Layer name -> the device tensors load_state_dict built from it (unet_2d_condition.py's load paths)."""
    T: Dict[str, List[Place]] = OrderedDict()

    def w2d(get):  # a weight as the [N, K] matrix the kernel writes ([O, 3, 3, I] / [O, 16, I] flattened)
        return lambda: (lambda w: w.view(w.shape[0], -1))(get())

    for m, name in ((unet.time_lin1, "time_embedding.linear_1"), (unet.time_lin2, "time_embedding.linear_2"),
                    (unet.add_lin1, "add_embedding.linear_1"), (unet.add_lin2, "add_embedding.linear_2")):
        if m is not None:
            T[name] = [Place(lambda m=m: m.w)]
    for r in unet.resnets:
        T[r.name + ".conv1"] = [Place(w2d(lambda r=r: r.conv1.w), cols=_cols_conv3x3)]
        T[r.name + ".conv2"] = [Place(w2d(lambda r=r: r.conv2.w), cols=_cols_conv3x3)]
        if r.shortcut is not None:
            T[r.name + ".conv_shortcut"] = [Place(lambda r=r: r.shortcut.w)]
        T[r.name + ".time_emb_proj"] = [Place(lambda: unet.temb_w_all, r0=lambda r=r: r.temb_slice[0])]
    for blk in unet.down:
        if blk.down is not None:
            T[blk.down.name] = [Place(w2d(lambda c=blk.down: c.w), cols=_cols_conv3x3)]
    for blk in unet.up:
        if blk.up is not None:
            T[blk.up.name] = [Place(w2d(lambda c=blk.up: c.w), cols=_cols_conv3x3),
                              Place(w2d(lambda c=blk.up: c.w4), cols=_cols_up4)]
    for t in unet.transformers:
        T[t.proj_in.name] = [Place(lambda t=t: t.proj_in.w)]
        T[t.proj_out.name] = [Place(lambda t=t: t.proj_out.w)]
        for b in t.blocks:
            for a, norm in ((b.attn1, b.norm1), (b.attn2, b.norm2)):
                H, d, dp, inner = a.heads, a.head_dim, a.head_pad, a.inner
                pad = (lambda u, H=H, d=d, dp=dp: pad_head_rows(u, H, d, dp))

                def ln(a=a, norm=norm):
                    return norm.w, norm.b, a.ln_fold[1], a.ln_fold[2]
                fold = (lambda a=a: a.ln_fold[0])
                if a.is_cross:
                    T[a.name + ".to_q"] = [Place(lambda a=a: a.w_q, rows=pad), Place(fold, rows=pad, ln=ln)]
                    kv = (lambda a=a: unet._kv_groups[a.ctx_dim]["w"])
                    T[a.name + ".to_k"] = [Place(kv, r0=lambda a=a: a._kv_off, rows=pad)]
                    T[a.name + ".to_v"] = [Place(kv, r0=lambda a=a: a._kv_off + a.inner, rows=pad)]
                else:
                    for i, p in enumerate(("to_q", "to_k", "to_v")):
                        T[f"{a.name}.{p}"] = [Place(lambda a=a: a.w_qkv, r0=lambda i=i, n=inner: i * n, rows=pad),
                                              Place(fold, r0=lambda i=i, n=inner: i * n, rows=pad, ln=ln)]
                T[a.name + ".to_out.0"] = [Place(lambda a=a: a.w_o,
                                                 cols=lambda dd, H=H, d=d, dp=dp: pad_head_cols(dd, H, d, dp))]

            def ln3(b=b):
                return b.norm3.w, b.norm3.b, b.ff1_fold[1], b.ff1_fold[2]
            T[b.name + ".ff.net.0.proj"] = [Place(lambda b=b: b.ff1_w, rows=interleave_rows),
                                            Place(lambda b=b: b.ff1_fold[0], rows=interleave_rows, ln=ln3)]
            T[b.name + ".ff.net.2"] = [Place(lambda b=b: b.ff2.w)]
    return T


# ---- adapter state ---------------------------------------------------------------------------------------------------
def _pad8(n: int) -> int:
    return (n + 7) // 8 * 8


class _Adapter:
    __slots__ = ("factors", "weight", "fused_scale")

    def __init__(self, factors):
        self.factors = factors  # {layer: [(U_dev [n, r8], D_dev [r8, K]) per Place]}, alpha / r folded into U
        self.weight = 1.0
        self.fused_scale = None  # lora_scale * weight while fused


class LoraState:
    """Named adapters of one UNet and their realisation in its device weights."""

    def __init__(self, unet):
        self.unet = unet
        self.adapters: "OrderedDict[str, _Adapter]" = OrderedDict()
        self.active: List[str] = []
        self.scale = 1.0           # lam, the call scale the weights are realised at
        self.snap: Dict[tuple, dict] = {}  # (id(tensor), r0) -> snapshot of the target
        self._targets = None

    def targets(self):
        if self._targets is None:
            self._targets = targets(self.unet)
        return self._targets

    # -- loading -------------------------------------------------------------------------------------------------
    def add(self, name: str, parsed) -> None:
        """parsed: parse_lora's {layer: (up, down, scale)}. Builds the device factors, makes `name` the only active
        unfused adapter and realises."""
        if name in self.adapters:
            raise ValueError(f"Adapter name {name} already in use in the Unet - please select a new adapter name.")
        T = self.targets()
        dev = self.unet.device
        factors = {}
        for layer, (up, down, s) in parsed.items():
            r = up.shape[1]
            r8 = _pad8(r)
            u = torch.zeros(up.shape[0], r8, dtype=torch.float32)
            u[:, :r] = up * s
            dn = torch.zeros((r8,) + tuple(down.shape[1:]), dtype=torch.float32)
            dn[:r] = down
            u, dn = u.to(dev), dn.to(dev)
            factors[layer] = [(p.rows(u).contiguous(), p.cols(dn).contiguous()) for p in T[layer]]
        self.adapters[name] = _Adapter(factors)
        self.active = [name]
        self.realise()

    # -- state changes -------------------------------------------------------------------------------------------
    def set_adapters(self, names, weights=None):
        names = [names] if isinstance(names, str) else list(names)
        if weights is None:
            weights = [1.0] * len(names)
        elif isinstance(weights, (int, float)):
            weights = [float(weights)] * len(names)
        weights = list(weights)
        if len(weights) != len(names):
            raise ValueError(f"Length of adapter names {len(names)} is not equal to the length of their weights "
                             f"{len(weights)}.")
        for n in names:
            if n not in self.adapters:
                raise ValueError(f"Adapter {n} is not loaded; loaded adapters: {list(self.adapters)}")
            if self.adapters[n].fused_scale is not None:
                raise ValueError(f"Adapter {n} is fused: unfuse_lora() before changing its weight")
        for n, w in zip(names, weights):
            self.adapters[n].weight = float(w)
        self.active = names
        self.realise()

    def fuse(self, lora_scale=1.0):
        """Moves the active adapters into the fused set at lora_scale * weight; they stop responding to lam."""
        for n in self.active:
            a = self.adapters[n]
            a.fused_scale = float(lora_scale) * a.weight
        self.active = []
        self.realise()

    def unfuse(self):
        """Returns every fused adapter to the active unfused set."""
        for n, a in self.adapters.items():
            if a.fused_scale is not None:
                a.fused_scale = None
                if n not in self.active:
                    self.active.append(n)
        self.realise()

    def unload(self):
        """Drops the unfused adapters (fused ones stay in the weights, as in the reference)."""
        for n in [n for n, a in self.adapters.items() if a.fused_scale is None]:
            del self.adapters[n]
        self.active = []
        self.realise()

    def set_scale(self, lam: float):
        lam = float(lam)
        if lam == self.scale:
            return
        self.scale = lam
        if any(self.adapters[n].fused_scale is None for n in self.active):
            self.realise()

    # -- realisation ---------------------------------------------------------------------------------------------
    def coefficients(self) -> Dict[str, float]:
        c = {n: a.fused_scale for n, a in self.adapters.items() if a.fused_scale is not None}
        for n in self.active:
            c[n] = self.scale * self.adapters[n].weight
        return {n: v for n, v in c.items() if v != 0.0}

    def realise(self):
        """One b200mix_lora_apply launch over every target any adapter has touched since the snapshots were taken;
        with no adapter left, the snapshots are written back bit for bit and freed."""
        from .. import ops
        T = self.targets()
        coef = self.coefficients()
        dev = self.unet.device
        for layer, places in T.items():  # snapshot on first touch
            fac = next((a.factors[layer] for a in self.adapters.values() if layer in a.factors), None)
            for p, (u, _) in zip(places, fac or ()):
                self._snapshot(p, u.shape[0])
        items, bias_updates = [], []
        for layer, places in T.items():
            for i, p in enumerate(places):
                s = self.snap.get(self._key(p))
                if s is None:
                    continue
                parts = [(c, self.adapters[n].factors[layer][i]) for n, c in coef.items()
                         if layer in self.adapters[n].factors]
                if parts:
                    U = torch.cat([c * u for c, (u, _) in parts], 1).contiguous()
                    D = torch.cat([d for _, (_, d) in parts], 0).contiguous()
                else:
                    U = torch.zeros(s["base"].shape[0], 8, device=dev)
                    D = torch.zeros(8, s["base"].shape[1], device=dev)
                it = dict(out=s["out"], base=s["base"], U=U, D=D)
                if p.ln is not None:
                    gamma, beta, _, _ = p.ln()
                    it.update(col_scale=gamma, colsum=s["colsum"], colsum_base=s["colsum_base"])
                    bias_updates.append((s, U, D, beta))
                items.append(it)
        if items:
            ops.lora_apply(items)
        for s, U, D, beta in bias_updates:  # folded bias b' = b + W beta: dW beta = U (D beta), a [N, R] product
            delta = U @ (D @ beta.float())
            s["bias"].copy_(torch.where(delta == 0, s["bias_base"], s["bias_base"] + delta))
        if not self.adapters:
            self.snap.clear()

    @staticmethod
    def _key(p):
        return (p.tensor().data_ptr(), p.r0())

    def _snapshot(self, p, n):
        """Device copies of rows [r0, r0 + n) of the target (and of its folded colsum / bias)."""
        k = self._key(p)
        if k in self.snap:
            return
        r0 = p.r0()
        out = p.tensor()[r0: r0 + n]
        s = dict(out=out, base=out.clone())
        if p.ln is not None:
            _, _, colsum, bias = p.ln()
            s.update(colsum=colsum[r0: r0 + n], bias=bias[r0: r0 + n])
            s.update(colsum_base=s["colsum"].clone(), bias_base=s["bias"].clone())
        self.snap[k] = s

    def snapshot_bytes(self) -> int:
        return sum(t.numel() * t.element_size() for s in self.snap.values()
                   for k, t in s.items() if k.endswith("_base") or k == "base")


def warn_text_encoder(n: int):
    if n:
        warnings.warn(f"{n} text-encoder LoRA entries are not applied: the pipelines here take prompt_embeds, so the "
                      "text encoders are outside this package", stacklevel=3)
