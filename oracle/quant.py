"""ORACLE (test infrastructure, not product code): CPU fp32 restatement of weight-only int8 quantization as PaddleNLP's
inference models apply it at load time (quant_type="weight_only_int8": paddle.nn.quant.weight_quantize on the four
projection weights of every decoder layer, qwen/modeling.py:194-235, llama/modeling.py:523-578). The rule is the one
PaddleMIX's weight_only_int8 kernel spells out (paddlemix/triton_ops/triton_ops.py:481,505-508): per output channel
scale = max|w| / 127, q = clip(round(w / scale), -127, 127), and the layer computes x @ (q * scale) + bias.

Weights here are torch-layout [N, K] (one row per output channel). The device quantizes the fused matrices
paddlemix_b200.decoder builds (q|k|v rows concatenated, gate / up rows interleaved); per-row scales make that the same
as quantizing each projection on its own, and dequantize_decoder_params goes through the fused form anyway.
"""
from typing import Dict

import torch

Params = Dict[str, torch.Tensor]


def weight_quantize(w: torch.Tensor):
    """w [N, K] -> (q int8 [N, K], scale fp32 [N]). scale = absmax / 127 and w / scale are fp32 divisions; the
    rounding is half away from zero (paddle.round), computed in fp64 on the fp32 quotient: torch.round rounds half to
    even, and floor(x + 0.5) in fp32 rounds 0.49999997 up. An all-zero row gets scale 0 and q 0 (not 0 / 0)."""
    w = w.detach().to(torch.float32).cpu()
    scale = w.abs().amax(1) / torch.tensor(127.0, dtype=torch.float32)
    safe = torch.where(scale == 0, torch.ones_like(scale), scale)
    x = (w / safe[:, None]).double()
    r = torch.sign(x) * torch.floor(x.abs() + 0.5)
    q = r.clamp(-127, 127).to(torch.int8)
    q[scale == 0] = 0
    return q, scale


def dequantize(q: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """q * scale in fp32, [N, K]."""
    return q.to(torch.float32) * scale[:, None]


def dequantize_decoder_params(cfg, P: Params, prefix: str = "model") -> Params:
    """P with the q / k / v / o / gate / up / down weights of every decoder layer replaced by their weight-only int8
    values (q * scale, fp32, Paddle [in, out] layout), quantized as the device does it: q|k|v concatenated, gate / up
    interleaved (value = up at even rows, gate at odd rows), o and down as they are; then split back to the names of P."""
    out = dict(P)
    H, I = cfg["hidden_size"], cfg["intermediate_size"]
    kv = cfg["num_key_value_heads"] * (H // cfg["num_attention_heads"])

    def wq(w):
        return dequantize(*weight_quantize(w))

    for i in range(cfg["num_hidden_layers"]):
        b = f"{prefix}.layers.{i}"
        names = [f"{b}.self_attn.{n}_proj.weight" for n in "qkv"]
        qkv = wq(torch.cat([P[n].float().t() for n in names], 0))  # [H + 2 kv, H]
        for n, part in zip(names, torch.split(qkv, [H, kv, kv], 0)):
            out[n] = part.t().contiguous()
        for n in (f"{b}.self_attn.o_proj.weight", f"{b}.mlp.down_proj.weight"):
            out[n] = wq(P[n].float().t()).t().contiguous()
        up, gate = P[f"{b}.mlp.up_proj.weight"].float().t(), P[f"{b}.mlp.gate_proj.weight"].float().t()  # [I, H]
        gu = wq(torch.stack([up, gate], 1).reshape(2 * I, -1))
        out[f"{b}.mlp.up_proj.weight"] = gu[0::2].t().contiguous()
        out[f"{b}.mlp.gate_proj.weight"] = gu[1::2].t().contiguous()
    return out
