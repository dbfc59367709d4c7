"""Weight-only int8 without a GPU: the oracle's quantization rule on hand-made rows, the fused / split round trip of
dequantize_decoder_params, and the quant_type key of the configs."""
import pytest
import torch

from oracle import qwen2vl as O
from oracle import llama as OL
from oracle.quant import dequantize, dequantize_decoder_params, weight_quantize


def test_weight_quantize_rounds_half_away_from_zero():
    # absmax 127 -> scale 1 exactly: the quotients are the values themselves
    row = torch.tensor([127.0, 0.5, -0.5, 1.5, -1.5, 2.5, -2.5, 0.49999997, -0.49999997, 126.5, -3.0, 0.0])
    q, s = weight_quantize(row[None])
    assert s.tolist() == [1.0]
    assert q[0].tolist() == [127, 1, -1, 2, -2, 3, -3, 0, 0, 127, -3, 0]
    assert q.dtype == torch.int8


def test_weight_quantize_zero_row_and_negative_absmax():
    w = torch.tensor([[0.0, 0.0, 0.0, 0.0], [0.1, -0.7, 0.35, 0.0], [-0.0, 0.0, -0.0, 0.0]])
    q, s = weight_quantize(w)
    assert s[0] == 0 and s[2] == 0 and not torch.isnan(s).any()
    assert q[0].abs().sum() == 0 and q[2].abs().sum() == 0
    # the largest magnitude is negative: it maps to -127, scale = 0.7 / 127 in fp32
    assert q[1, 1] == -127
    assert s[1] == torch.tensor(0.7, dtype=torch.float32) / torch.tensor(127.0, dtype=torch.float32)
    x = torch.tensor([0.1, 0.35], dtype=torch.float32) / s[1]
    assert q[1, 0] == int(torch.floor(x[0].double() + 0.5)) and q[1, 2] == int(torch.floor(x[1].double() + 0.5))


def test_weight_quantize_bounds_and_error():
    g = torch.Generator().manual_seed(0)
    w = torch.randn(64, 256, generator=g)
    q, s = weight_quantize(w)
    assert int(q.abs().max()) == 127 and int(q.min()) >= -127
    err = (dequantize(q, s) - w).abs()
    assert bool((err <= s[:, None] / 2 * (1 + 1e-6)).all())


@pytest.mark.parametrize("which", ["qwen2vl", "llama"])
def test_dequantize_decoder_params_keeps_names_and_shapes(which):
    if which == "qwen2vl":
        cfg = O.QWEN2VL_CONFIGS["tiny"]
        P, prefix, shapes = O.init_qwen2vl_params(cfg, seed=3), "model", O.qwen2vl_param_shapes(cfg)
    else:
        cfg = OL.LLAMA_CONFIGS["tiny"]
        shapes = OL.llama_param_shapes(cfg)
        g = torch.Generator().manual_seed(3)
        P, prefix = {k: torch.randn(*v, generator=g) * 0.05 for k, v in shapes.items()}, "llama"
    D = dequantize_decoder_params(cfg, P, prefix=prefix)
    assert set(D) == set(shapes) and all(tuple(D[k].shape) == tuple(shapes[k]) for k in shapes)
    proj = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")
    for k in shapes:
        if any(f".{p}.weight" in k for p in proj) and ".layers." in k:
            assert not torch.equal(D[k], P[k]), k
            # every output column of the Paddle [in, out] layout holds at most 255 distinct levels of one scale
            col = D[k][:, 0]
            scale = col.abs().max() / 127
            assert torch.allclose(col / scale, (col / scale).round(), atol=1e-3), k
        else:
            assert D[k] is P[k], k


def test_qwen2vl_config_keeps_quant_type():
    from paddlemix_b200.qwen2_vl.modeling_qwen2_vl import Qwen2VLConfig
    assert Qwen2VLConfig().quant_type is None
    assert Qwen2VLConfig(quant_type="weight_only_int8").quant_type == "weight_only_int8"


@pytest.mark.parametrize("bad", ["weight_only_int4", "int8", "a8w8"])
def test_unknown_quant_type_is_refused_before_device_work(bad, monkeypatch):
    from paddlemix_b200 import ops
    from paddlemix_b200.llava.modeling_llava import LlamaForCausalLM
    from paddlemix_b200.qwen2_vl import Qwen2VLForConditionalGeneration

    def no_device(*a, **k):
        raise AssertionError("device work before the quant_type check")
    monkeypatch.setattr(ops, "init", no_device)
    monkeypatch.setattr(ops, "quantize_w8", no_device)
    with pytest.raises(ValueError, match="quant_type"):
        Qwen2VLForConditionalGeneration(dict(O.QWEN2VL_CONFIGS["tiny"], quant_type=bad))
    with pytest.raises(ValueError, match="quant_type"):
        LlamaForCausalLM(dict(OL.LLAMA_CONFIGS["tiny"], quant_type=bad))
