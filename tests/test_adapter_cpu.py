"""T2I-Adapter host logic without a GPU: parameter names and shapes against the reference constructors' layout
(oracle.adapter), downscale factors, LightAdapter's padded device shapes, the refusals that come before any device work,
the adapter_conditioning_factor cut-off and the GEMM wrappers' refusal of ACT_RELU."""
import pytest
import torch

from oracle import adapter as OA
from paddlemix_b200 import _lib, ops
from paddlemix_b200._lib import ACT_RELU
from paddlemix_b200.ppdiffusers.adapter import MultiAdapter, T2IAdapter

bf16 = torch.bfloat16


def make(name, **kw):
    return T2IAdapter(**{**OA.ADAPTER_CONFIGS[name], **kw})


@pytest.mark.parametrize("name", list(OA.ADAPTER_CONFIGS))
def test_state_dict_shapes_match_the_reference_layout(name):
    cfg = OA.ADAPTER_CONFIGS[name]
    assert make(name).state_dict_shapes() == OA.adapter_param_shapes(cfg)


def test_reference_parameter_names():
    full = make("sd15").state_dict_shapes()
    assert full["adapter.conv_in.weight"] == (320, 192, 3, 3)
    assert full["adapter.body.1.in_conv.weight"] == (640, 320, 1, 1)
    assert full["adapter.body.3.resnets.1.block2.weight"] == (1280, 1280, 1, 1)
    assert "adapter.body.0.in_conv.weight" not in full and "adapter.body.3.in_conv.weight" not in full
    xl = make("sdxl").state_dict_shapes()
    assert xl["adapter.conv_in.weight"] == (320, 768, 3, 3)
    assert xl["adapter.body.1.in_conv.weight"] == (640, 320, 1, 1) and xl["adapter.body.2.in_conv.weight"] == (1280, 640, 1, 1)
    light = make("sd15_light").state_dict_shapes()
    assert "adapter.conv_in.weight" not in light
    assert light["adapter.body.0.in_conv.weight"] == (80, 192, 1, 1)
    assert light["adapter.body.3.resnets.3.block2.weight"] == (320, 320, 3, 3)
    assert light["adapter.body.3.out_conv.weight"] == (1280, 320, 1, 1)


@pytest.mark.parametrize("name,total,f", [("sd15", 64, 8), ("sdxl", 32, 16), ("sd15_light", 64, 8), ("tiny_sd", 32, 8),
                                          ("tiny_xl", 32, 16), ("tiny_sd_light", 32, 8)])
def test_downscale_factors(name, total, f):
    a = make(name)
    assert a.total_downscale_factor == total == OA.total_downscale_factor(OA.ADAPTER_CONFIGS[name])
    assert a.downscale_factor == f


def test_feature_shapes():
    assert make("sdxl").feature_shapes(1024, 1024) == [(64, 64, 320), (64, 64, 640), (32, 32, 1280), (32, 32, 1280)]
    assert make("sd15").feature_shapes(512, 512) == [(64, 64, 320), (32, 32, 640), (16, 16, 1280), (8, 8, 1280)]
    assert make("sd15_light").feature_shapes(512, 512) == [(64, 64, 320), (32, 32, 640), (16, 16, 1280), (8, 8, 1280)]
    assert make("sd15").feature_shapes(8 * 9, 8 * 5) == [(9, 5, 320), (5, 3, 640), (3, 2, 1280), (2, 1, 1280)]


def test_light_adapter_pads_mid_channels_at_load(monkeypatch):
    """80 / 160 / 320 mid channels become 128 / 192 / 320 on the device, with zero filters and biases; the CPU stands
    in for the device here (bind only initialises the library)."""
    from oracle.unet import init_params
    monkeypatch.setattr(ops, "init", lambda dev=0: None)
    P = init_params(OA.adapter_param_shapes(OA.ADAPTER_CONFIGS["sd15_light"]), seed=3)
    a = make("sd15_light").load_state_dict(P, device="cpu")
    for b, mid, pad in ((0, 80, 128), (1, 160, 192), (2, 320, 320), (3, 320, 320)):
        blk = a.blocks[b]
        assert tuple(blk.in_conv.w.shape) == (pad, blk.in_conv.cin) and tuple(blk.in_conv.b.shape) == (pad,)
        for b1, b2 in blk.resnets:
            assert tuple(b1.w.shape) == (pad, 3, 3, pad) and tuple(b2.w.shape) == (pad, 3, 3, pad)
            assert not b1.w[mid:].any() and not b1.w[..., mid:].any() and not b1.b[mid:].any()
            assert not b2.w[mid:].any() and not b2.w[..., mid:].any() and not b2.b[mid:].any()
        assert tuple(blk.out_conv.w.shape) == (blk.cout, pad) and not blk.out_conv.w[:, mid:].any()
        assert not blk.in_conv.w[mid:].any() and not blk.in_conv.b[mid:].any()
        ref = P[f"adapter.body.{b}.resnets.0.block1.weight"].permute(0, 2, 3, 1)
        assert torch.equal(blk.resnets[0][0].w[:mid, :, :, :mid].float(), ref)


# ---- refusals ---------------------------------------------------------------------------------------------------------
def test_unknown_adapter_type():
    with pytest.raises(ValueError, match="Unsupported adapter_type: 'half_adapter'"):
        T2IAdapter(adapter_type="half_adapter")


@pytest.mark.parametrize("kw", [dict(channels=(320, 600, 1280, 1280)), dict(channels=(96, 128, 256)),
                                dict(downscale_factor=4), dict(adapter_type="light_adapter", channels=(320, 644, 1280)),
                                dict(adapter_type="full_adapter_xl", channels=(320, 640, 1280, 640))])
def test_unsupported_channels_are_refused_before_device_work(kw, monkeypatch):
    touched = []
    monkeypatch.setattr(ops, "init", lambda *a: touched.append(a))
    monkeypatch.setattr(_lib, "lib", None)
    with pytest.raises(NotImplementedError):
        T2IAdapter(**kw)
    assert not touched


def test_multi_adapter_refusals():
    a8, a16 = make("tiny_sd"), make("tiny_xl")
    with pytest.raises(ValueError, match="same downscaling behavior"):
        MultiAdapter([a8, a16])
    with pytest.raises(ValueError, match="at least one adapter"):
        MultiAdapter([])
    with pytest.raises(ValueError, match="single adapter"):
        MultiAdapter([a8])
    for bad in (0.5, (0.5,), [0.5, "1"], [0.5, 0.5, 0.5], torch.tensor([0.5, 0.5])):
        with pytest.raises(ValueError, match="list of 2 floats"):
            MultiAdapter([a8, make("tiny_sd")], bad)
    m = MultiAdapter([a8, make("tiny_sd")])
    assert m.weights() == [0.5, 0.5] and m.weights([0.25, 1]) == [0.25, 1.0]
    assert MultiAdapter([a8, make("tiny_sd")], [0.3, 0.7]).weights() == [0.3, 0.7]
    assert m.total_downscale_factor == 32 and m.downscale_factor == 8


def test_pipeline_refuses_image_count_before_device_work():
    from paddlemix_b200.ppdiffusers.pipelines import StableDiffusionAdapterPipeline
    pipe = StableDiffusionAdapterPipeline(unet=None, adapter=[make("tiny_sd"), make("tiny_sd")], scheduler=None)
    img = torch.zeros(1, 3, 64, 64)
    with pytest.raises(ValueError, match="same number of images as adapters"):
        pipe(prompt_embeds=torch.zeros(1, 4, 8), image=[img], num_inference_steps=2)
    with pytest.raises(ValueError, match="not a list"):
        pipe(prompt_embeds=torch.zeros(1, 4, 8), image=img, num_inference_steps=2)
    with pytest.raises(ValueError, match="list of 2 floats"):
        pipe(prompt_embeds=torch.zeros(1, 4, 8), image=[img, img], adapter_conditioning_scale=0.5)
    single = StableDiffusionAdapterPipeline(unet=None, adapter=make("tiny_sd"), scheduler=None)
    with pytest.raises(ValueError, match="one image tensor"):
        single(prompt_embeds=torch.zeros(1, 4, 8), image=[img, img])
    with pytest.raises(ValueError, match="image"):
        single(prompt_embeds=torch.zeros(1, 4, 8))


# ---- adapter_conditioning_factor --------------------------------------------------------------------------------------
@pytest.mark.parametrize("factor,steps,expected", [
    (0.0, 1, 0), (0.0, 7, 0), (0.0, 50, 0),
    (0.5, 1, 0), (0.5, 7, 3), (0.5, 50, 25),
    (1.0, 1, 1), (1.0, 7, 7), (1.0, 50, 50)])
def test_factor_cut_off(factor, steps, expected, monkeypatch):
    """Steps i < int(steps * factor) get the residuals; the pipeline zeroes its buffers at step int(steps * factor)."""
    on = OA.residual_steps(steps, factor)
    assert on == [True] * expected + [False] * (steps - expected)
    from paddlemix_b200.ppdiffusers.pipelines import StableDiffusionAdapterPipeline
    pipe = StableDiffusionAdapterPipeline(unet=None, adapter=make("tiny_sd"), scheduler=None)
    pipe._adapter = dict(cut=int(steps * factor), bufs=[torch.zeros(1, 8)])
    zeroed = []
    monkeypatch.setattr(ops, "zero_", lambda t: zeroed.append(i))
    for i in range(steps):
        with pytest.raises(AttributeError):  # no UNet here: only the cut-off bookkeeping before it runs
            pipe._predict(None, i, 0, None, None, None, i == 0)
    assert zeroed == ([] if expected == steps else [expected])


# ---- ReLU is element-wise only ----------------------------------------------------------------------------------------
class _NoKernels:
    def __getattr__(self, name):
        raise AssertionError(f"{name} was reached")


@pytest.mark.parametrize("call", [
    lambda: ops.linear(torch.zeros(4, 64, dtype=bf16), torch.zeros(128, 64, dtype=bf16), act=ACT_RELU),
    lambda: ops.linear(torch.zeros(4, 64, dtype=bf16),
                       ops.Int8Weight(torch.zeros(128 * 64, dtype=torch.int8), torch.zeros(128), 128, 64, None),
                       act=ACT_RELU),
    lambda: ops.linear_batched(torch.zeros(2, 8, 64, dtype=bf16), torch.zeros(128, 64, dtype=bf16),
                               out=torch.zeros(2, 8, 128, dtype=bf16), act=ACT_RELU),
    lambda: ops.conv3x3(torch.zeros(1, 8, 8, 64, dtype=bf16), torch.zeros(64, 3, 3, 64, dtype=bf16), act=ACT_RELU),
    lambda: ops.conv3x3_up2x(torch.zeros(1, 4, 4, 64, dtype=bf16), torch.zeros(64, 16, 64, dtype=bf16), act=ACT_RELU)])
def test_gemm_wrappers_refuse_relu_before_any_c_call(call, monkeypatch):
    monkeypatch.setattr(ops, "lib", _NoKernels())
    with pytest.raises(ValueError, match="not a GEMM epilogue activation"):
        call()


def test_activation_accepts_relu_and_refuses_unknown(monkeypatch):
    monkeypatch.setattr(ops, "lib", _NoKernels())
    with pytest.raises(_lib.B200MixError, match="CUDA tensor"):
        ops.activation(torch.zeros(16, dtype=bf16), ACT_RELU)
    with pytest.raises(ValueError, match="unknown act"):
        ops.activation(torch.zeros(16, dtype=bf16), 6)


# ---- the new wrappers' own refusals -----------------------------------------------------------------------------------
@pytest.mark.parametrize("call,err,pattern", [
    (lambda: ops.pixel_unshuffle(torch.zeros(1, 3, 64, 64), 8), _lib.B200MixError, "CUDA tensor"),
    (lambda: ops.pixel_unshuffle(torch.zeros(1, 3, 60, 64), 8), ValueError, "multiples of 8"),
    (lambda: ops.pixel_unshuffle(torch.zeros(1, 3, 64, 64), 4), ValueError, "8 or 16"),
    (lambda: ops.pixel_unshuffle(torch.zeros(1, 3, 64, 64, dtype=torch.float16), 8), TypeError, "x must be"),
    (lambda: ops.pixel_unshuffle(torch.zeros(1, 64, 64, 3).permute(0, 3, 1, 2), 8), ValueError, "contiguous"),
    (lambda: ops.pixel_unshuffle(torch.zeros(1 + 3 * 64 * 64)[1:].view(1, 3, 64, 64), 8), ValueError, "16-byte"),
    (lambda: ops.avgpool2x2_nhwc(torch.zeros(1, 5, 7, 64, dtype=bf16)), _lib.B200MixError, "CUDA tensor"),
    (lambda: ops.avgpool2x2_nhwc(torch.zeros(1, 5, 7, 12, dtype=bf16)), ValueError, "multiple of 8"),
    (lambda: ops.avgpool2x2_nhwc(torch.zeros(1, 5, 7, 64)), TypeError, "x must be"),
    (lambda: ops.weighted_sum_rows([torch.zeros(2, 4, 8, dtype=bf16)], [1.0], torch.zeros(4, 4, 8, dtype=bf16)),
     _lib.B200MixError, "CUDA tensor"),
    (lambda: ops.weighted_sum_rows([torch.zeros(2, 4, 8, dtype=bf16)], [1.0, 2.0], torch.zeros(4, 4, 8, dtype=bf16)),
     ValueError, "one weight each"),
    (lambda: ops.weighted_sum_rows([torch.zeros(2, 4, 16, dtype=bf16)], [1.0], torch.zeros(4, 4, 8, dtype=bf16)),
     ValueError, "xs\\[0\\] must be"),
    (lambda: ops.weighted_sum_rows([torch.zeros(2, 3, dtype=bf16)], [1.0], torch.zeros(4, 3, dtype=bf16)),
     ValueError, "multiple of 8"),
    (lambda: ops.weighted_sum_rows([torch.zeros(2, 8, dtype=bf16)] * 9, [1.0] * 9, torch.zeros(4, 8, dtype=bf16)),
     ValueError, "1 to 8 inputs")])
def test_new_wrappers_check_their_inputs(call, err, pattern, monkeypatch):
    monkeypatch.setattr(ops, "lib", _NoKernels())
    with pytest.raises(err, match=pattern):
        call()
