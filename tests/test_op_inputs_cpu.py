"""Every launching wrapper in ops refuses a malformed tensor before anything reaches a kernel. The kernels see pointers
and the sizes and strides passed beside them, never the tensors, so a wrong dtype, a short buffer or an unviewable
output would otherwise be misread, written out of bounds or silently lost. The checks run before the CUDA-placement
check, so CPU tensors show every refusal here, and a well-formed call on CPU tensors gets as far as that check."""
import ast
import pathlib

import pytest
import torch

from paddlemix_b200 import _lib, ops
from paddlemix_b200._lib import ACT_SILU, GLU_SWIGLU

bf16, f32, f16, i32, i64 = torch.bfloat16, torch.float32, torch.float16, torch.int32, torch.int64


def t(*shape, dtype=bf16):
    return torch.zeros(shape, dtype=dtype)


class _NoKernels:
    def __getattr__(self, name):
        raise AssertionError(f"{name} was reached with invalid inputs")


def _beam(**over):
    B, nb, V, max_new = 2, 2, 64, 5
    rows = B * nb
    kw = dict(state=t(4, dtype=i64), next_ids=t(rows, dtype=i64), beam_scores=t(rows, dtype=f32),
              tokens=t(max_new, rows, dtype=i64), parents=t(max_new, rows, dtype=i32), hyp_score=t(rows, dtype=torch.float64),
              hyp_step=t(rows, dtype=i32), hyp_slot=t(rows, dtype=i32), hyp_count=t(B, dtype=i32),
              hyp_worst=t(B, dtype=torch.float64), done=t(B, dtype=i32), presence=t(2, rows, 2, dtype=i32))
    kw.update(over)
    return ops.beam_search_step(t(rows, V, dtype=f32), nb, t(256, dtype=torch.uint8), **kw)


def _sample(**over):
    kw = dict(logits=t(2, 64, dtype=f32), presence=t(2, 2, dtype=i32), finished=t(2, dtype=i32), state=t(4, dtype=i64),
              out=t(2, 5, dtype=i64), next_ids=t(2, dtype=i64))
    kw.update(over)
    return ops.sample_tokens(**kw)


# op -> a call whose keyword arguments replace well-formed defaults
CALLS = {
    "linear": lambda a=t(4, 6, 64), w=t(128, 64), **kw: ops.linear(a, w, **kw),
    "linear_w8": lambda a=t(4, 64), out=None, **kw: ops.linear(a, ops.Int8Weight(t(128 * 64, dtype=torch.int8),
                                                                              t(128, dtype=f32), 128, 64, None), out=out, **kw),
    "linear_batched": lambda a=t(2, 8, 64), w=t(128, 64), out=t(2, 8, 128), **kw: ops.linear_batched(a, w, out=out, **kw),
    "quantize_w8": lambda w=t(128, 64), workspace=t(128 * 64): ops.quantize_w8(w, workspace),
    "patchify": lambda x=t(2, 4, 8, 8): ops.patchify(x, 2),
    "unpatchify": lambda x=t(2, 16, 16), out_dtype=bf16: ops.unpatchify(x, 4, 4, 4, 2, out_dtype=out_dtype),
    "conv3x3": lambda x=t(2, 8, 8, 64), w=t(128, 3, 3, 64), **kw: ops.conv3x3(x, w, **kw),
    "conv3x3_up2x": lambda x=t(2, 4, 4, 64), w4=t(128, 16, 64), **kw: ops.conv3x3_up2x(x, w4, **kw),
    "conv3x3_small_cin": lambda x=t(2, 8, 8, 4, dtype=f32), w=t(64, 3, 3, 4), bias=t(64, dtype=f32):
        ops.conv3x3_small_cin(x, w, bias),
    "conv3x3_narrow": lambda x=t(2, 8, 8, 3), w=t(16, 3, 3, 3), **kw: ops.conv3x3_narrow(x, w, **kw),
    "sdpa": lambda q=t(2, 16, 4, 64), k=t(2, 32, 2, 64), v=t(2, 32, 2, 64), **kw: ops.sdpa(q, k, v, **kw),
    "groupnorm_nhwc": lambda x1=t(2, 4, 4, 64), gamma=t(96, dtype=f32), beta=t(96, dtype=f32), x2=t(2, 4, 4, 32):
        ops.groupnorm_nhwc(x1, gamma, beta, x2=x2),
    "layernorm": lambda x=t(4, 64), **kw: ops.layernorm(x, **kw),
    "softmax_rows": lambda x=t(8, 64, dtype=f32), **kw: ops.softmax_rows(x, **kw),
    "timestep_embedding": lambda ts=t(2, dtype=f32), **kw: ops.timestep_embedding(ts, 64, **kw),
    "activation": lambda x=t(8), out_dtype=None: ops.activation(x, ACT_SILU, out_dtype),
    "upsample_nearest2x": lambda x=t(2, 4, 4, 8): ops.upsample_nearest2x(x),
    "concat_channels": lambda x1=t(2, 4, 8), x2=t(2, 4, 16): ops.concat_channels(x1, x2),
    "nchw_to_nhwc": lambda x=t(2, 8, 4, 4): ops.nchw_to_nhwc(x),
    "nhwc_to_nchw": lambda x=t(2, 4, 4, 8), **kw: ops.nhwc_to_nchw(x, **kw),
    "add_residual_nhwc": lambda a=t(2, 4, 4, 8), r=t(2, 8, 4, 4, dtype=f32), **kw: ops.add_residual_nhwc(a, r, r_nchw=True, **kw),
    "iddpm_step": lambda m=t(4, 8, 16, dtype=f32), x=t(2, 4, 16, dtype=f32), **kw:
        ops.iddpm_step(m, x, 4.0, 4, (1.0,) * 6, True, **kw),
    "scale_model_input": lambda x=t(8, dtype=f32), **kw: ops.scale_model_input(x, 2.0, **kw),
    "cast": lambda x=t(8, dtype=f32), dtype=bf16: ops.cast(x, dtype),
    "rope_inplace": lambda x=t(6, 2, 64), cos=t(6, 64, dtype=f32), sin=t(6, 64, dtype=f32), **kw:
        ops.rope_inplace(x, cos, sin, **kw),
    "decode_rope_cache": lambda qkv=t(2, 4 * 64), rows=t(2, dtype=i64), cache_k=t(16, 64), cache_v=t(16, 64):
        ops.decode_rope_cache(qkv, 2, 1, 64, t(2, 64, dtype=f32), t(2, 64, dtype=f32), rows, cache_k, cache_v),
    "sample_tokens": _sample,
    "beam_search_step": _beam,
    "kv_reorder": lambda layer_kv=t(4, dtype=i64), cache_k=t(4, 16, 2, 8), parents=t(5, 4, dtype=i32), done=t(2, dtype=i32):
        ops.kv_reorder(layer_kv, cache_k, 2, 3, parents, t(4, dtype=i64), done),
    "gather_rows": lambda table=t(32, 64), ids=t(5, dtype=i64): ops.gather_rows(table, ids),
    "scatter_rows": lambda src=t(5, 64), idx=t(5, dtype=i64), dst=t(32, 64): ops.scatter_rows(src, idx, dst),
    "broadcast_add": lambda x=t(2, 64, dtype=f32), table=t(6, 64, dtype=f32): ops.broadcast_add(x, table),
    "head_rmsnorm_inplace": lambda x=t(8, 2, 128), weight=t(72, dtype=f32): ops.head_rmsnorm_inplace(x, weight, 72),
    "small_attention": lambda qkv=t(2 * 4 * 3, 3 * 2 * 16), **kw: ops.small_attention(qkv, 2, 4, 3, 2, 16, scale=0.25, **kw),
    "patchify3d": lambda x=t(2, 4, 3, 8, 8): ops.patchify3d(x, 2),
    "unpatchify3d": lambda x=t(2, 3 * 16, 16): ops.unpatchify3d(x, 4, 3, 4, 4, 2),
}
# the sampler steps (ddim_step, lcm_step, euler_step, dpmpp_2m_step, cfg_combine) are covered by test_step_inputs_cpu

BAD = {  # (op, its keyword arguments, the error, a pattern of its message)
    "linear: out of the wrong dtype": ("linear", lambda: dict(out_fp32=True, out=t(4, 6, 128)), TypeError, "out must be"),
    "linear: out too small": ("linear", lambda: dict(out=t(4, 5, 128)), ValueError, "out has"),
    "linear: unviewable out": ("linear", lambda: dict(out=t(6, 4, 128).transpose(0, 1)), ValueError, "cannot be viewed"),
    "linear: strided out": ("linear", lambda: dict(out=t(4, 6, 256)[..., ::2]), ValueError, "out needs a contiguous last"),
    "linear: residual rows": ("linear", lambda: dict(residual=t(20, 128)), ValueError, "residual of shape"),
    "linear: residual columns": ("linear", lambda: dict(residual=t(24, 64)), ValueError, "residual of shape"),
    "linear: bias length": ("linear", lambda: dict(bias=t(64, dtype=f32)), ValueError, "bias has"),
    "linear: bias dtype": ("linear", lambda: dict(bias=t(128)), TypeError, "bias must be"),
    "linear: weight K": ("linear", lambda: dict(w=t(128, 32)), ValueError, "weight must be"),
    "linear: weight strides": ("linear", lambda: dict(w=t(64, 128).t()), ValueError, "weight needs a contiguous"),
    "linear: stats table": ("linear", lambda: dict(stats=t(24, 3, dtype=i64)), ValueError, "stats must be"),
    "linear: int8 out dtype": ("linear_w8", lambda: dict(out_fp32=True, out=t(4, 128)), TypeError, "out must be"),
    "linear: int8 residual rows": ("linear_w8", lambda: dict(residual=t(3, 128)), ValueError, "residual of shape"),
    "linear: int8 input width": ("linear_w8", lambda: dict(a=t(4, 32)), ValueError, "a must be"),
    "linear_batched: out shape": ("linear_batched", lambda: dict(out=t(2, 7, 128)), ValueError, "out must be"),
    "linear_batched: residual": ("linear_batched", lambda: dict(residual=t(2, 8, 64)), ValueError, "residual must be"),
    "quantize_w8: weight dtype": ("quantize_w8", lambda: dict(w=t(128, 64, dtype=f16)), TypeError, "w must be"),
    "quantize_w8: workspace": ("quantize_w8", lambda: dict(workspace=t(100)), ValueError, "workspace holds"),
    "patchify: strided x": ("patchify", lambda: dict(x=t(2, 4, 8, 8).transpose(2, 3)), ValueError, "x must be contiguous"),
    "unpatchify: short x": ("unpatchify", lambda: dict(x=t(2, 15, 16)), ValueError, "x has"),
    "unpatchify: fp16 output": ("unpatchify", lambda: dict(out_dtype=f16), TypeError, "out must be"),
    "conv3x3: weight Cin": ("conv3x3", lambda: dict(w=t(128, 3, 3, 32)), ValueError, "w must be"),
    "conv3x3: residual": ("conv3x3", lambda: dict(residual=t(2, 8, 8, 64)), ValueError, "residual must be"),
    "conv3x3: out of a stride-2 conv": ("conv3x3", lambda: dict(stride=2, out=t(2, 8, 8, 128)), ValueError, "out must be"),
    "conv3x3: row_add groups": ("conv3x3", lambda: dict(row_add=t(1, 128, dtype=f32)), ValueError, "does not cover"),
    "conv3x3_up2x: folded weight": ("conv3x3_up2x", lambda: dict(w4=t(128, 9, 64)), ValueError, "w4 must be"),
    "conv3x3_up2x: out": ("conv3x3_up2x", lambda: dict(out=t(2, 4, 4, 128)), ValueError, "out must be"),
    "conv3x3_small_cin: fp16 x": ("conv3x3_small_cin", lambda: dict(x=t(2, 8, 8, 4, dtype=f16)), TypeError, "x must be"),
    "conv3x3_small_cin: bias": ("conv3x3_small_cin", lambda: dict(bias=t(32, dtype=f32)), ValueError, "bias has"),
    "conv3x3_narrow: bias": ("conv3x3_narrow", lambda: dict(bias=t(16)), TypeError, "bias must be"),
    "sdpa: int64 cu_seqlens": ("sdpa", lambda: dict(cu_seqlens=t(3, dtype=i64)), TypeError, "cu_seqlens must be"),
    "sdpa: int64 kv_lens": ("sdpa", lambda: dict(kv_lens=t(2, dtype=i64)), TypeError, "kv_lens must be"),
    "sdpa: kv_lens length": ("sdpa", lambda: dict(kv_lens=t(3, dtype=i32)), ValueError, "kv_lens has"),
    "sdpa: k batch": ("sdpa", lambda: dict(k=t(1, 32, 2, 64)), ValueError, "k must be"),
    "sdpa: k head size": ("sdpa", lambda: dict(k=t(2, 32, 2, 128)), ValueError, "k must be"),
    "sdpa: v shape": ("sdpa", lambda: dict(v=t(2, 16, 2, 64)), ValueError, "v must be"),
    "sdpa: query heads": ("sdpa", lambda: dict(k=t(2, 32, 3, 64), v=t(2, 32, 3, 64)), ValueError, "query heads"),
    "sdpa: q strides": ("sdpa", lambda: dict(q=t(2, 16, 4, 68)[..., :64]), ValueError, "multiples of 8"),
    "groupnorm_nhwc: gamma": ("groupnorm_nhwc", lambda: dict(gamma=t(64, dtype=f32)), ValueError, "gamma has"),
    "groupnorm_nhwc: beta dtype": ("groupnorm_nhwc", lambda: dict(beta=t(96)), TypeError, "beta must be"),
    "groupnorm_nhwc: x2 rows": ("groupnorm_nhwc", lambda: dict(x2=t(2, 4, 2, 32)), ValueError, "x2 must be"),
    "layernorm: weight": ("layernorm", lambda: dict(weight=t(32, dtype=f32)), ValueError, "weight has"),
    "layernorm: delta": ("layernorm", lambda: dict(delta=t(3, 64)), ValueError, "delta must be"),
    "layernorm: fp16 x": ("layernorm", lambda: dict(x=t(4, 64, dtype=f16)), TypeError, "x must be"),
    "softmax_rows: out": ("softmax_rows", lambda: dict(out=t(8, 32)), ValueError, "out must be"),
    "timestep_embedding: columns": ("timestep_embedding", lambda: dict(out=t(2, 96), col0=40), ValueError, "do not fit"),
    "timestep_embedding: out rows": ("timestep_embedding", lambda: dict(out=t(3, 64)), ValueError, "out must be"),
    "activation: fp16 x": ("activation", lambda: dict(x=t(8, dtype=f16)), TypeError, "x must be"),
    "activation: fp16 out": ("activation", lambda: dict(out_dtype=f16), TypeError, "out must be"),
    "upsample_nearest2x: strided x": ("upsample_nearest2x", lambda: dict(x=t(2, 4, 4, 16)[..., :8]), ValueError,
                                      "x must be contiguous"),
    "concat_channels: x2 rows": ("concat_channels", lambda: dict(x2=t(2, 3, 16)), ValueError, "x2 must be"),
    "concat_channels: x2 dtype": ("concat_channels", lambda: dict(x2=t(2, 4, 16, dtype=f32)), TypeError, "x2 must be"),
    "nchw_to_nhwc: fp16 x": ("nchw_to_nhwc", lambda: dict(x=t(2, 8, 4, 4, dtype=f16)), TypeError, "x must be"),
    "nhwc_to_nchw: out": ("nhwc_to_nchw", lambda: dict(out=t(2, 4, 4, 8, dtype=f32)), ValueError, "out must be"),
    "add_residual_nhwc: r shape": ("add_residual_nhwc", lambda: dict(r=t(2, 4, 4, 8, dtype=f32)), ValueError, "residual shape"),
    "add_residual_nhwc: out": ("add_residual_nhwc", lambda: dict(out=t(2, 4, 4, 8, dtype=f32)), TypeError, "out must be"),
    "iddpm_step: model_out": ("iddpm_step", lambda: dict(m=t(4, 4, 16, dtype=f32)), ValueError, "model_out must be"),
    "iddpm_step: noise": ("iddpm_step", lambda: dict(noise=t(2, 4, 8, dtype=f32)), ValueError, "noise must be"),
    "iddpm_step: out_dup": ("iddpm_step", lambda: dict(out_dup=t(2, 4, 16)), TypeError, "out_dup must be"),
    "scale_model_input: out": ("scale_model_input", lambda: dict(out=t(4, dtype=f32)), ValueError, "out has"),
    "cast: fp16 x": ("cast", lambda: dict(x=t(8, dtype=f16)), TypeError, "x must be"),
    "cast: fp16 out": ("cast", lambda: dict(dtype=f16), TypeError, "out must be"),
    "rope_inplace: bf16 table": ("rope_inplace", lambda: dict(cos=t(6, 64)), TypeError, "cos must be"),
    "rope_inplace: table rows": ("rope_inplace", lambda: dict(sin=t(5, 64, dtype=f32)), ValueError, "sin must be"),
    "rope_inplace: rot_dim": ("rope_inplace", lambda: dict(rot_dim=128), ValueError, "rot_dim"),
    "decode_rope_cache: qkv width": ("decode_rope_cache", lambda: dict(qkv=t(2, 3 * 64)), ValueError, "qkv must be"),
    "decode_rope_cache: rows dtype": ("decode_rope_cache", lambda: dict(rows=t(2, dtype=i32)), TypeError, "rows must be"),
    "decode_rope_cache: cache": ("decode_rope_cache", lambda: dict(cache_v=t(16, 128)), ValueError, "cache_v must be"),
    "sample_tokens: presence": ("sample_tokens", lambda: dict(presence=t(2, 1, dtype=i32)), ValueError, "presence must be"),
    "sample_tokens: finished": ("sample_tokens", lambda: dict(finished=t(3, dtype=i32)), ValueError, "finished has"),
    "sample_tokens: out dtype": ("sample_tokens", lambda: dict(out=t(2, 5, dtype=i32)), TypeError, "out must be"),
    "beam_search_step: hyp_score": ("beam_search_step", lambda: dict(hyp_score=t(4, dtype=f32)), TypeError,
                                    "hyp_score must be"),
    "beam_search_step: parents": ("beam_search_step", lambda: dict(parents=t(4, 4, dtype=i32)), ValueError,
                                  "parents must be"),
    "kv_reorder: parents": ("kv_reorder", lambda: dict(parents=t(5, 3, dtype=i32)), ValueError, "parents must be"),
    "kv_reorder: done": ("kv_reorder", lambda: dict(done=t(4, dtype=i32)), ValueError, "done has"),
    "gather_rows: strided table": ("gather_rows", lambda: dict(table=t(64, 32).t()), ValueError, "table must be contiguous"),
    "gather_rows: ids dtype": ("gather_rows", lambda: dict(ids=t(5, dtype=i32)), TypeError, "ids must be"),
    "scatter_rows: dst width": ("scatter_rows", lambda: dict(dst=t(32, 128)), ValueError, "dst must be"),
    "scatter_rows: idx length": ("scatter_rows", lambda: dict(idx=t(6, dtype=i64)), ValueError, "idx has"),
    "scatter_rows: strided src": ("scatter_rows", lambda: dict(src=t(5, 128)[:, ::2]), ValueError, "src must be contiguous"),
    "broadcast_add: table width": ("broadcast_add", lambda: dict(table=t(6, 32, dtype=f32)), ValueError, "table must be"),
    "head_rmsnorm_inplace: weight": ("head_rmsnorm_inplace", lambda: dict(weight=t(64, dtype=f32)), ValueError, "weight has"),
    "small_attention: qkv rows": ("small_attention", lambda: dict(qkv=t(20, 96)), ValueError, "qkv must be"),
    "small_attention: qkv width": ("small_attention", lambda: dict(qkv=t(24, 90)), ValueError, "qkv has 90 columns"),
    "small_attention: out width": ("small_attention", lambda: dict(out=t(24, 16)), ValueError, "out has 16 columns"),
    "small_attention: rope table": ("small_attention", lambda: dict(rope_cos=t(4, 16, dtype=f32), rope_sin=t(4, 8, dtype=f32)),
                                    ValueError, "rope_cos must be"),
    "small_attention: norm weight": ("small_attention", lambda: dict(q_norm_w=t(16), k_norm_w=t(16, dtype=f32)), TypeError,
                                     "q_norm_w must be"),
    "unpatchify3d: short x": ("unpatchify3d", lambda: dict(x=t(2, 47, 16)), ValueError, "x has"),
}


@pytest.mark.parametrize("op", list(CALLS))
def test_op_passes_well_formed_inputs_to_the_device_check(op, monkeypatch):
    monkeypatch.setattr(ops, "lib", _NoKernels())
    with pytest.raises(_lib.B200MixError, match="CUDA tensor"):
        CALLS[op]()


@pytest.mark.parametrize("case", list(BAD))
def test_op_refuses_malformed_inputs_before_launch(case, monkeypatch):
    monkeypatch.setattr(ops, "lib", _NoKernels())
    op, kwargs, err, pattern = BAD[case]
    with pytest.raises(err, match=pattern):
        CALLS[op](**kwargs())


def test_ops_has_no_assert():
    """python -O strips assert statements: no input check in ops may be one."""
    tree = ast.parse(pathlib.Path(ops.__file__).read_text())
    assert not [n.lineno for n in ast.walk(tree) if isinstance(n, ast.Assert)]


def test_stdit2_refuses_hidden_size_not_divisible_by_3():
    from paddlemix_b200.opensora.stdit2 import STDiT2
    with pytest.raises(ValueError, match="divisible by 3"):
        STDiT2(dict(hidden_size=64, depth=1, num_heads=2))
