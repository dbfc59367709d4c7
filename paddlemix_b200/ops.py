"""Tensor-level wrappers over the C ABI. torch is used for device memory and streams only: every function below
enqueues hand-written sm_90a kernels from libb200mix.so on torch's current CUDA stream and raises if that fails.
"""
import ctypes
from typing import Optional

import torch

from . import _lib
from ._lib import (ACT_GELU_ERF, ACT_GELU_TANH, ACT_NONE, ACT_QUICK_GELU, ACT_SILU, GLU_GEGLU, GLU_NONE, GLU_SWIGLU,
                   Epilogue, check, lib)

bf16 = torch.bfloat16
_launches = 0  # number of our kernels launched (bench.py reports it as gpu_launches)


def launches() -> int:
    return _launches


def reset_launches():
    global _launches
    _launches = 0


def _count(n=1):
    global _launches
    _launches += n


# ---- optional per-launch timing (bench.py's roofline section): CUDA events on the launching stream ----------------
_prof = None  # list of (kind, work, unit, start_event, end_event) while profiling


def profile_begin():
    global _prof
    _prof = []


def profile_end(by_tag=False):
    """Returns {kind: dict(ms, work, unit, calls)} for the launches since profile_begin(); by_tag=True keys the table
    by the per-call shape tag ("lin 8192x1280x640 b+res", ...) instead of the kernel family."""
    global _prof
    recs, _prof = _prof, None
    torch.cuda.synchronize()
    out = {}
    for kind, tag, work, unit, e0, e1 in recs:
        d = out.setdefault((tag or kind) if by_tag else kind, dict(ms=0.0, work=0.0, unit=unit, calls=0))
        d["ms"] += e0.elapsed_time(e1)
        d["work"] += work
        d["calls"] += 1
    return out


class _Timed:
    __slots__ = ("kind", "work", "unit", "e0", "tag")

    def __init__(self, kind, work, unit, tag=None):
        self.kind, self.work, self.unit, self.tag = kind, work, unit, tag

    def __enter__(self):
        if _prof is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e0.record()

    def __exit__(self, *a):
        if _prof is not None:
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            _prof.append((self.kind, self.tag() if callable(self.tag) else self.tag, self.work, self.unit, self.e0, e1))


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t: Optional[torch.Tensor]):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _req(t, dtype, name):
    if not t.is_cuda:
        raise _lib.B200MixError(f"{name} must be a CUDA tensor (b200mix has no CPU path)")
    if t.dtype != dtype:
        raise TypeError(f"{name} must be {dtype}, got {t.dtype}")
    return t


def init(device: int = 0):
    check(lib.b200mix_init(int(device)), "b200mix_init")


def _check_mod_views(op, **mods):
    """Per-group vectors (AdaLN scale / shift / gate, row_add / row_gate) reach the kernels as (pointer, stride(0)) and
    are read at group * stride(0) + column: a [groups, width] view is fine, a column stride other than 1 is not, and
    vectors passed together must share stride(0) (one stride reaches the kernel)."""
    given = {k: v for k, v in mods.items() if v is not None}
    for name, v in given.items():
        if v.dim() == 0 or (v.dim() > 1 and v.shape[-1] > 1 and v.stride(-1) != 1):
            raise ValueError(f"{op}: {name} must be a [groups, width] view with a contiguous last dimension, "
                             f"got shape {tuple(v.shape)} strides {v.stride()}")
        if v.dim() == 1 and v.shape[0] > 1 and v.stride(0) != 1:
            raise ValueError(f"{op}: {name} must be contiguous, got stride {v.stride(0)}")
    lds = {v.stride(0) for v in given.values() if v.dim() > 1 and v.shape[0] > 1}
    if len(lds) > 1:
        raise ValueError(f"{op}: {', '.join(given)} must share one row stride, got {sorted(lds)}")


def _check_mod_groups(op, rows, rows_per_group, width, **mods):
    """Row r of the output reads per-group vector r // rows_per_group (one group when rows_per_group is 0), columns
    0..width-1. A [groups, *] view must cover every group and every column, and a view with several groups used with
    rows_per_group = 0 would apply its first row to all rows."""
    for name, v in mods.items():
        if v is None or v.dim() < 2:
            if v is not None and v.shape[-1] < width:
                raise ValueError(f"{op}: {name} has {v.shape[-1]} columns, the output has {width}")
            continue
        groups = 1 if rows_per_group <= 0 else -(-rows // rows_per_group)
        if rows_per_group <= 0 and v.shape[0] > 1:
            raise ValueError(f"{op}: {name} holds {v.shape[0]} groups but rows_per_group is not set")
        if v.shape[0] < groups or v.shape[-1] < width:
            raise ValueError(f"{op}: {name} of shape {tuple(v.shape)} does not cover {groups} groups x {width} columns "
                             f"({rows} rows, rows_per_group {rows_per_group})")


def make_epilogue(bias=None, row_add=None, row_gate=None, ld_row=0, rows_per_group=0, residual=None, ldr=0,
                  act=ACT_NONE, glu=GLU_NONE, out_fp32=False, out_scale=1.0, residual_row_mod=0, stats_out=None,
                  ln=None) -> Epilogue:
    e = Epilogue()
    e.bias = None if bias is None else _req(bias, torch.float32, "bias").data_ptr()
    e.row_add = None if row_add is None else _req(row_add, torch.float32, "row_add").data_ptr()
    e.row_gate = None if row_gate is None else _req(row_gate, torch.float32, "row_gate").data_ptr()
    e.ld_row = int(ld_row)
    e.rows_per_group = int(rows_per_group)
    e.residual = None if residual is None else _req(residual, bf16, "residual").data_ptr()
    e.ldr = int(ldr)
    e.act = int(act)
    e.glu = int(glu)
    e.out_fp32 = 1 if out_fp32 else 0
    e.out_scale = float(out_scale)
    e.residual_row_mod = int(residual_row_mod)
    e.stats_out = None if stats_out is None else _req(stats_out, torch.int64, "stats_out").data_ptr()
    if ln is not None:  # folded LayerNorm, consumer side: (RowStats of the input rows, colsum [N] fp32, eps[, rms])
        stats, colsum, eps = ln[:3]
        e.ln_stats = _req(stats.buf, torch.int64, "ln_stats").data_ptr()
        e.ln_colsum = _req(colsum, torch.float32, "ln_colsum").data_ptr()
        e.ln_eps, e.ln_rms = float(eps), int(bool(ln[3])) if len(ln) > 3 else 0
    return e


class RowStats:
    """Sum and sum of squares of every row of a bf16 [M, N] GEMM output, accumulated by that GEMM's epilogue
    (linear(..., stats=...)) as 2^24 fixed point: buf int64 [M, 2], zeroed before the producing call. Consumed by
    linear(..., ln=(stats, colsum, eps))."""
    SCALE = float(1 << 24)

    def __init__(self, buf: torch.Tensor, width: int):
        self.buf, self.width = buf, width

    @staticmethod
    def arena(n: int, rows: int, device) -> torch.Tensor:
        """n zeroed [rows, 2] tables in one allocation / one memset (a transformer stack takes 1 + 3 per block)."""
        buf = torch.empty(n, rows, 2, device=device, dtype=torch.int64)
        check(lib.b200mix_zero_bytes(_p(buf), buf.numel() * 8, _stream()), "b200mix_zero_bytes")
        return buf

    def mean_rstd(self, eps: float):
        """(mean, rstd) per row, the way the consuming epilogue rebuilds them (for tests)."""
        t = self.buf.double() / self.SCALE
        mean = t[:, 0] / self.width
        var = (t[:, 1] / self.width - mean * mean).clamp_min(0)
        return mean.float(), torch.rsqrt(var.float() + eps)


def fold_layernorm_into_linear(w: torch.Tensor, gamma: torch.Tensor, beta=None, bias=None):
    """w: fp32 [N, K] (the consumer's weight), gamma / beta: the LayerNorm affine over K, bias: the consumer's bias or None.
    Returns (W' bf16 [N, K], colsum fp32 [N], bias' fp32 [N]) for linear(h, W', bias', ln=(stats, colsum, eps)) ==
    linear(layernorm(h) * gamma + beta, w, bias)."""
    wf = w.float()
    w2 = (wf * gamma.float()[None, :]).to(bf16).contiguous()
    colsum = w2.float().sum(1).contiguous()
    b2 = torch.zeros(w.shape[0], device=w.device, dtype=torch.float32) if bias is None else bias.float().clone()
    if beta is not None:
        b2 = b2 + wf @ beta.float()
    return w2, colsum, b2.contiguous()



def _epi_tag(e) -> str:
    parts = [n for n, on in (("ln", e.ln_stats), ("bias", e.bias), ("radd", e.row_add), ("gate", e.row_gate),
                             ("res", e.residual), (f"act{e.act}", e.act), (f"glu{e.glu}", e.glu), ("f32", e.out_fp32),
                             ("stats", e.stats_out)) if on]
    return (" " + "+".join(parts)) if parts else ""


class Int8Weight:
    """A Linear weight [N, K] quantized to int8 with one fp32 scale per output row (quantize_w8). q holds the N * K
    bytes in the device layout of b200mix_quantize_w8 (only the kernels read it); workspace is the bf16 buffer linear()
    expands the weight into when M is above the weight-streaming range, shared by every weight of a model (None: such
    calls are refused)."""
    __slots__ = ("q", "scale", "N", "K", "workspace")

    def __init__(self, q: torch.Tensor, scale: torch.Tensor, N: int, K: int, workspace: Optional[torch.Tensor]):
        self.q, self.scale, self.N, self.K, self.workspace = q, scale, N, K, workspace


def quantize_w8(w: torch.Tensor, workspace: Optional[torch.Tensor]) -> Int8Weight:
    """Weight-only int8 of w fp32 or bf16 [N, K] on the device (N % 16 == 0, K % 64 == 0): per row scale = absmax / 127,
    q = clip(round(w / scale), -127, 127), rounding half away from zero; an all-zero row gets scale 0. workspace: bf16
    with at least N * K elements, or None."""
    if w.dtype not in (torch.float32, bf16):
        raise TypeError(f"quantize_w8 takes an fp32 or bf16 weight, got {w.dtype}")
    _req(w, w.dtype, "w")
    if w.dim() != 2:
        raise ValueError(f"quantize_w8 takes a [N, K] weight, got {tuple(w.shape)}")
    N, K = w.shape
    if workspace is not None and (_req(workspace, bf16, "workspace").numel() < N * K):
        raise ValueError(f"the workspace holds {workspace.numel()} bf16 elements, a [{N}, {K}] weight needs {N * K}")
    w = w.contiguous()
    q = torch.empty(N * K, device=w.device, dtype=torch.int8)
    scale = torch.empty(N, device=w.device, dtype=torch.float32)
    check(lib.b200mix_quantize_w8(_p(w), 1 if w.dtype == torch.float32 else 0, _p(q), _p(scale), N, K, _stream()),
          "b200mix_quantize_w8")
    _count()
    return Int8Weight(q, scale, N, K, workspace)


def _linear_w8(a, w: Int8Weight, bias, act, glu, residual, out_fp32, out):
    _req(a, bf16, "a")
    K = a.shape[-1]
    if K != w.K:
        raise ValueError(f"input has {K} features, the weight takes {w.K}")
    a2 = a.reshape(-1, K)
    if a2.stride(-1) != 1 or a2.data_ptr() % 16 or a2.stride(0) % 8:
        a2 = a2.contiguous()
    M, N = a2.shape[0], w.N
    n_out = N // 2 if glu else N
    if out is None:
        out = torch.empty(*a.shape[:-1], n_out, device=a.device, dtype=torch.float32 if out_fp32 else bf16)
    res2 = None if residual is None else residual.reshape(-1, residual.shape[-1])
    e = make_epilogue(bias=bias, residual=res2, ldr=0 if res2 is None else res2.stride(0), act=act, glu=glu,
                      out_fp32=out_fp32)
    out2 = out.reshape(-1, n_out)
    ws = w.workspace
    with _Timed("w8gemm", 2.0 * M * N * K, "flop", lambda: f"w8 {M}x{N}x{K}" + _epi_tag(e)):
        check(lib.b200mix_linear_w8(_p(a2), a2.stride(0), _p(w.q), _p(w.scale), _p(out2), out2.stride(0), M, N, K,
                                    ctypes.byref(e), _p(ws), 0 if ws is None else 2 * ws.numel(), _stream()),
              "b200mix_linear_w8")
    _count()
    return out


def linear(a: torch.Tensor, w, bias=None, *, act=ACT_NONE, glu=GLU_NONE, residual=None, row_add=None,
           row_gate=None, rows_per_group=0, out_fp32=False, out=None, out_scale=1.0, residual_row_mod=0, stats=False,
           ln=None):
    """out[M, N(/2)] = epilogue(a[M, K] @ w[N, K]^T). a: bf16 [..., K] (last dim contiguous), w: bf16 [N, K] or an
    Int8Weight (then only bias / act / glu / residual / out_fp32 / out apply).
    stats=True or a ZEROED int64 [M, 2] tensor (RowStats.arena): also returns the RowStats of the output rows
    (-> (out, RowStats)); ln=(RowStats of a's rows, colsum, eps[, rms]): a is the UN-normalised tensor and w / bias carry
    the folded affine (fold_layernorm_into_linear)."""
    if isinstance(w, Int8Weight):
        unsupported = [n for n, on in (("row_add", row_add is not None), ("row_gate", row_gate is not None),
                                       ("rows_per_group", rows_per_group), ("out_scale", out_scale != 1.0),
                                       ("residual_row_mod", residual_row_mod), ("stats", stats is not None and stats is not False),
                                       ("ln", ln is not None)) if on]
        if unsupported:
            raise ValueError(f"an Int8Weight linear does not support {', '.join(unsupported)}")
        return _linear_w8(a, w, bias, act, glu, residual, out_fp32, out)
    _req(a, bf16, "a"), _req(w, bf16, "w")
    K = a.shape[-1]
    if w.dim() != 2 or w.shape[1] != K:
        raise ValueError(f"linear: weight must be [N, {K}] for an input with {K} features, got {tuple(w.shape)}")
    a2 = a.reshape(-1, K)
    if a2.stride(-1) != 1:
        a2 = a2.contiguous()
    M, N = a2.shape[0], w.shape[0]
    n_out = N // 2 if glu else N
    if out is None:
        out = torch.empty(*a.shape[:-1], n_out, device=a.device, dtype=torch.float32 if out_fp32 else bf16)
    res2 = None
    if residual is not None:
        res2 = residual.reshape(-1, residual.shape[-1])
    mod = row_add if row_add is not None else row_gate
    if mod is not None:
        _check_mod_views("linear", row_add=row_add, row_gate=row_gate)
        _check_mod_groups("linear", M, rows_per_group, N, row_add=row_add, row_gate=row_gate)
    rs = None
    want_stats = stats is not None and stats is not False
    if want_stats:
        buf = RowStats.arena(1, M, a.device)[0] if stats is True else stats
        if tuple(buf.shape) != (M, 2):
            raise ValueError(f"stats table must be int64 [{M}, 2], got {tuple(buf.shape)}")
        rs = RowStats(buf, N)
    if ln is not None and (ln[0].buf.shape[0] != M or ln[0].width != K):
        raise ValueError(f"row statistics are for a [{ln[0].buf.shape[0]}, {ln[0].width}] tensor, the input is [{M}, {K}]")
    e = make_epilogue(bias=bias, row_add=row_add, row_gate=row_gate, ld_row=0 if mod is None else mod.stride(0),
                      rows_per_group=rows_per_group, residual=res2, ldr=0 if res2 is None else res2.stride(0), act=act,
                      glu=glu, out_fp32=out_fp32, out_scale=out_scale, residual_row_mod=residual_row_mod,
                      stats_out=None if rs is None else rs.buf, ln=ln)
    out2 = out.reshape(-1, n_out)
    with _Timed("igemm", 2.0 * M * N * K, "flop", lambda: f"lin {M}x{N}x{K}" + _epi_tag(e)):
        check(lib.b200mix_linear(_p(a2), a2.stride(0), _p(w), w.stride(0), _p(out2), out2.stride(0), M, N, K,
                                 ctypes.byref(e), _stream()), "b200mix_linear")
    _count()
    return (out, rs) if want_stats else out


def linear_batched(a: torch.Tensor, w: torch.Tensor, bias=None, *, out: torch.Tensor, act=ACT_NONE, glu=GLU_NONE,
                   residual=None, row_add=None, row_gate=None) -> torch.Tensor:
    """a: bf16 [B, rows, K] view (last dim contiguous, arbitrary row / batch strides); out: [B, rows, N(/2)] view with
    last dim contiguous (e.g. a token range of a joint [B, n_img+n_txt, *] buffer). Per-batch row_add / row_gate."""
    _req(a, bf16, "a"), _req(w, bf16, "w")
    B, rows, K = a.shape
    N = w.shape[0]
    if w.dim() != 2 or w.shape[1] != K:
        raise ValueError(f"linear_batched: weight must be [N, {K}] for an input with {K} features, got {tuple(w.shape)}")
    n_out = N // 2 if glu else N
    if out.dim() != 3 or tuple(out.shape) != (B, rows, n_out):
        raise ValueError(f"linear_batched: out must be [{B}, {rows}, {n_out}], got {tuple(out.shape)}")
    if residual is not None and tuple(residual.shape) != tuple(out.shape):
        raise ValueError(f"linear_batched: residual must be {tuple(out.shape)}, got {tuple(residual.shape)}")
    if a.stride(-1) != 1 or out.stride(-1) != 1 or (residual is not None and residual.stride(-1) != 1):
        raise ValueError("linear_batched: a, out and residual need a contiguous last dimension")
    mod = row_add if row_add is not None else row_gate
    if mod is not None:
        _check_mod_views("linear_batched", row_add=row_add, row_gate=row_gate)
        _check_mod_groups("linear_batched", B * rows, rows, n_out, row_add=row_add, row_gate=row_gate)
    e = make_epilogue(bias=bias, row_add=row_add, row_gate=row_gate, ld_row=0 if mod is None else mod.stride(0),
                      rows_per_group=rows, residual=residual, ldr=0 if residual is None else residual.stride(1),
                      act=act, glu=glu, out_fp32=(out.dtype == torch.float32))
    with _Timed("igemm", 2.0 * B * rows * N * K, "flop", lambda: f"linb {B}*{rows}x{N}x{K}" + _epi_tag(e)):
        check(lib.b200mix_linear_batched(_p(a), a.stride(1), a.stride(0), _p(w), w.stride(0), _p(out), out.stride(1),
                                         out.stride(0), rows, B, N, K, ctypes.byref(e),
                                         0 if residual is None else residual.stride(0), _stream()),
              "b200mix_linear_batched")
    _count()
    return out


def patchify(x: torch.Tensor, p: int) -> torch.Tensor:
    B, C, H, W = x.shape
    assert x.is_contiguous() and x.dtype in (torch.float32, bf16)
    out = torch.empty(B, (H // p) * (W // p), C * p * p, device=x.device, dtype=bf16)
    check(lib.b200mix_patchify(_p(x), 1 if x.dtype == torch.float32 else 0, _p(out), B, C, H, W, p, _stream()),
          "b200mix_patchify")
    _count()
    return out


def unpatchify(x: torch.Tensor, C: int, h: int, w: int, p: int, out_dtype=bf16) -> torch.Tensor:
    B = x.shape[0]
    assert x.is_contiguous() and x.dtype == bf16
    out = torch.empty(B, C, h * p, w * p, device=x.device, dtype=out_dtype)
    check(lib.b200mix_unpatchify(_p(x), _p(out), 1 if out_dtype == torch.float32 else 0, B, C, h, w, p, _stream()),
          "b200mix_unpatchify")
    _count()
    return out


def conv3x3(x: torch.Tensor, w: torch.Tensor, bias=None, *, stride=1, row_add=None, residual=None, act=ACT_NONE,
            out_scale=1.0, out=None) -> torch.Tensor:
    """x: bf16 NHWC [B,H,W,Cin] contiguous; w: bf16 [Cout,3,3,Cin] contiguous; returns bf16 NHWC."""
    _req(x, bf16, "x"), _req(w, bf16, "w")
    B, H, W, Cin = x.shape
    Cout = w.shape[0]
    assert x.is_contiguous() and w.is_contiguous()
    Ho, Wo = H // stride, W // stride
    if out is None:
        out = torch.empty(B, Ho, Wo, Cout, device=x.device, dtype=bf16)
    if row_add is not None:
        _check_mod_views("conv3x3", row_add=row_add)
    e = make_epilogue(bias=bias, row_add=row_add, ld_row=0 if row_add is None else row_add.stride(0),
                      rows_per_group=Ho * Wo, residual=residual, ldr=Cout, act=act, out_scale=out_scale)
    with _Timed("igemm", 2.0 * B * Ho * Wo * Cout * 9 * Cin, "flop",
                lambda: f"conv{stride} {B * Ho * Wo}x{Cout}x{9 * Cin}" + _epi_tag(e)):
        check(lib.b200mix_conv3x3(_p(x), _p(w), _p(out), B, H, W, Cin, Cout, stride, ctypes.byref(e), _stream()),
              "b200mix_conv3x3")
    _count()
    return out


def fold_upsample_conv_weight(w: torch.Tensor) -> torch.Tensor:
    """w: [Cout, 3, 3, Cin] (any float dtype; fold from the fp32 master weights when they exist) -> bf16 [Cout, 16, Cin],
    the per-output-parity 2x2 filters of nearest-2x-upsample + conv3x3 (b200mix_conv3x3_up2x). Row index =
    (py*2 + px)*4 + a*2 + b; taps that read the same low-resolution pixel are summed in fp32 and rounded once."""
    O, _, _, I = w.shape
    wf = w.float()
    groups = {0: ((0,), (1, 2)), 1: ((0, 1), (2,))}  # parity -> (taps folded into a = 0, taps folded into a = 1)
    out = torch.empty(O, 2, 2, 2, 2, I, dtype=torch.float32, device=w.device)
    for py in range(2):
        for px in range(2):
            for a in range(2):
                for b in range(2):
                    out[:, py, px, a, b] = sum(wf[:, ky, kx] for ky in groups[py][a] for kx in groups[px][b])
    return out.reshape(O, 16, I).to(bf16).contiguous()


def conv3x3_up2x(x: torch.Tensor, w4: torch.Tensor, bias=None, *, row_add=None, residual=None, act=ACT_NONE,
                 out_scale=1.0, out=None) -> torch.Tensor:
    """conv3x3(nearest_upsample_2x(x)) from the low-resolution x: bf16 NHWC [B,H,W,Cin]; w4 = fold_upsample_conv_weight(w).
    Returns bf16 NHWC [B,2H,2W,Cout] (Upsample2D, resnet.py:169-218)."""
    _req(x, bf16, "x"), _req(w4, bf16, "w4")
    B, H, W, Cin = x.shape
    Cout = w4.shape[0]
    assert x.is_contiguous() and w4.is_contiguous() and tuple(w4.shape[1:]) == (16, Cin)
    if out is None:
        out = torch.empty(B, 2 * H, 2 * W, Cout, device=x.device, dtype=bf16)
    if row_add is not None:
        _check_mod_views("conv3x3_up2x", row_add=row_add)
    e = make_epilogue(bias=bias, row_add=row_add, ld_row=0 if row_add is None else row_add.stride(0),
                      rows_per_group=4 * H * W, residual=residual, ldr=Cout, act=act, out_scale=out_scale)
    with _Timed("igemm", 2.0 * B * 4 * H * W * Cout * 4 * Cin, "flop",
                lambda: f"convup {B * 4 * H * W}x{Cout}x{4 * Cin}" + _epi_tag(e)):
        check(lib.b200mix_conv3x3_up2x(_p(x), _p(w4), _p(out), B, H, W, Cin, Cout, ctypes.byref(e), _stream()),
              "b200mix_conv3x3_up2x")
    _count()
    return out


def conv3x3_small_cin(x: torch.Tensor, w: torch.Tensor, bias=None) -> torch.Tensor:
    B, H, W, Cin = x.shape
    Cout = w.shape[0]
    assert x.is_contiguous() and w.is_contiguous() and x.dtype in (torch.float32, bf16)
    out = torch.empty(B, H, W, Cout, device=x.device, dtype=bf16)
    check(lib.b200mix_conv3x3_small_cin(_p(x), 1 if x.dtype == torch.float32 else 0, _p(w), _p(bias), _p(out), B, H, W,
                                        Cin, Cout, _stream()), "b200mix_conv3x3_small_cin")
    _count()
    return out


def conv3x3_narrow(x: torch.Tensor, w: torch.Tensor, bias=None, *, stride=1, act=ACT_NONE, out=None) -> torch.Tensor:
    """act(conv3x3(x) + bias) for 1 <= Cin <= 128 (the ControlNet conditioning embedding). x: bf16 NHWC [B,H,W,Cin]
    contiguous; w: bf16 [Cout,3,3,Cin] contiguous; bias fp32 [Cout] or None; act ACT_NONE | ACT_SILU. Returns bf16 NHWC
    [B,H/stride,W/stride,Cout]."""
    _req(x, bf16, "x"), _req(w, bf16, "w")
    B, H, W, Cin = x.shape
    Cout = w.shape[0]
    assert x.is_contiguous() and w.is_contiguous() and tuple(w.shape[1:]) == (3, 3, Cin)
    if out is None:
        out = torch.empty(B, H // stride, W // stride, Cout, device=x.device, dtype=bf16)
    with _Timed("conv_narrow", 2.0 * B * (H // stride) * (W // stride) * Cout * 9 * Cin, "flop",
                lambda: f"convn{stride} {B}x{H}x{W}x{Cin}->{Cout}"):
        check(lib.b200mix_conv3x3_narrow(_p(x), _p(w), _p(None if bias is None else _req(bias, torch.float32, "bias")),
                                         _p(out), B, H, W, Cin, Cout, int(stride), int(act), _stream()),
              "b200mix_conv3x3_narrow")
    _count()
    return out


def sdpa(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, *, scale: Optional[float] = None, causal=False,
         cu_seqlens: Optional[torch.Tensor] = None, kv_lens: Optional[torch.Tensor] = None,
         attn_mask: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """q: [B,Sq,Hq,D], k/v: [B,Sk,Hkv,D] bf16 views (head_dim contiguous; other strides arbitrary multiples of 8).
    attn_mask: additive bias (bf16 / fp32) broadcastable to [B,Hq,Sq,Sk] with a contiguous key axis (the reference's
    `attn_mask` argument, paddle_patch.py:418). Returns [B,Sq,Hq,D] (the layout of scaled_dot_product_attention_)."""
    _req(q, bf16, "q"), _req(k, bf16, "k"), _req(v, bf16, "v")
    B, Sq, Hq, D = q.shape
    _, Sk, Hkv, _ = k.shape
    assert q.stride(-1) == 1 and k.stride(-1) == 1 and v.stride(-1) == 1
    if out is None:
        out = torch.empty(B, Sq, Hq, D, device=q.device, dtype=bf16)
    if scale is None:
        scale = D ** -0.5
    nseq = 0 if cu_seqlens is None else cu_seqlens.numel() - 1
    m_fp32, msb, msh, msq = 0, 0, 0, 0
    if attn_mask is not None:
        if attn_mask.dtype not in (torch.float32, bf16):
            raise TypeError(f"attn_mask must be an additive float32 / bfloat16 bias, got {attn_mask.dtype}")
        while attn_mask.dim() < 4:
            attn_mask = attn_mask.unsqueeze(0)
        if attn_mask.shape[-1] != Sk or any(a not in (1, n) for a, n in zip(attn_mask.shape[:3], (B, Hq, Sq))):
            raise ValueError(f"attn_mask shape {tuple(attn_mask.shape)} does not broadcast to {(B, Hq, Sq, Sk)}")
        if attn_mask.stride(-1) != 1 and Sk > 1:
            attn_mask = attn_mask.contiguous()
        attn_mask = _req(attn_mask, attn_mask.dtype, "attn_mask")
        m_fp32 = 1 if attn_mask.dtype == torch.float32 else 0
        msb, msh, msq = (0 if attn_mask.shape[i] == 1 else attn_mask.stride(i) for i in range(3))
    with _Timed("attention", 4.0 * B * Hq * Sq * Sk * D * (0.5 if causal else 1.0), "flop",
                lambda: f"attn B{B} H{Hq} Sq{Sq} Sk{Sk} D{D}" + (" causal" if causal else "")):
        check(lib.b200mix_sdpa(_p(q), _p(k), _p(v), _p(out), B, Hq, Hkv, Sq, Sk, D, q.stride(0), q.stride(1),
                               q.stride(2), k.stride(0), k.stride(1), k.stride(2), v.stride(0), v.stride(1),
                               v.stride(2), out.stride(0), out.stride(1), out.stride(2), float(scale),
                               1 if causal else 0, _p(cu_seqlens), nseq, _p(kv_lens), _p(attn_mask), m_fp32, msb, msh,
                               msq, _stream()), "b200mix_sdpa")
    _count()
    return out


_gn_scratch = {}


def groupnorm_nhwc(x1: torch.Tensor, gamma, beta, *, x2=None, groups=32, eps=1e-5, silu=False, out=None):
    """x1: bf16 [B,H,W,C1] (optionally concatenated on channels with x2 [B,H,W,C2]); returns bf16 [B,H,W,C1+C2]."""
    _req(x1, bf16, "x1")
    B, C1 = x1.shape[0], x1.shape[-1]
    HW = x1.numel() // (B * C1)
    C2 = 0 if x2 is None else x2.shape[-1]
    assert x1.is_contiguous() and (x2 is None or x2.is_contiguous())
    if out is None:
        out = torch.empty(*x1.shape[:-1], C1 + C2, device=x1.device, dtype=bf16)
    # per-(device, stream, B, groups) scratch: two streams never share partial sums, and the size is exact for the key
    key = (x1.device, torch.cuda.current_stream().cuda_stream, B, groups)
    st = _gn_scratch.get(key)
    if st is None:
        # zero-filled once: the first 4 KB hold the per-batch arrival counters, which every call leaves at zero
        st = torch.zeros(512 + (1024 + 2 * B) * groups * 2, device=x1.device, dtype=torch.float64)
        _gn_scratch[key] = st
    with _Timed("groupnorm", 2.0 * 2 * B * HW * (C1 + C2), "byte", lambda: f"gn {B}x{HW}x{C1 + C2}"):  # algorithmic: read once + write once (bf16)
        check(lib.b200mix_groupnorm_nhwc(_p(x1), C1, _p(x2), C2, _p(gamma), _p(beta), _p(out), _p(st), st.numel() * 8, B,
                                         HW, groups, float(eps), 1 if silu else 0, _stream()), "b200mix_groupnorm_nhwc")
    _count(2)
    return out


def layernorm(x: torch.Tensor, weight=None, bias=None, *, eps=1e-5, rms=False, delta=None, gate=None, scale=None,
              shift=None, rows_per_group=0, want_resid=False, out=None):
    """Row-wise (RMS/Layer)Norm with optional fused residual update x + gate*delta and AdaLN modulation.
    Returns y, or (resid, y) when want_resid."""
    _req(x, bf16, "x")
    N = x.shape[-1]
    x2 = x.reshape(-1, N)
    assert x2.is_contiguous()
    M = x2.shape[0]
    if out is None:
        out = torch.empty_like(x)
    resid = torch.empty_like(x) if (want_resid and delta is not None) else None
    mod = gate if gate is not None else (scale if scale is not None else shift)
    if mod is not None:
        _check_mod_views("layernorm", gate=gate, scale=scale, shift=shift)
        _check_mod_groups("layernorm", M, rows_per_group, N, gate=gate, scale=scale, shift=shift)
    ld_mod = 0 if mod is None else mod.stride(0)
    nbytes = 2.0 * M * N * (2 + (1 if delta is not None else 0) + (1 if resid is not None else 0))
    with _Timed("layernorm", nbytes, "byte", lambda: f"ln {M}x{N}" + (" +delta" if delta is not None else "")):
        check(lib.b200mix_layernorm(_p(x2), _p(delta), _p(gate), _p(resid), _p(out), _p(weight), _p(bias), _p(scale),
                                    _p(shift), ld_mod, rows_per_group, M, N, float(eps), 1 if rms else 0, _stream()),
              "b200mix_layernorm")
    _count()
    if want_resid:
        return (resid if resid is not None else x), out
    return out


def softmax_rows(x: torch.Tensor, scale: float = 1.0, out=None) -> torch.Tensor:
    """x: fp32 [M, N] (row stride arbitrary multiple of 4) -> bf16 softmax(x * scale) [M, N]."""
    _req(x, torch.float32, "x")
    M, N = x.shape
    assert x.stride(1) == 1
    if out is None:
        out = torch.empty(M, N, device=x.device, dtype=bf16)
    with _Timed("softmax", 4.0 * M * N + 2.0 * M * N, "byte", lambda: f"softmax {M}x{N}"):
        check(lib.b200mix_softmax_rows(_p(x), _p(out), M, N, x.stride(0), out.stride(0), float(scale), _stream()),
              "b200mix_softmax_rows")
    _count()
    return out


def timestep_embedding(t: torch.Tensor, dim: int, *, flip_sin_to_cos=True, downscale_freq_shift=0.0, scale=1.0,
                       max_period=10000.0, out=None, col0=0, out_dtype=bf16):
    _req(t, torch.float32, "t")
    B = t.numel()
    if out is None:
        out = torch.empty(B, dim, device=t.device, dtype=out_dtype)
    check(lib.b200mix_timestep_embedding(_p(t), _p(out), 1 if out.dtype == torch.float32 else 0, B, dim, out.stride(0),
                                         col0, 1 if flip_sin_to_cos else 0, float(downscale_freq_shift), float(scale),
                                         float(max_period), _stream()), "b200mix_timestep_embedding")
    _count()
    return out


def activation(x: torch.Tensor, act: int, out_dtype=None):
    assert x.is_contiguous() and x.dtype in (torch.float32, bf16)
    out = torch.empty_like(x, dtype=out_dtype or x.dtype)
    check(lib.b200mix_activation(_p(x), _p(out), x.numel(), act, 1 if x.dtype == torch.float32 else 0,
                                 1 if out.dtype == torch.float32 else 0, _stream()), "b200mix_activation")
    _count()
    return out


def upsample_nearest2x(x: torch.Tensor):
    _req(x, bf16, "x")
    B, H, W, C = x.shape
    out = torch.empty(B, 2 * H, 2 * W, C, device=x.device, dtype=bf16)
    check(lib.b200mix_upsample_nearest2x_nhwc(_p(x), _p(out), B, H, W, C, _stream()), "b200mix_upsample")
    _count()
    return out


def concat_channels(x1: torch.Tensor, x2: torch.Tensor):
    C1, C2 = x1.shape[-1], x2.shape[-1]
    rows = x1.numel() // C1
    out = torch.empty(*x1.shape[:-1], C1 + C2, device=x1.device, dtype=bf16)
    check(lib.b200mix_concat_channels(_p(x1), C1, _p(x2), C2, _p(out), rows, _stream()), "b200mix_concat_channels")
    _count()
    return out


def nchw_to_nhwc(x: torch.Tensor):
    B, C, H, W = x.shape
    assert x.is_contiguous() and x.dtype in (torch.float32, bf16)
    out = torch.empty(B, H, W, C, device=x.device, dtype=bf16)
    check(lib.b200mix_nchw_to_nhwc(_p(x), 1 if x.dtype == torch.float32 else 0, _p(out), B, C, H, W, _stream()),
          "b200mix_nchw_to_nhwc")
    _count()
    return out


def nhwc_to_nchw(x: torch.Tensor, out_dtype=torch.float32, out=None):
    B, H, W, C = x.shape
    _req(x, bf16, "x")
    if out is None:
        out = torch.empty(B, C, H, W, device=x.device, dtype=out_dtype)
    check(lib.b200mix_nhwc_to_nchw(_p(x), _p(out), 1 if out.dtype == torch.float32 else 0, B, C, H, W, _stream()),
          "b200mix_nhwc_to_nchw")
    _count()
    return out


def add_residual_nhwc(a: torch.Tensor, r: torch.Tensor, *, r_nchw: bool, out=None) -> torch.Tensor:
    """a: bf16 NHWC [B,H,W,C]; r: the same values as NHWC bf16, or NCHW fp32 / bf16 [B,C,H,W] (r_nchw). Returns a + r."""
    _req(a, bf16, "a")
    B, H, W, C = a.shape
    want = (B, C, H, W) if r_nchw else (B, H, W, C)
    if tuple(r.shape) != want:
        raise ValueError(f"residual shape {tuple(r.shape)} does not match the activation {want}")
    if r.dtype not in (torch.float32, bf16):
        r = r.float()
    r = r.to(a.device).contiguous()
    assert a.is_contiguous()
    if out is None:
        out = torch.empty_like(a)
    check(lib.b200mix_add_residual_nhwc(_p(a), _p(r), 1 if r.dtype == torch.float32 else 0, 1 if r_nchw else 0, _p(out),
                                        B, C, H, W, _stream()), "b200mix_add_residual_nhwc")
    _count()
    return out


def _step_tensors(op, x, m_u, m_c, out, **fp32_bufs):
    """Checks the tensors of a sampler step before anything is launched; returns (m_u's dtype flag, out), allocating out
    like x (like m_u when x is None) if it is None. The kernels read every tensor flat over x's element count (m_u's
    when x is None) and m_c with m_u's dtype flag, so each given tensor must be contiguous, have that many elements and
    the dtype below: x, out and fp32_bufs fp32, m_u fp32 or bf16, m_c m_u's dtype."""
    f32 = (torch.float32,)
    want = {"x": (x, f32), "model output": (m_u, (torch.float32, bf16)), "model_output_cond": (m_c, (m_u.dtype,)),
            "out": (out, f32), **{k: (t, f32) for k, t in fp32_bufs.items()}}
    given = {k: v for k, v in want.items() if v[0] is not None}
    n = (m_u if x is None else x).numel()
    for name, (t, dtypes) in given.items():
        if t.dtype not in dtypes:
            raise TypeError(f"{op}: {name} must be {' or '.join(map(str, dtypes))}, got {t.dtype}")
        if t.numel() != n:
            raise ValueError(f"{op}: {name} has {t.numel()} elements, expected {n}")
        if not t.is_contiguous():
            raise ValueError(f"{op}: {name} must be contiguous, got strides {t.stride()} for shape {tuple(t.shape)}")
    for name, (t, _) in given.items():
        if not t.is_cuda:
            raise _lib.B200MixError(f"{op}: {name} must be a CUDA tensor (b200mix has no CPU path)")
    if out is None:
        like = m_u if x is None else x
        out = torch.empty(like.shape, device=like.device, dtype=torch.float32)
    return (1 if m_u.dtype == torch.float32 else 0), out


PRED_TYPES = {"epsilon": 0, "sample": 1, "v_prediction": 2}


def ddim_step(m_u, m_c, guidance, x, sa_t, sb_t, sa_p, sb_p, prediction_type="epsilon", clip_sample_range=0.0, out=None):
    """DDIM step for any prediction_type, optional x0 clipping (clip_sample_range > 0), fused CFG combine."""
    fp32, out = _step_tensors("ddim_step", x, m_u, m_c, out)
    check(lib.b200mix_ddim_step_ex(_p(m_u), _p(m_c), fp32, float(guidance), _p(x), _p(out), x.numel(), float(sa_t),
                                   float(sb_t), float(sa_p), float(sb_p), PRED_TYPES[prediction_type],
                                   float(clip_sample_range), _stream()), "b200mix_ddim_step_ex")
    _count()
    return out


def lcm_step(m_u, m_c, guidance, x, noise, sa_t, sb_t, c_skip, c_out, sa_p, sb_p, prediction_type="epsilon",
             clip_sample_range=0.0, out=None, denoised=None):
    """LCMScheduler.step; noise None = final step (x_prev = denoised)."""
    fp32, out = _step_tensors("lcm_step", x, m_u, m_c, out, noise=noise, denoised=denoised)
    check(lib.b200mix_lcm_step(_p(m_u), _p(m_c), fp32, float(guidance), _p(x), _p(noise), _p(out), _p(denoised),
                               x.numel(), float(sa_t), float(sb_t), float(c_skip), float(c_out), float(sa_p), float(sb_p),
                               PRED_TYPES[prediction_type], float(clip_sample_range), _stream()), "b200mix_lcm_step")
    _count()
    return out


def iddpm_step(model_out, x, cfg_scale, cfg_channel, scalars, add_noise, seed=0, step=0, noise=None, out=None, out_dup=None):
    """Open-Sora IDDPM p_sample behind forward_with_cfg (b200mix_iddpm_step). model_out [2B, 2C, ...] fp32 | bf16 with
    the conditional rows first; x fp32 [B, C, ...]; scalars = (sqrt_recip_ac, sqrt_recipm1_ac, coef1, coef2, max_log,
    min_log) as fp32 values; noise fp32 like x, or None for Philox noise keyed by (seed, step). out may be x itself;
    out_dup receives a second copy of the result. Returns out."""
    _req(x, torch.float32, "x")
    B, C = x.shape[:2]
    if model_out.dtype not in (torch.float32, bf16) or not model_out.is_contiguous():
        raise ValueError("model_out must be contiguous fp32 or bf16")
    if tuple(model_out.shape) != (2 * B, 2 * C, *x.shape[2:]):
        raise ValueError(f"model_out {tuple(model_out.shape)} must be [2B, 2C, ...] for x {tuple(x.shape)}")
    if noise is not None:
        _req(noise, torch.float32, "noise")
        assert noise.shape == x.shape
    if out is None:
        out = torch.empty_like(x)
    for t in (out, out_dup):
        if t is not None:
            _req(t, torch.float32, "out")
            assert t.shape == x.shape
    if not all(t is None or t.is_contiguous() for t in (x, noise, out, out_dup)):
        raise ValueError("iddpm_step: x, noise and the outputs must be contiguous")
    check(lib.b200mix_iddpm_step(_p(model_out), 1 if model_out.dtype == torch.float32 else 0, _p(x), _p(noise), _p(out),
                                 _p(out_dup), B, C, x.numel() // (B * C), float(cfg_scale), int(cfg_channel),
                                 *(float(v) for v in scalars), 1 if add_noise else 0, int(seed), int(step), _stream()),
          "b200mix_iddpm_step")
    _count()
    return out


def cfg_combine(eps_u, eps_c, guidance, guidance_rescale=0.0, out=None):
    """noise_pred_uncond + g * (noise_pred_text - noise_pred_uncond), then rescale_noise_cfg when guidance_rescale > 0
    (pipeline_stable_diffusion.py:69-80, :882-888). eps_*: [B, ...] bf16 / fp32 contiguous. Returns fp32."""
    fp32, out = _step_tensors("cfg_combine", None, eps_u, eps_c, out)
    if eps_c is None or eps_c.shape != eps_u.shape:
        raise ValueError(f"cfg_combine: eps_c must have eps_u's shape {tuple(eps_u.shape)}: samples are along dim 0")
    B = eps_u.shape[0]
    nps = eps_u.numel() // B
    ratio = None
    if guidance_rescale > 0.0:
        ratio = torch.empty(B, device=eps_u.device, dtype=torch.float32)
        check(lib.b200mix_cfg_rescale_ratio(_p(eps_u), _p(eps_c), fp32, float(guidance), _p(ratio), B, nps, _stream()),
              "b200mix_cfg_rescale_ratio")
        _count()
    check(lib.b200mix_cfg_combine(_p(eps_u), _p(eps_c), fp32, float(guidance), _p(ratio), float(guidance_rescale), nps,
                                  _p(out), eps_u.numel(), _stream()), "b200mix_cfg_combine")
    _count()
    return out


def euler_step(v_u, v_c, guidance, x, sigma, dt, out=None):
    fp32, out = _step_tensors("euler_step", x, v_u, v_c, out)
    check(lib.b200mix_euler_step(_p(v_u), _p(v_c), fp32, float(guidance), _p(x), _p(out), x.numel(), float(sigma),
                                 float(dt), _stream()), "b200mix_euler_step")
    _count()
    return out


def dpmpp_2m_step(eps_u, eps_c, guidance, x, m_prev, m_out, sigma_cur, alpha_cur, A, C, halfC, inv_r0, out=None):
    """DPM-Solver++ 2M update (see include/b200mix.h); m_prev None = first-order step; m_out receives x0."""
    fp32, out = _step_tensors("dpmpp_2m_step", x, eps_u, eps_c, out, m_prev=m_prev, m_out=m_out)
    check(lib.b200mix_dpmpp_2m_step(_p(eps_u), _p(eps_c), fp32, float(guidance), _p(x), _p(m_prev), _p(out), _p(m_out),
                                    x.numel(), float(sigma_cur), float(alpha_cur), float(A), float(C), float(halfC),
                                    float(inv_r0), _stream()), "b200mix_dpmpp_2m_step")
    _count()
    return out


def scale_model_input(x: torch.Tensor, denom: float, out=None) -> torch.Tensor:
    """EulerDiscreteScheduler.scale_model_input: x / denom in fp32 (IEEE division)."""
    _req(x, torch.float32, "x")
    assert x.is_contiguous()
    if out is None:
        out = torch.empty_like(x)
    check(lib.b200mix_scale_model_input(_p(x), _p(out), x.numel(), float(denom), _stream()), "b200mix_scale_model_input")
    _count()
    return out


def cast(x: torch.Tensor, dtype):
    assert x.is_contiguous()
    out = torch.empty_like(x, dtype=dtype)
    check(lib.b200mix_cast(_p(x), _p(out), x.numel(), 1 if x.dtype == torch.float32 else 0,
                           1 if dtype == torch.float32 else 0, _stream()), "b200mix_cast")
    _count()
    return out


def rope_inplace(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, rot_dim: Optional[int] = None):
    """x: bf16 [T, H, Dpad] view (last dim contiguous); cos/sin fp32 [T, rot_dim]."""
    T, H, Dp = x.shape
    D = rot_dim or Dp
    check(lib.b200mix_rope_inplace(_p(x), T, H, D, x.stride(0), x.stride(1), _p(cos), _p(sin), _stream()),
          "b200mix_rope_inplace")
    _count()
    return x


def decode_rope_cache(qkv: torch.Tensor, heads: int, kv_heads: int, head_dim: int, cos: torch.Tensor, sin: torch.Tensor,
                      rows: torch.Tensor, cache_k: torch.Tensor, cache_v: torch.Tensor):
    """qkv bf16 [B, (heads + 2*kv_heads) * head_dim] of a single-token step: RoPE on the q heads in place, RoPE'd k heads and
    the v heads written into row rows[b] (int64, device) of the flattened caches [*, kv_heads * head_dim]."""
    _req(qkv, bf16, "qkv"), _req(rows, torch.int64, "rows"), _req(cache_k, bf16, "cache_k"), _req(cache_v, bf16, "cache_v")
    assert qkv.stride(1) == 1 and qkv.shape[1] == (heads + 2 * kv_heads) * head_dim
    assert cache_k.is_contiguous() and cache_v.is_contiguous() and cos.is_contiguous() and sin.is_contiguous()
    check(lib.b200mix_decode_rope_cache(_p(qkv), qkv.stride(0), qkv.shape[0], heads, kv_heads, head_dim, _p(cos), _p(sin),
                                        _p(rows), _p(cache_k), _p(cache_v), _stream()), "b200mix_decode_rope_cache")
    _count()


def sample_tokens(logits: torch.Tensor, presence: torch.Tensor, finished: torch.Tensor, state: torch.Tensor,
                  out: torch.Tensor, next_ids: torch.Tensor, eos_ids: Optional[torch.Tensor] = None, pad_token_id=0, *,
                  do_sample=False, temperature=1.0, top_k=0, top_p=1.0, repetition_penalty=1.0, seed=0):
    """One generation step (b200mix_sample_tokens, see include/b200mix.h): logits fp32 [B, V] view with a contiguous
    vocabulary axis (any row stride: logits[:, -1] of prefill logits [B, S, V] is read in place); presence int32
    [B, ceil(V/32)] bitmap of the ids seen so far; finished int32 [B]; state int64 [4] (step, arrivals, all finished,
    step of the last finish; zero before the first step); out int64 [B, max_new]; next_ids int64 [B]; eos_ids int64
    [n] on the device or None. Every buffer except logits is updated on the device."""
    _req(logits, torch.float32, "logits"), _req(presence, torch.int32, "presence"), _req(finished, torch.int32, "finished")
    _req(state, torch.int64, "state"), _req(out, torch.int64, "out"), _req(next_ids, torch.int64, "next_ids")
    B, V = logits.shape
    if logits.stride(1) != 1 and V > 1:
        raise ValueError("logits must have a contiguous vocabulary axis")
    words = (V + 31) // 32
    if tuple(presence.shape) != (B, words) or not presence.is_contiguous():
        raise ValueError(f"presence must be a contiguous int32 [{B}, {words}] bitmap, got {tuple(presence.shape)}")
    if finished.numel() != B or next_ids.numel() != B or state.numel() != 4 or out.shape[0] != B or out.stride(1) != 1:
        raise ValueError("finished / next_ids must have B entries, state 4, out [B, max_new] with contiguous rows")
    n_eos = 0
    if eos_ids is not None:
        _req(eos_ids, torch.int64, "eos_ids")
        n_eos = eos_ids.numel()
    with _Timed("sampling", 4.0 * B * V, "byte", lambda: f"sample {B}x{V}"):
        check(lib.b200mix_sample_tokens(_p(logits), logits.stride(0), B, V, _p(presence), _p(finished), _p(state),
                                        _p(out), out.stride(0), out.shape[1], _p(next_ids), _p(eos_ids), n_eos,
                                        int(pad_token_id), 1 if do_sample else 0, float(temperature), int(top_k),
                                        float(top_p), float(repetition_penalty), int(seed) & (2 ** 64 - 1), _stream()),
              "b200mix_sample_tokens")
    _count()


def beam_search_workspace_bytes(B: int, num_beams: int, V: int) -> int:
    n = ctypes.c_int64(0)
    check(lib.b200mix_beam_search_workspace_size(B, num_beams, V, ctypes.byref(n)), "b200mix_beam_search_workspace_size")
    return n.value


def beam_search_step(logits: torch.Tensor, num_beams: int, workspace: torch.Tensor, *, state, next_ids, beam_scores,
                     tokens, parents, hyp_score, hyp_step, hyp_slot, hyp_count, hyp_worst, done, presence=None,
                     eos_token_id=-1, pad_token_id=0, repetition_penalty=1.0, diversity_rate=0.0, length_penalty=1.0,
                     early_stopping=False):
    """One beam-search step (b200mix_beam_search_step, see include/b200mix.h): logits fp32 [B * nb, V] view with a
    contiguous vocabulary axis (any row stride); state int64 [4]; next_ids int64 [B*nb]; beam_scores fp32 [B*nb]; tokens
    int64 / parents int32 [max_new, B*nb]; hyp_score fp64 / hyp_step, hyp_slot int32 [B, nb]; hyp_count int32 [B];
    hyp_worst fp64 [B]; done int32 [B]; presence int32 [2, B*nb, ceil(V/32)] or None (penalty 1); workspace uint8 of
    beam_search_workspace_bytes(B, nb, V). Everything but logits is updated on the device; eos_token_id -1 = none."""
    _req(logits, torch.float32, "logits")
    rows, V = logits.shape
    nb = int(num_beams)
    if logits.stride(1) != 1 or rows % nb:
        raise ValueError(f"logits must be [B * {nb}, V] with a contiguous vocabulary axis, got {tuple(logits.shape)}")
    B = rows // nb
    for t, dt, n, name in ((state, torch.int64, 4, "state"), (next_ids, torch.int64, rows, "next_ids"),
                           (beam_scores, torch.float32, rows, "beam_scores"), (hyp_score, torch.float64, B * nb, "hyp_score"),
                           (hyp_step, torch.int32, B * nb, "hyp_step"), (hyp_slot, torch.int32, B * nb, "hyp_slot"),
                           (hyp_count, torch.int32, B, "hyp_count"), (hyp_worst, torch.float64, B, "hyp_worst"),
                           (done, torch.int32, B, "done")):
        _req(t, dt, name)
        if t.numel() != n or not t.is_contiguous():
            raise ValueError(f"{name} must be a contiguous tensor of {n} elements, got {tuple(t.shape)}")
    _req(tokens, torch.int64, "tokens"), _req(parents, torch.int32, "parents"), _req(workspace, torch.uint8, "workspace")
    max_new = tokens.shape[0]
    if tuple(tokens.shape) != (max_new, rows) or tuple(parents.shape) != (max_new, rows) or not (
            tokens.is_contiguous() and parents.is_contiguous()):
        raise ValueError(f"tokens / parents must be contiguous [max_new, {rows}]")
    if presence is not None:
        _req(presence, torch.int32, "presence")
        if tuple(presence.shape) != (2, rows, (V + 31) // 32) or not presence.is_contiguous():
            raise ValueError(f"presence must be a contiguous int32 [2, {rows}, {(V + 31) // 32}] bitmap pair")
    st = _lib.BeamState(*(t.data_ptr() for t in (state, next_ids, beam_scores, tokens, parents, hyp_score, hyp_step,
                                                 hyp_slot, hyp_count, hyp_worst, done)),
                        None if presence is None else presence.data_ptr())
    with _Timed("beam_search", 4.0 * rows * V, "byte", lambda: f"beam {B}x{nb}x{V}"):
        check(lib.b200mix_beam_search_step(_p(logits), logits.stride(0), B, nb, V, ctypes.byref(st), _p(workspace),
                                           workspace.numel(), max_new, int(eos_token_id), int(pad_token_id),
                                           float(repetition_penalty), float(diversity_rate), float(length_penalty),
                                           1 if early_stopping else 0, _stream()), "b200mix_beam_search_step")
    _count(3)


def kv_reorder(layer_kv: torch.Tensor, cache_k, num_beams: int, prompt_len: int, parents: torch.Tensor,
               state: torch.Tensor, done: torch.Tensor):
    """b200mix_kv_reorder: layer_kv int64 [2 * L] device table of the K / V base pointers (K_0, V_0, K_1, ...) of caches
    shaped like cache_k (bf16 [B * nb, max_len, kv_heads, head_dim], contiguous); moves the generated positions
    [prompt_len, prompt_len + state[3]) from parent beam to child (parents int32 [max_new, B * nb], column state[0] - 1)
    for every item whose done flag is 0."""
    _req(layer_kv, torch.int64, "layer_kv"), _req(cache_k, bf16, "cache_k"), _req(parents, torch.int32, "parents")
    _req(state, torch.int64, "state"), _req(done, torch.int32, "done")
    rows, max_len = cache_k.shape[:2]
    nb = int(num_beams)
    if rows % nb or not cache_k.is_contiguous() or layer_kv.numel() % 2 or parents.shape[1] != rows:
        raise ValueError("kv_reorder: cache / parents shapes do not match num_beams")
    check(lib.b200mix_kv_reorder(_p(layer_kv), layer_kv.numel() // 2, rows // nb, nb, max_len,
                                 cache_k[0, 0].numel(), int(prompt_len), parents.shape[0], _p(parents), _p(state),
                                 _p(done), _stream()), "b200mix_kv_reorder")
    _count()


def gather_rows(table: torch.Tensor, ids: torch.Tensor) -> torch.Tensor:
    """table bf16 [V, D], ids int64 [n] (device) -> bf16 [n, D]."""
    _req(table, bf16, "table"), _req(ids, torch.int64, "ids")
    n, D = ids.numel(), table.shape[1]
    out = torch.empty(n, D, device=table.device, dtype=bf16)
    check(lib.b200mix_gather_rows(_p(table), _p(ids), _p(out), n, D, _stream()), "b200mix_gather_rows")
    _count()
    return out


def scatter_rows(src: torch.Tensor, idx: torch.Tensor, dst: torch.Tensor) -> torch.Tensor:
    """dst[idx[i]] = src[i]; src bf16 [n, D], idx int64 [n] (device), dst bf16 [*, D] (in place)."""
    _req(src, bf16, "src"), _req(idx, torch.int64, "idx"), _req(dst, bf16, "dst")
    check(lib.b200mix_scatter_rows(_p(src), _p(idx), _p(dst), idx.numel(), src.shape[-1], _stream()),
          "b200mix_scatter_rows")
    _count()
    return dst


def broadcast_add(x: torch.Tensor, table: torch.Tensor) -> torch.Tensor:
    """x fp32 [B, N], table fp32 [G, N] -> fp32 [B, G, N]."""
    _req(x, torch.float32, "x"), _req(table, torch.float32, "table")
    B, N = x.shape
    G = table.shape[0]
    out = torch.empty(B, G, N, device=x.device, dtype=torch.float32)
    check(lib.b200mix_broadcast_add(_p(x), _p(table), _p(out), B, G, N, _stream()), "b200mix_broadcast_add")
    _count()
    return out


def head_rmsnorm_inplace(x: torch.Tensor, weight: torch.Tensor, d: int, eps: float = 1e-6) -> torch.Tensor:
    """x bf16 [rows, H, Dpad] view (last dim contiguous): RMSNorm over the first d channels of every head."""
    _req(x, bf16, "x"), _req(weight, torch.float32, "weight")
    rows, H, _ = x.shape
    check(lib.b200mix_head_rmsnorm_inplace(_p(x), rows, H, d, x.stride(0), x.stride(1), _p(weight), float(eps), _stream()),
          "b200mix_head_rmsnorm_inplace")
    _count()
    return x


def small_attention(qkv: torch.Tensor, B: int, T: int, S: int, H: int, d: int, *, scale: float, rope_cos=None,
                    rope_sin=None, q_norm_w=None, k_norm_w=None, eps: float = 1e-6, out=None) -> torch.Tensor:
    """qkv bf16 [B*T*S, 3*H*d] (row = (b*T+t)*S+s) -> bf16 [B*T*S, H*d]; attention along the T axis. qkv and out may
    be row-strided views (last dim contiguous)."""
    _req(qkv, bf16, "qkv")
    if out is None:
        out = torch.empty(qkv.shape[0], H * d, device=qkv.device, dtype=bf16)
    _req(out, bf16, "out")
    if qkv.stride(-1) != 1 or out.stride(-1) != 1:
        raise ValueError("small_attention: qkv and out need a contiguous last dimension")
    with _Timed("small_attention", 2.0 * 2 * qkv.shape[0] * 4 * H * d, "byte"):
        check(lib.b200mix_small_attention(_p(qkv), _p(out), B, T, S, H, d, qkv.stride(0), out.stride(0), _p(rope_cos),
                                          _p(rope_sin), _p(q_norm_w), _p(k_norm_w), float(eps), float(scale), _stream()),
              "b200mix_small_attention")
    _count()
    return out


def patchify3d(x: torch.Tensor, p: int) -> torch.Tensor:
    B, C, T, H, W = x.shape
    assert x.is_contiguous() and x.dtype in (torch.float32, bf16)
    out = torch.empty(B, T * (H // p) * (W // p), C * p * p, device=x.device, dtype=bf16)
    check(lib.b200mix_patchify3d(_p(x), 1 if x.dtype == torch.float32 else 0, _p(out), B, C, T, H, W, p, _stream()),
          "b200mix_patchify3d")
    _count()
    return out


def unpatchify3d(x: torch.Tensor, C: int, T: int, h: int, w: int, p: int) -> torch.Tensor:
    B = x.shape[0]
    assert x.is_contiguous() and x.dtype == bf16
    out = torch.empty(B, C, T, h * p, w * p, device=x.device, dtype=torch.float32)
    check(lib.b200mix_unpatchify3d(_p(x), _p(out), B, C, T, h, w, p, _stream()), "b200mix_unpatchify3d")
    _count()
    return out
