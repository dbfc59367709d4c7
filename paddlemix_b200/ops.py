"""Tensor-level wrappers over the C ABI. torch is used for device memory and streams only: every function below
enqueues hand-written sm_90a kernels from libb200mix.so on torch's current CUDA stream and raises if that fails.
"""
import ctypes
from typing import Optional

import torch

from . import _lib
from ._lib import (ACT_GELU_ERF, ACT_GELU_TANH, ACT_NONE, ACT_QUICK_GELU, ACT_RELU, ACT_SILU, GEMM_ACTS, GLU_GEGLU,
                   GLU_NONE, GLU_SWIGLU, Epilogue, check, lib)

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


def _launch(name, *args, kernels=1):
    """Calls lib.<name>(*args, stream) with tensors passed as their device pointers; raises if it fails and adds the
    `kernels` it starts to launches()."""
    check(getattr(lib, name)(*(_p(a) if isinstance(a, torch.Tensor) else a for a in args), _stream()), name)
    _count(kernels)


F32, BF16, FLOAT, I32, I64 = (torch.float32,), (bf16,), (torch.float32, bf16), (torch.int32,), (torch.int64,)
CONTIG = "contiguous"   # read flat: only a pointer reaches the kernel
STRIDED = "strided"     # the last dimension contiguous; the other strides are passed on
ROWS = "rows"           # STRIDED, with the passed strides multiples of 8 elements (16-byte TMA / vector strides)


def _fits(shape, want):
    if ... in want:
        i = want.index(...)
        head, tail = want[:i], want[i + 1:]
        return (len(shape) >= len(head) + len(tail) and _fits(shape[:i], head)
                and _fits(shape[len(shape) - len(tail):], tail))
    return len(shape) == len(want) and all(w is None or s == w for s, w in zip(shape, want))


class _Args:
    """The tensors one call hands its kernels, checked against what the kernels read. The kernels see pointers and
    the sizes and strides passed beside them, never the tensors, so these checks are what keeps a caller's mistake from
    becoming an out-of-bounds access. c(name, t, dtypes, shape, layout, numel) checks one tensor (None passes) and
    returns its shape; shape entries are sizes, None for any size, and at most one ... for any number of dimensions;
    layout None leaves the layout to the wrapper, which copies the tensor or checks it itself. c.on_cuda() then checks that every tensor seen is on the device: placement comes last, so CPU tensors reach every
    other refusal."""

    def __init__(self, op):
        self.op, self.seen = op, []

    def __call__(self, name, t, dtypes, shape=None, layout=CONTIG, numel=None):
        if t is None:
            return None
        op = self.op
        if t.dtype not in dtypes:
            raise TypeError(f"{op}: {name} must be {' or '.join(map(str, dtypes))}, got {t.dtype}")
        if layout == CONTIG and not t.is_contiguous():
            raise ValueError(f"{op}: {name} must be contiguous, got strides {t.stride()} for shape {tuple(t.shape)}")
        elif layout is not None and t.dim() and (
                (t.shape[-1] > 1 and t.stride(-1) != 1) or
                (layout == ROWS and any(s % 8 for n, s in zip(t.shape[:-1], t.stride()) if n > 1))):
            raise ValueError(f"{op}: {name} needs a contiguous last dimension"
                             f"{' and strides that are multiples of 8' if layout == ROWS else ''}, got strides "
                             f"{t.stride()} for shape {tuple(t.shape)}")
        if shape is not None and not _fits(t.shape, shape):
            want = ", ".join("..." if s is ... else "*" if s is None else str(s) for s in shape)
            raise ValueError(f"{op}: {name} must be [{want}], got {tuple(t.shape)}")
        if numel is not None and t.numel() != numel:
            raise ValueError(f"{op}: {name} has {t.numel()} elements, expected {numel}")
        self.seen.append((name, t))
        return t.shape

    def on_cuda(self):
        for name, t in self.seen:
            if not t.is_cuda:
                raise _lib.B200MixError(f"{self.op}: {name} must be a CUDA tensor (b200mix has no CPU path)")


def _gemm_act(op, act):
    """The GEMM epilogues implement ACT_NONE .. ACT_QUICK_GELU; ACT_RELU is an element-wise pass (activation())."""
    if act not in GEMM_ACTS:
        raise ValueError(f"{op}: act {act} is not a GEMM epilogue activation (ReLU runs through ops.activation)")


def _aligned16(op, **tensors):
    for name, t in tensors.items():
        if t is not None and t.data_ptr() % 16:
            raise ValueError(f"{op}: {name} must start on a 16-byte boundary")


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
    """The epilogue struct of tensors the calling wrapper has checked."""
    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    e = Epilogue()
    e.bias, e.row_add, e.row_gate, e.residual, e.stats_out = map(ptr, (bias, row_add, row_gate, residual, stats_out))
    e.ld_row = int(ld_row)
    e.rows_per_group = int(rows_per_group)
    e.ldr = int(ldr)
    e.act = int(act)
    e.glu = int(glu)
    e.out_fp32 = 1 if out_fp32 else 0
    e.out_scale = float(out_scale)
    e.residual_row_mod = int(residual_row_mod)
    if ln is not None:  # folded LayerNorm, consumer side: (RowStats of the input rows, colsum [N] fp32, eps[, rms])
        stats, colsum, eps = ln[:3]
        e.ln_stats, e.ln_colsum = stats.buf.data_ptr(), colsum.data_ptr()
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
        check(lib.b200mix_zero_bytes(_p(buf), buf.numel() * 8, _stream()), "b200mix_zero_bytes")  # a memset, not a kernel
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
    c = _Args("quantize_w8")
    N, K = c("w", w, FLOAT, (None, None), layout=None)
    c("workspace", workspace, BF16)
    if workspace is not None and workspace.numel() < N * K:
        raise ValueError(f"quantize_w8: the workspace holds {workspace.numel()} bf16 elements, a [{N}, {K}] weight "
                         f"needs {N * K}")
    c.on_cuda()
    w = w.contiguous()
    q = torch.empty(N * K, device=w.device, dtype=torch.int8)
    scale = torch.empty(N, device=w.device, dtype=torch.float32)
    _launch("b200mix_quantize_w8", w, 1 if w.dtype == torch.float32 else 0, q, scale, N, K)
    return Int8Weight(q, scale, N, K, workspace)


def _linear_io(c, a, K, n_out, out_fp32, out, residual, residual_row_mod):
    """Checks linear's a [..., K], out [..., n_out] and residual [rows, >= n_out] (rows >= M, or >= residual_row_mod
    when that is set). Returns a as a [M, K] matrix and out as the [M, n_out] view the kernel writes (None if out is)."""
    c("a", a, BF16, (..., K), layout=None)
    a2 = a.reshape(-1, K)
    M = a2.shape[0]
    c("out", out, F32 if out_fp32 else BF16, (..., n_out), STRIDED, numel=M * n_out)
    try:
        out2 = None if out is None else out.view(-1, n_out)
    except RuntimeError:
        raise ValueError(f"{c.op}: out of shape {tuple(out.shape)} and strides {out.stride()} cannot be viewed as "
                         f"[{M}, {n_out}]") from None
    res2 = None if residual is None else residual.reshape(-1, residual.shape[-1])
    c("residual", res2, BF16, (None, None), STRIDED)
    rows = residual_row_mod or M
    if res2 is not None and (res2.shape[0] < rows or res2.shape[1] < n_out):
        raise ValueError(f"{c.op}: residual of shape {tuple(residual.shape)} does not cover {rows} rows x {n_out} "
                         f"columns")
    return a2, out2, res2


def _linear_w8(a, w: Int8Weight, bias, act, glu, residual, out_fp32, out):
    c = _Args("linear")
    N, K = w.N, w.K
    n_out = N // 2 if glu else N
    a2, out2, res2 = _linear_io(c, a, K, n_out, out_fp32, out, residual, 0)
    c("bias", bias, F32, numel=N)
    c.on_cuda()
    if a2.stride(-1) != 1 or a2.data_ptr() % 16 or a2.stride(0) % 8:
        a2 = a2.contiguous()
    M = a2.shape[0]
    if out is None:
        out = torch.empty(*a.shape[:-1], n_out, device=a.device, dtype=torch.float32 if out_fp32 else bf16)
        out2 = out.view(-1, n_out)
    e = make_epilogue(bias=bias, residual=res2, ldr=0 if res2 is None else res2.stride(0), act=act, glu=glu,
                      out_fp32=out_fp32)
    ws = w.workspace
    need = ctypes.c_int64(0)  # above the weight-streaming range, the weight is expanded to bf16 first: two kernels
    check(lib.b200mix_linear_w8_workspace_size(M, N, K, ctypes.byref(need)), "b200mix_linear_w8_workspace_size")
    with _Timed("w8gemm", 2.0 * M * N * K, "flop", lambda: f"w8 {M}x{N}x{K}" + _epi_tag(e)):
        _launch("b200mix_linear_w8", a2, a2.stride(0), w.q, w.scale, out2, out2.stride(0), M, N, K, ctypes.byref(e), ws,
                0 if ws is None else 2 * ws.numel(), kernels=2 if need.value else 1)
    return out


def linear(a: torch.Tensor, w, bias=None, *, act=ACT_NONE, glu=GLU_NONE, residual=None, row_add=None,
           row_gate=None, rows_per_group=0, out_fp32=False, out=None, out_scale=1.0, residual_row_mod=0, stats=False,
           ln=None):
    """out[M, N(/2)] = epilogue(a[M, K] @ w[N, K]^T). a: bf16 [..., K] (last dim contiguous), w: bf16 [N, K] or an
    Int8Weight (then only bias / act / glu / residual / out_fp32 / out apply).
    stats=True or a ZEROED int64 [M, 2] tensor (RowStats.arena): also returns the RowStats of the output rows
    (-> (out, RowStats)); ln=(RowStats of a's rows, colsum, eps[, rms]): a is the UN-normalised tensor and w / bias carry
    the folded affine (fold_layernorm_into_linear)."""
    _gemm_act("linear", act)
    if isinstance(w, Int8Weight):
        unsupported = [n for n, on in (("row_add", row_add is not None), ("row_gate", row_gate is not None),
                                       ("rows_per_group", rows_per_group), ("out_scale", out_scale != 1.0),
                                       ("residual_row_mod", residual_row_mod), ("stats", stats is not None and stats is not False),
                                       ("ln", ln is not None)) if on]
        if unsupported:
            raise ValueError(f"an Int8Weight linear does not support {', '.join(unsupported)}")
        return _linear_w8(a, w, bias, act, glu, residual, out_fp32, out)
    c = _Args("linear")
    K = a.shape[-1]
    N = c("weight", w, BF16, (None, K), ROWS)[0]
    n_out = N // 2 if glu else N
    a2, out2, res2 = _linear_io(c, a, K, n_out, out_fp32, out, residual, residual_row_mod)
    M = a2.shape[0]
    c("bias", bias, F32, numel=N)
    c("row_add", row_add, F32, layout=None), c("row_gate", row_gate, F32, layout=None)
    mod = row_add if row_add is not None else row_gate
    if mod is not None:
        _check_mod_views("linear", row_add=row_add, row_gate=row_gate)
        _check_mod_groups("linear", M, rows_per_group, N, row_add=row_add, row_gate=row_gate)
    want_stats = stats is not None and stats is not False
    if want_stats and stats is not True:
        c("stats", stats, I64, (M, 2))
    if ln is not None:
        if ln[0].buf.shape[0] != M or ln[0].width != K:
            raise ValueError(f"row statistics are for a [{ln[0].buf.shape[0]}, {ln[0].width}] tensor, the input is [{M}, {K}]")
        c("ln stats", ln[0].buf, I64, (M, 2)), c("ln colsum", ln[1], F32, numel=N)
    c.on_cuda()
    if a2.stride(-1) != 1:
        a2 = a2.contiguous()
    if out is None:
        out = torch.empty(*a.shape[:-1], n_out, device=a.device, dtype=torch.float32 if out_fp32 else bf16)
        out2 = out.view(-1, n_out)
    rs = RowStats(RowStats.arena(1, M, a.device)[0] if stats is True else stats, N) if want_stats else None
    e = make_epilogue(bias=bias, row_add=row_add, row_gate=row_gate, ld_row=0 if mod is None else mod.stride(0),
                      rows_per_group=rows_per_group, residual=res2, ldr=0 if res2 is None else res2.stride(0), act=act,
                      glu=glu, out_fp32=out_fp32, out_scale=out_scale, residual_row_mod=residual_row_mod,
                      stats_out=None if rs is None else rs.buf, ln=ln)
    with _Timed("igemm", 2.0 * M * N * K, "flop", lambda: f"lin {M}x{N}x{K}" + _epi_tag(e)):
        _launch("b200mix_linear", a2, a2.stride(0), w, w.stride(0), out2, out2.stride(0), M, N, K, ctypes.byref(e))
    return (out, rs) if want_stats else out


def linear_batched(a: torch.Tensor, w: torch.Tensor, bias=None, *, out: torch.Tensor, act=ACT_NONE, glu=GLU_NONE,
                   residual=None, row_add=None, row_gate=None) -> torch.Tensor:
    """a: bf16 [B, rows, K] view (last dim contiguous, arbitrary row / batch strides); out: [B, rows, N(/2)] view with
    last dim contiguous (e.g. a token range of a joint [B, n_img+n_txt, *] buffer). Per-batch row_add / row_gate."""
    c = _Args("linear_batched")
    _gemm_act("linear_batched", act)
    B, rows, K = c("a", a, BF16, (None, None, None), ROWS)
    N = c("weight", w, BF16, (None, K), ROWS)[0]
    n_out = N // 2 if glu else N
    c("out", out, FLOAT, (B, rows, n_out), STRIDED)
    c("residual", residual, BF16, (B, rows, n_out), STRIDED)
    c("bias", bias, F32, numel=N)
    c("row_add", row_add, F32, layout=None), c("row_gate", row_gate, F32, layout=None)
    mod = row_add if row_add is not None else row_gate
    if mod is not None:
        _check_mod_views("linear_batched", row_add=row_add, row_gate=row_gate)
        _check_mod_groups("linear_batched", B * rows, rows, n_out, row_add=row_add, row_gate=row_gate)
    c.on_cuda()
    e = make_epilogue(bias=bias, row_add=row_add, row_gate=row_gate, ld_row=0 if mod is None else mod.stride(0),
                      rows_per_group=rows, residual=residual, ldr=0 if residual is None else residual.stride(1),
                      act=act, glu=glu, out_fp32=(out.dtype == torch.float32))
    with _Timed("igemm", 2.0 * B * rows * N * K, "flop", lambda: f"linb {B}*{rows}x{N}x{K}" + _epi_tag(e)):
        _launch("b200mix_linear_batched", a, a.stride(1), a.stride(0), w, w.stride(0), out, out.stride(1), out.stride(0),
                rows, B, N, K, ctypes.byref(e), 0 if residual is None else residual.stride(0))
    return out


def patchify(x: torch.Tensor, p: int) -> torch.Tensor:
    c = _Args("patchify")
    B, C, H, W = c("x", x, FLOAT, (None,) * 4)
    c.on_cuda()
    out = torch.empty(B, (H // p) * (W // p), C * p * p, device=x.device, dtype=bf16)
    _launch("b200mix_patchify", x, 1 if x.dtype == torch.float32 else 0, out, B, C, H, W, p)
    return out


def unpatchify(x: torch.Tensor, C: int, h: int, w: int, p: int, out_dtype=bf16) -> torch.Tensor:
    c = _Args("unpatchify")
    B = x.shape[0]
    c("x", x, BF16, numel=B * h * w * p * p * C)
    out = torch.empty(B, C, h * p, w * p, device=x.device, dtype=out_dtype)
    c("out", out, FLOAT)
    c.on_cuda()
    _launch("b200mix_unpatchify", x, out, 1 if out_dtype == torch.float32 else 0, B, C, h, w, p)
    return out


def conv3x3(x: torch.Tensor, w: torch.Tensor, bias=None, *, stride=1, row_add=None, residual=None, act=ACT_NONE,
            out_scale=1.0, out=None) -> torch.Tensor:
    """x: bf16 NHWC [B,H,W,Cin] contiguous; w: bf16 [Cout,3,3,Cin] contiguous; returns bf16 NHWC."""
    c = _Args("conv3x3")
    _gemm_act("conv3x3", act)
    B, H, W, Cin = c("x", x, BF16, (None,) * 4)
    Cout = c("w", w, BF16, (None, 3, 3, Cin))[0]
    Ho, Wo = H // stride, W // stride
    c("out", out, BF16, (B, Ho, Wo, Cout)), c("residual", residual, BF16, (B, Ho, Wo, Cout))
    c("bias", bias, F32, numel=Cout), c("row_add", row_add, F32, layout=None)
    if row_add is not None:
        _check_mod_views("conv3x3", row_add=row_add)
        _check_mod_groups("conv3x3", B * Ho * Wo, Ho * Wo, Cout, row_add=row_add)
    c.on_cuda()
    if out is None:
        out = torch.empty(B, Ho, Wo, Cout, device=x.device, dtype=bf16)
    e = make_epilogue(bias=bias, row_add=row_add, ld_row=0 if row_add is None else row_add.stride(0),
                      rows_per_group=Ho * Wo, residual=residual, ldr=Cout, act=act, out_scale=out_scale)
    with _Timed("igemm", 2.0 * B * Ho * Wo * Cout * 9 * Cin, "flop",
                lambda: f"conv{stride} {B * Ho * Wo}x{Cout}x{9 * Cin}" + _epi_tag(e)):
        _launch("b200mix_conv3x3", x, w, out, B, H, W, Cin, Cout, stride, ctypes.byref(e))
    return out


def fold_upsample_conv_weight(w: torch.Tensor) -> torch.Tensor:
    """w: [Cout, 3, 3, Cin] (any float dtype; fold from the fp32 master weights when they exist) -> bf16 [Cout, 16, Cin],
    the per-output-parity 2x2 filters of nearest-2x-upsample + conv3x3 (b200mix_conv3x3_up2x). Row index =
    (py*2 + px)*4 + a*2 + b; taps that read the same low-resolution pixel are summed in fp32 and rounded once."""
    return fold_upsample_taps(w).to(bf16).contiguous()


def fold_upsample_taps(w: torch.Tensor) -> torch.Tensor:
    """The fp32 tap sums of fold_upsample_conv_weight, before rounding: [O, 3, 3, I] -> fp32 [O, 16, I]. Linear in w,
    so it also maps a LoRA down factor's taps [r, 3, 3, I] to its columns in the folded layout."""
    O, _, _, I = w.shape
    wf = w.float()
    groups = {0: ((0,), (1, 2)), 1: ((0, 1), (2,))}  # parity -> (taps folded into a = 0, taps folded into a = 1)
    out = torch.empty(O, 2, 2, 2, 2, I, dtype=torch.float32, device=w.device)
    for py in range(2):
        for px in range(2):
            for a in range(2):
                for b in range(2):
                    out[:, py, px, a, b] = sum(wf[:, ky, kx] for ky in groups[py][a] for kx in groups[px][b])
    return out.reshape(O, 16, I)


def conv3x3_up2x(x: torch.Tensor, w4: torch.Tensor, bias=None, *, row_add=None, residual=None, act=ACT_NONE,
                 out_scale=1.0, out=None) -> torch.Tensor:
    """conv3x3(nearest_upsample_2x(x)) from the low-resolution x: bf16 NHWC [B,H,W,Cin]; w4 = fold_upsample_conv_weight(w).
    Returns bf16 NHWC [B,2H,2W,Cout] (Upsample2D, resnet.py:169-218)."""
    c = _Args("conv3x3_up2x")
    _gemm_act("conv3x3_up2x", act)
    B, H, W, Cin = c("x", x, BF16, (None,) * 4)
    Cout = c("w4", w4, BF16, (None, 16, Cin))[0]
    c("out", out, BF16, (B, 2 * H, 2 * W, Cout)), c("residual", residual, BF16, (B, 2 * H, 2 * W, Cout))
    c("bias", bias, F32, numel=Cout), c("row_add", row_add, F32, layout=None)
    if row_add is not None:
        _check_mod_views("conv3x3_up2x", row_add=row_add)
        _check_mod_groups("conv3x3_up2x", B * 4 * H * W, 4 * H * W, Cout, row_add=row_add)
    c.on_cuda()
    if out is None:
        out = torch.empty(B, 2 * H, 2 * W, Cout, device=x.device, dtype=bf16)
    e = make_epilogue(bias=bias, row_add=row_add, ld_row=0 if row_add is None else row_add.stride(0),
                      rows_per_group=4 * H * W, residual=residual, ldr=Cout, act=act, out_scale=out_scale)
    with _Timed("igemm", 2.0 * B * 4 * H * W * Cout * 4 * Cin, "flop",
                lambda: f"convup {B * 4 * H * W}x{Cout}x{4 * Cin}" + _epi_tag(e)):
        _launch("b200mix_conv3x3_up2x", x, w4, out, B, H, W, Cin, Cout, ctypes.byref(e))
    return out


def conv3x3_small_cin(x: torch.Tensor, w: torch.Tensor, bias=None) -> torch.Tensor:
    c = _Args("conv3x3_small_cin")
    B, H, W, Cin = c("x", x, FLOAT, (None,) * 4)
    Cout = c("w", w, BF16, (None, 3, 3, Cin))[0]
    c("bias", bias, F32, numel=Cout)
    c.on_cuda()
    out = torch.empty(B, H, W, Cout, device=x.device, dtype=bf16)
    _launch("b200mix_conv3x3_small_cin", x, 1 if x.dtype == torch.float32 else 0, w, bias, out, B, H, W, Cin, Cout)
    return out


def conv3x3_narrow(x: torch.Tensor, w: torch.Tensor, bias=None, *, stride=1, act=ACT_NONE, out=None) -> torch.Tensor:
    """act(conv3x3(x) + bias) for 1 <= Cin <= 128 (the ControlNet conditioning embedding). x: bf16 NHWC [B,H,W,Cin]
    contiguous; w: bf16 [Cout,3,3,Cin] contiguous; bias fp32 [Cout] or None; act ACT_NONE | ACT_SILU. Returns bf16 NHWC
    [B,H/stride,W/stride,Cout]."""
    c = _Args("conv3x3_narrow")
    B, H, W, Cin = c("x", x, BF16, (None,) * 4)
    Cout = c("w", w, BF16, (None, 3, 3, Cin))[0]
    c("bias", bias, F32, numel=Cout), c("out", out, BF16, (B, H // stride, W // stride, Cout))
    c.on_cuda()
    if out is None:
        out = torch.empty(B, H // stride, W // stride, Cout, device=x.device, dtype=bf16)
    with _Timed("conv_narrow", 2.0 * B * (H // stride) * (W // stride) * Cout * 9 * Cin, "flop",
                lambda: f"convn{stride} {B}x{H}x{W}x{Cin}->{Cout}"):
        _launch("b200mix_conv3x3_narrow", x, w, bias, out, B, H, W, Cin, Cout, int(stride), int(act))
    return out


def sdpa(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, *, scale: Optional[float] = None, causal=False,
         cu_seqlens: Optional[torch.Tensor] = None, kv_lens: Optional[torch.Tensor] = None,
         attn_mask: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """q: [B,Sq,Hq,D], k/v: [B,Sk,Hkv,D] bf16 views (head_dim contiguous; other strides arbitrary multiples of 8).
    attn_mask: additive bias (bf16 / fp32) broadcastable to [B,Hq,Sq,Sk] with a contiguous key axis (the reference's
    `attn_mask` argument, paddle_patch.py:418). Returns [B,Sq,Hq,D] (the layout of scaled_dot_product_attention_)."""
    c = _Args("sdpa")
    B, Sq, Hq, D = c("q", q, BF16, (None,) * 4, ROWS)
    _, Sk, Hkv, _ = c("k", k, BF16, (B, None, None, D), ROWS)
    c("v", v, BF16, (B, Sk, Hkv, D), ROWS), c("out", out, BF16, (B, Sq, Hq, D), ROWS)
    if Hq % Hkv:
        raise ValueError(f"sdpa: {Hq} query heads cannot share {Hkv} key / value heads")
    c("cu_seqlens", cu_seqlens, I32, (None,)), c("kv_lens", kv_lens, I32, numel=B)
    m_fp32, msb, msh, msq = 0, 0, 0, 0
    if attn_mask is not None:
        if attn_mask.dtype not in FLOAT:
            raise TypeError(f"attn_mask must be an additive float32 / bfloat16 bias, got {attn_mask.dtype}")
        while attn_mask.dim() < 4:
            attn_mask = attn_mask.unsqueeze(0)
        if attn_mask.shape[-1] != Sk or any(a not in (1, n) for a, n in zip(attn_mask.shape[:3], (B, Hq, Sq))):
            raise ValueError(f"attn_mask shape {tuple(attn_mask.shape)} does not broadcast to {(B, Hq, Sq, Sk)}")
        c("attn_mask", attn_mask, FLOAT, layout=None)
    c.on_cuda()
    if out is None:
        out = torch.empty(B, Sq, Hq, D, device=q.device, dtype=bf16)
    if scale is None:
        scale = D ** -0.5
    nseq = 0 if cu_seqlens is None else cu_seqlens.numel() - 1
    if attn_mask is not None:
        if attn_mask.stride(-1) != 1 and Sk > 1:
            attn_mask = attn_mask.contiguous()
        m_fp32 = 1 if attn_mask.dtype == torch.float32 else 0
        msb, msh, msq = (0 if attn_mask.shape[i] == 1 else attn_mask.stride(i) for i in range(3))
    with _Timed("attention", 4.0 * B * Hq * Sq * Sk * D * (0.5 if causal else 1.0), "flop",
                lambda: f"attn B{B} H{Hq} Sq{Sq} Sk{Sk} D{D}" + (" causal" if causal else "")):
        _launch("b200mix_sdpa", q, k, v, out, B, Hq, Hkv, Sq, Sk, D, q.stride(0), q.stride(1), q.stride(2), k.stride(0),
                k.stride(1), k.stride(2), v.stride(0), v.stride(1), v.stride(2), out.stride(0), out.stride(1),
                out.stride(2), float(scale), 1 if causal else 0, cu_seqlens, nseq, kv_lens, attn_mask, m_fp32, msb, msh,
                msq)
    return out


_gn_scratch = {}


def groupnorm_nhwc(x1: torch.Tensor, gamma, beta, *, x2=None, groups=32, eps=1e-5, silu=False, out=None):
    """x1: bf16 [B,H,W,C1] (optionally concatenated on channels with x2 [B,H,W,C2]); returns bf16 [B,H,W,C1+C2]."""
    c = _Args("groupnorm_nhwc")
    pix = c("x1", x1, BF16, (None, ...))[:-1]
    B, C1 = x1.shape[0], x1.shape[-1]
    C2 = 0 if x2 is None else c("x2", x2, BF16, (*pix, None))[-1]
    c("gamma", gamma, F32, numel=C1 + C2), c("beta", beta, F32, numel=C1 + C2)
    c("out", out, BF16, (*pix, C1 + C2))
    c.on_cuda()
    HW = x1.numel() // (B * C1)
    if out is None:
        out = torch.empty(*pix, C1 + C2, device=x1.device, dtype=bf16)
    # per-(device, stream, B, groups) scratch: two streams never share partial sums, and the size is exact for the key
    key = (x1.device, torch.cuda.current_stream().cuda_stream, B, groups)
    st = _gn_scratch.get(key)
    if st is None:
        # zero-filled once: the first 4 KB hold the per-batch arrival counters, which every call leaves at zero
        st = torch.zeros(512 + (1024 + 2 * B) * groups * 2, device=x1.device, dtype=torch.float64)
        _gn_scratch[key] = st
    with _Timed("groupnorm", 2.0 * 2 * B * HW * (C1 + C2), "byte", lambda: f"gn {B}x{HW}x{C1 + C2}"):  # algorithmic: read once + write once (bf16)
        _launch("b200mix_groupnorm_nhwc", x1, C1, x2, C2, gamma, beta, out, st, st.numel() * 8, B, HW, groups,
                float(eps), 1 if silu else 0, kernels=2)
    return out


def layernorm(x: torch.Tensor, weight=None, bias=None, *, eps=1e-5, rms=False, delta=None, gate=None, scale=None,
              shift=None, rows_per_group=0, want_resid=False, out=None):
    """Row-wise (RMS/Layer)Norm with optional fused residual update x + gate*delta and AdaLN modulation.
    Returns y, or (resid, y) when want_resid."""
    c = _Args("layernorm")
    N = c("x", x, BF16, (..., None), layout=None)[-1]
    M = x.numel() // N
    c("delta", delta, BF16, x.shape), c("out", out, BF16, x.shape)
    c("weight", weight, F32, numel=N), c("bias", bias, F32, numel=N)
    for name, v in (("gate", gate), ("scale", scale), ("shift", shift)):
        c(name, v, F32, layout=None)
    mod = gate if gate is not None else (scale if scale is not None else shift)
    if mod is not None:
        _check_mod_views("layernorm", gate=gate, scale=scale, shift=shift)
        _check_mod_groups("layernorm", M, rows_per_group, N, gate=gate, scale=scale, shift=shift)
    c.on_cuda()
    x2 = x.reshape(-1, N).contiguous()
    if out is None:
        out = torch.empty_like(x2).view(x.shape)
    resid = torch.empty_like(x2).view(x.shape) if (want_resid and delta is not None) else None
    ld_mod = 0 if mod is None else mod.stride(0)
    nbytes = 2.0 * M * N * (2 + (1 if delta is not None else 0) + (1 if resid is not None else 0))
    with _Timed("layernorm", nbytes, "byte", lambda: f"ln {M}x{N}" + (" +delta" if delta is not None else "")):
        _launch("b200mix_layernorm", x2, delta, gate, resid, out, weight, bias, scale, shift, ld_mod, rows_per_group, M,
                N, float(eps), 1 if rms else 0)
    if want_resid:
        return (resid if resid is not None else x), out
    return out


def softmax_rows(x: torch.Tensor, scale: float = 1.0, out=None) -> torch.Tensor:
    """x: fp32 [M, N] (row stride arbitrary multiple of 4) -> bf16 softmax(x * scale) [M, N]."""
    c = _Args("softmax_rows")
    M, N = c("x", x, F32, (None, None), STRIDED)
    c("out", out, BF16, (M, N), STRIDED)
    c.on_cuda()
    if out is None:
        out = torch.empty(M, N, device=x.device, dtype=bf16)
    with _Timed("softmax", 4.0 * M * N + 2.0 * M * N, "byte", lambda: f"softmax {M}x{N}"):
        _launch("b200mix_softmax_rows", x, out, M, N, x.stride(0), out.stride(0), float(scale))
    return out


def timestep_embedding(t: torch.Tensor, dim: int, *, flip_sin_to_cos=True, downscale_freq_shift=0.0, scale=1.0,
                       max_period=10000.0, out=None, col0=0, out_dtype=bf16):
    c = _Args("timestep_embedding")
    c("t", t, F32)
    B = t.numel()
    if out is None:
        out = torch.empty(B, dim, device=t.device, dtype=out_dtype)
    width = c("out", out, FLOAT, (B, None), STRIDED)[1]
    if col0 < 0 or col0 + dim > width:
        raise ValueError(f"timestep_embedding: columns [{col0}, {col0 + dim}) do not fit out's {width}")
    c.on_cuda()
    _launch("b200mix_timestep_embedding", t, out, 1 if out.dtype == torch.float32 else 0, B, dim, out.stride(0), col0,
            1 if flip_sin_to_cos else 0, float(downscale_freq_shift), float(scale), float(max_period))
    return out


def activation(x: torch.Tensor, act: int, out_dtype=None):
    """act(x) element-wise, bf16 / fp32 in and out; act is any ACT_* (ACT_RELU only here, not in the GEMMs)."""
    c = _Args("activation")
    if act not in GEMM_ACTS + (ACT_RELU,):
        raise ValueError(f"activation: unknown act {act}")
    c("x", x, FLOAT)
    out = torch.empty_like(x, dtype=out_dtype or x.dtype)
    c("out", out, FLOAT)
    c.on_cuda()
    _launch("b200mix_activation", x, out, x.numel(), act, 1 if x.dtype == torch.float32 else 0,
            1 if out.dtype == torch.float32 else 0)
    return out


def upsample_nearest2x(x: torch.Tensor):
    c = _Args("upsample_nearest2x")
    B, H, W, C = c("x", x, BF16, (None,) * 4)
    c.on_cuda()
    out = torch.empty(B, 2 * H, 2 * W, C, device=x.device, dtype=bf16)
    _launch("b200mix_upsample_nearest2x_nhwc", x, out, B, H, W, C)
    return out


def concat_channels(x1: torch.Tensor, x2: torch.Tensor):
    c = _Args("concat_channels")
    C1 = c("x1", x1, BF16, (..., None))[-1]
    C2 = c("x2", x2, BF16, (*x1.shape[:-1], None))[-1]
    c.on_cuda()
    out = torch.empty(*x1.shape[:-1], C1 + C2, device=x1.device, dtype=bf16)
    _launch("b200mix_concat_channels", x1, C1, x2, C2, out, x1.numel() // C1)
    return out


def nchw_to_nhwc(x: torch.Tensor):
    c = _Args("nchw_to_nhwc")
    B, C, H, W = c("x", x, FLOAT, (None,) * 4)
    c.on_cuda()
    out = torch.empty(B, H, W, C, device=x.device, dtype=bf16)
    _launch("b200mix_nchw_to_nhwc", x, 1 if x.dtype == torch.float32 else 0, out, B, C, H, W)
    return out


def nhwc_to_nchw(x: torch.Tensor, out_dtype=torch.float32, out=None):
    c = _Args("nhwc_to_nchw")
    B, H, W, C = c("x", x, BF16, (None,) * 4)
    if out is None:
        out = torch.empty(B, C, H, W, device=x.device, dtype=out_dtype)
    c("out", out, FLOAT, (B, C, H, W))
    c.on_cuda()
    _launch("b200mix_nhwc_to_nchw", x, out, 1 if out.dtype == torch.float32 else 0, B, C, H, W)
    return out


def pixel_unshuffle(x: torch.Tensor, f: int) -> torch.Tensor:
    """nn.PixelUnshuffle(f) + the cast to bf16: x fp32 / bf16 NCHW [B,C,H,W] (H, W multiples of f; f 8 or 16) ->
    bf16 NHWC [B,H/f,W/f,C*f*f], channel c*f*f + i*f + j = x[b, c, h*f + i, w*f + j]."""
    c = _Args("pixel_unshuffle")
    B, C, H, W = c("x", x, FLOAT, (None,) * 4)
    if f not in (8, 16):
        raise ValueError(f"pixel_unshuffle: downscale factor must be 8 or 16, got {f}")
    if H % f or W % f:
        raise ValueError(f"pixel_unshuffle: H={H} and W={W} must be multiples of {f}")
    _aligned16("pixel_unshuffle", x=x)
    c.on_cuda()
    out = torch.empty(B, H // f, W // f, C * f * f, device=x.device, dtype=bf16)
    nbytes = x.numel() * x.element_size() + out.numel() * 2
    with _Timed("adapter_io", nbytes, "byte", lambda: f"unshuffle{f} {B}x{C}x{H}x{W}"):
        _launch("b200mix_pixel_unshuffle", x, 1 if x.dtype == torch.float32 else 0, out, B, C, H, W, int(f))
    return out


def avgpool2x2_nhwc(x: torch.Tensor) -> torch.Tensor:
    """nn.AvgPool2D(kernel_size=2, stride=2, ceil_mode=True) (exclusive: a window over an odd edge averages its valid
    pixels) on bf16 NHWC [B,H,W,C], C % 8 == 0. Returns bf16 NHWC [B,ceil(H/2),ceil(W/2),C]."""
    c = _Args("avgpool2x2_nhwc")
    B, H, W, C = c("x", x, BF16, (None,) * 4)
    if C % 8:
        raise ValueError(f"avgpool2x2_nhwc: C={C} must be a multiple of 8")
    _aligned16("avgpool2x2_nhwc", x=x)
    c.on_cuda()
    out = torch.empty(B, (H + 1) // 2, (W + 1) // 2, C, device=x.device, dtype=bf16)
    with _Timed("adapter_io", 2.0 * (x.numel() + out.numel()), "byte", lambda: f"avgpool {B}x{H}x{W}x{C}"):
        _launch("b200mix_avgpool2x2_nhwc", x, out, B, H, W, C)
    return out


def weighted_sum_rows(xs, weights, out: torch.Tensor) -> torch.Tensor:
    """out[r] = sum_k weights[k] * xs[k][r % xs[k].shape[0]], summed in fp32 and rounded to bf16 once. xs: 1 to 8 bf16
    contiguous tensors [rows_k, ...] with out's trailing shape; out: bf16 contiguous [rows, ...], not overlapping any
    input; the row size a multiple of 8. The T2I-Adapter residual write: weighted sum, scale, tile and CFG doubling."""
    c = _Args("weighted_sum_rows")
    xs, weights = list(xs), [float(w) for w in weights]
    if not 1 <= len(xs) <= 8 or len(weights) != len(xs):
        raise ValueError(f"weighted_sum_rows: 1 to 8 inputs with one weight each, got {len(xs)} and {len(weights)}")
    tail = c("out", out, BF16, (None, ...))[1:]
    for k, x in enumerate(xs):
        c(f"xs[{k}]", x, BF16, (None, *tail))
    row = out[0].numel()
    if row % 8:
        raise ValueError(f"weighted_sum_rows: {row} elements per row, must be a multiple of 8")
    _aligned16("weighted_sum_rows", out=out, **{f"xs[{k}]": x for k, x in enumerate(xs)})
    c.on_cuda()
    n = len(xs)
    ptrs = (ctypes.c_void_p * n)(*[x.data_ptr() for x in xs])
    rows = (ctypes.c_int64 * n)(*[x.shape[0] for x in xs])
    ws = (ctypes.c_float * n)(*weights)
    with _Timed("adapter_io", 2.0 * (sum(x.numel() for x in xs) + out.numel()), "byte",
                lambda: f"wsum {n}x{out.shape[0]}x{row}"):
        _launch("b200mix_weighted_sum_rows", n, ptrs, rows, ws, out, out.shape[0], row)
    return out


def _span(t: torch.Tensor):
    """[first byte, last byte + 1) of a tensor whose last dimension is contiguous."""
    n = 1 + sum((s - 1) * st for s, st in zip(t.shape, t.stride()))
    return t.data_ptr(), t.data_ptr() + n * t.element_size()


def lora_apply(items) -> None:
    """Rebuilds LoRA targets in one launch (b200mix_lora_apply). items: sequence of dicts with
      out  bf16 [N, K] (a weight or a row slice of one: last dimension contiguous, row stride a multiple of 8),
      base bf16 [N, K] (the snapshot; same layout rules), U fp32 [N, R], D fp32 [R, K] (contiguous),
      and optionally col_scale fp32 [K], colsum / colsum_base fp32 [N] (together).
    out[n, k] = bf16(base[n, k] + col_scale[k] * (U @ D)[n, k]); colsum = colsum_base + row sums of (out - base).
    R must be a multiple of 8 (pad with zero columns / rows) and at most 512; K a multiple of 8. Every item is checked
    before anything is launched; outputs must not overlap each other or any input."""
    c = _Args("lora_apply")
    items = list(items)
    if not items:
        raise ValueError("lora_apply: no items")
    spans = []
    for i, it in enumerate(items):
        unknown = set(it) - {"out", "base", "U", "D", "col_scale", "colsum", "colsum_base"}
        if unknown:
            raise ValueError(f"lora_apply: item {i} has unknown fields {sorted(unknown)}")
        N, K = c(f"items[{i}].out", it["out"], BF16, (None, None), ROWS)
        R = c(f"items[{i}].U", it["U"], F32, (N, None))[1]
        c(f"items[{i}].base", it["base"], BF16, (N, K), ROWS)
        c(f"items[{i}].D", it["D"], F32, (R, K))
        c(f"items[{i}].col_scale", it.get("col_scale"), F32, (K,))
        c(f"items[{i}].colsum", it.get("colsum"), F32, (N,))
        c(f"items[{i}].colsum_base", it.get("colsum_base"), F32, (N,))
        if (it.get("colsum") is None) != (it.get("colsum_base") is None):
            raise ValueError(f"lora_apply: items[{i}]: colsum and colsum_base go together")
        if R == 0 or R % 8 or R > _lib.LORA_MAX_RANK or K % 8:
            raise ValueError(f"lora_apply: items[{i}]: R = {R} must be a positive multiple of 8 up to "
                             f"{_lib.LORA_MAX_RANK} and K = {K} a multiple of 8")
        _aligned16("lora_apply", **{f"items[{i}].{k}": it[k] for k in ("out", "base", "U", "D")})
        ins = [_span(it[k]) for k in ("base", "U", "D", "col_scale", "colsum_base") if it.get(k) is not None]
        for k in ("out", "colsum"):
            if it.get(k) is not None:
                o0, o1 = _span(it[k])
                if any(a < o1 and o0 < b for a, b in ins):
                    raise ValueError(f"lora_apply: items[{i}].{k} overlaps one of the item's inputs")
                spans.append((o0, o1, f"items[{i}].{k}"))
    spans.sort()
    for (a0, a1, na), (b0, b1, nb) in zip(spans, spans[1:]):
        if b0 < a1:
            raise ValueError(f"lora_apply: {na} and {nb} overlap")
    c.on_cuda()
    arr = (_lib.LoraItem * len(items))()
    for i, it in enumerate(items):
        o, b = it["out"], it["base"]
        arr[i] = _lib.LoraItem(o.data_ptr(), b.data_ptr(), it["U"].data_ptr(), it["D"].data_ptr(),
                               *(None if it.get(k) is None else it[k].data_ptr()
                                 for k in ("col_scale", "colsum", "colsum_base")),
                               o.stride(0), b.stride(0), o.shape[0], o.shape[1], it["U"].shape[1])
    need = ctypes.c_int64()
    check(lib.b200mix_lora_workspace_size(len(items), ctypes.byref(need)), "b200mix_lora_workspace_size")
    ws = torch.empty(need.value, dtype=torch.uint8, device=items[0]["out"].device)
    moved = sum(4.0 * it["out"].numel() + 4.0 * (it["U"].numel() + it["D"].numel()) for it in items)
    with _Timed("lora", moved, "byte", lambda: f"lora {len(items)} items"):
        _launch("b200mix_lora_apply", arr, len(items), ws, need.value)


def zero_(t: torch.Tensor) -> torch.Tensor:
    """Sets a contiguous device tensor to zero (a memset on the current stream, not a kernel)."""
    c = _Args("zero_")
    c("t", t, (bf16, torch.float32, torch.int32, torch.int64))
    c.on_cuda()
    check(lib.b200mix_zero_bytes(_p(t), t.numel() * t.element_size(), _stream()), "b200mix_zero_bytes")
    return t


def add_residual_nhwc(a: torch.Tensor, r: torch.Tensor, *, r_nchw: bool, out=None) -> torch.Tensor:
    """a: bf16 NHWC [B,H,W,C]; r: the same values as NHWC bf16, or NCHW fp32 / bf16 [B,C,H,W] (r_nchw). Returns a + r."""
    c = _Args("add_residual_nhwc")
    B, H, W, C = c("a", a, BF16, (None,) * 4)
    want = (B, C, H, W) if r_nchw else (B, H, W, C)
    if tuple(r.shape) != want:
        raise ValueError(f"residual shape {tuple(r.shape)} does not match the activation {want}")
    c("out", out, BF16, (B, H, W, C))
    c.on_cuda()
    if r.dtype not in FLOAT:
        r = r.float()
    r = r.to(a.device).contiguous()
    if out is None:
        out = torch.empty_like(a)
    _launch("b200mix_add_residual_nhwc", a, r, 1 if r.dtype == torch.float32 else 0, 1 if r_nchw else 0, out, B, C, H,
            W)
    return out


def _step_tensors(op, x, m_u, m_c, out, **fp32_bufs):
    """Checks the tensors of a sampler step before anything is launched; returns (m_u's dtype flag, out), allocating out
    like x (like m_u when x is None) if it is None. The kernels read every tensor flat over x's element count (m_u's
    when x is None) and m_c with m_u's dtype flag, so each given tensor must be contiguous, have that many elements and
    the dtype below: x, out and fp32_bufs fp32, m_u fp32 or bf16, m_c m_u's dtype."""
    c = _Args(op)
    n = (m_u if x is None else x).numel()
    c("x", x, F32, numel=n), c("model output", m_u, FLOAT, numel=n)
    c("model_output_cond", m_c, (m_u.dtype,), numel=n), c("out", out, F32, numel=n)
    for name, t in fp32_bufs.items():
        c(name, t, F32, numel=n)
    c.on_cuda()
    if out is None:
        like = m_u if x is None else x
        out = torch.empty(like.shape, device=like.device, dtype=torch.float32)
    return (1 if m_u.dtype == torch.float32 else 0), out


PRED_TYPES = {"epsilon": 0, "sample": 1, "v_prediction": 2}


def ddim_step(m_u, m_c, guidance, x, sa_t, sb_t, sa_p, sb_p, prediction_type="epsilon", clip_sample_range=0.0, out=None):
    """DDIM step for any prediction_type, optional x0 clipping (clip_sample_range > 0), fused CFG combine."""
    fp32, out = _step_tensors("ddim_step", x, m_u, m_c, out)
    _launch("b200mix_ddim_step_ex", m_u, m_c, fp32, float(guidance), x, out, x.numel(), float(sa_t), float(sb_t),
            float(sa_p), float(sb_p), PRED_TYPES[prediction_type], float(clip_sample_range))
    return out


def lcm_step(m_u, m_c, guidance, x, noise, sa_t, sb_t, c_skip, c_out, sa_p, sb_p, prediction_type="epsilon",
             clip_sample_range=0.0, out=None, denoised=None):
    """LCMScheduler.step; noise None = final step (x_prev = denoised)."""
    fp32, out = _step_tensors("lcm_step", x, m_u, m_c, out, noise=noise, denoised=denoised)
    _launch("b200mix_lcm_step", m_u, m_c, fp32, float(guidance), x, noise, out, denoised, x.numel(), float(sa_t),
            float(sb_t), float(c_skip), float(c_out), float(sa_p), float(sb_p), PRED_TYPES[prediction_type],
            float(clip_sample_range))
    return out


def iddpm_step(model_out, x, cfg_scale, cfg_channel, scalars, add_noise, seed=0, step=0, noise=None, out=None, out_dup=None):
    """Open-Sora IDDPM p_sample behind forward_with_cfg (b200mix_iddpm_step). model_out [2B, 2C, ...] fp32 | bf16 with
    the conditional rows first; x fp32 [B, C, ...]; scalars = (sqrt_recip_ac, sqrt_recipm1_ac, coef1, coef2, max_log,
    min_log) as fp32 values; noise fp32 like x, or None for Philox noise keyed by (seed, step). out may be x itself;
    out_dup receives a second copy of the result. Returns out."""
    c = _Args("iddpm_step")
    B, C = c("x", x, F32, (None, None, ...))[:2]
    c("model_out", model_out, FLOAT, (2 * B, 2 * C, *x.shape[2:]))
    c("noise", noise, F32, x.shape), c("out", out, F32, x.shape), c("out_dup", out_dup, F32, x.shape)
    c.on_cuda()
    if out is None:
        out = torch.empty_like(x)
    _launch("b200mix_iddpm_step", model_out, 1 if model_out.dtype == torch.float32 else 0, x, noise, out, out_dup, B, C,
            x.numel() // (B * C), float(cfg_scale), int(cfg_channel), *(float(v) for v in scalars),
            1 if add_noise else 0, int(seed), int(step))
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
        _launch("b200mix_cfg_rescale_ratio", eps_u, eps_c, fp32, float(guidance), ratio, B, nps)
    _launch("b200mix_cfg_combine", eps_u, eps_c, fp32, float(guidance), ratio, float(guidance_rescale), nps, out,
            eps_u.numel())
    return out


def euler_step(v_u, v_c, guidance, x, sigma, dt, out=None):
    fp32, out = _step_tensors("euler_step", x, v_u, v_c, out)
    _launch("b200mix_euler_step", v_u, v_c, fp32, float(guidance), x, out, x.numel(), float(sigma), float(dt))
    return out


def dpmpp_2m_step(eps_u, eps_c, guidance, x, m_prev, m_out, sigma_cur, alpha_cur, A, C, halfC, inv_r0, out=None):
    """DPM-Solver++ 2M update (see include/b200mix.h); m_prev None = first-order step; m_out receives x0."""
    fp32, out = _step_tensors("dpmpp_2m_step", x, eps_u, eps_c, out, m_prev=m_prev, m_out=m_out)
    _launch("b200mix_dpmpp_2m_step", eps_u, eps_c, fp32, float(guidance), x, m_prev, out, m_out, x.numel(),
            float(sigma_cur), float(alpha_cur), float(A), float(C), float(halfC), float(inv_r0))
    return out


def ddim_eta_step(m_u, m_c, guidance, x, noise, sa_t, sb_t, sa_p, sb_p, std_dev_t, prediction_type="epsilon",
                  clip_sample_range=0.0, use_clipped_model_output=False, seed=0, step=0, out=None):
    """DDIMScheduler.step with eta > 0 (b200mix_ddim_eta_step, see include/b200mix.h): sb_p is the direction coefficient
    (1 - a_prev - std_dev_t^2)^0.5; noise fp32 like x, or None for Philox normals keyed by (seed, step). out may be x."""
    fp32, out = _step_tensors("ddim_eta_step", x, m_u, m_c, out, noise=noise)
    _launch("b200mix_ddim_eta_step", m_u, m_c, fp32, float(guidance), x, noise, out, x.numel(), float(sa_t), float(sb_t),
            float(sa_p), float(sb_p), float(std_dev_t), PRED_TYPES[prediction_type], float(clip_sample_range),
            1 if use_clipped_model_output else 0, int(seed) & 0xFFFFFFFFFFFFFFFF, int(step))
    return out


def dpmpp_2m_sde_step(eps_u, eps_c, guidance, x, noise, m_prev, m_out, sigma_cur, alpha_cur, A, B, halfB, inv_r0, N,
                      seed=0, step=0, out=None):
    """DPM-Solver++ 2M SDE update (b200mix_dpmpp_2m_sde_step, see include/b200mix.h); m_prev None = first-order step;
    m_out receives x0; noise fp32 like x, or None for Philox normals keyed by (seed, step). out may be x."""
    if m_out is None:
        raise ValueError("dpmpp_2m_sde_step: m_out (the x0 history entry) is required")
    fp32, out = _step_tensors("dpmpp_2m_sde_step", x, eps_u, eps_c, out, noise=noise, m_prev=m_prev, m_out=m_out)
    _launch("b200mix_dpmpp_2m_sde_step", eps_u, eps_c, fp32, float(guidance), x, noise, m_prev, out, m_out, x.numel(),
            float(sigma_cur), float(alpha_cur), float(A), float(B), float(halfB), float(inv_r0), float(N),
            int(seed) & 0xFFFFFFFFFFFFFFFF, int(step))
    return out


def euler_ancestral_step(m_u, m_c, guidance, x, noise, sigma, c_out, s2p1, dt, sigma_up, prediction_type="epsilon",
                         seed=0, step=0, out=None):
    """EulerAncestralDiscreteScheduler.step (b200mix_euler_ancestral_step, see include/b200mix.h): noise fp32 like x,
    or None for Philox normals keyed by (seed, step). out may be x itself."""
    if prediction_type not in ("epsilon", "v_prediction"):
        raise ValueError(f"euler_ancestral_step: prediction_type {prediction_type!r} must be epsilon or v_prediction")
    fp32, out = _step_tensors("euler_ancestral_step", x, m_u, m_c, out, noise=noise)
    _launch("b200mix_euler_ancestral_step", m_u, m_c, fp32, float(guidance), x, noise, out, x.numel(),
            PRED_TYPES[prediction_type], float(sigma), float(c_out), float(s2p1), float(dt), float(sigma_up),
            int(seed) & 0xFFFFFFFFFFFFFFFF, int(step))
    return out


def unipc_step(m_u, m_c, guidance, x, coeffs, m_out, x_corr, last_sample=None, m_prev=None, hist_c=(), hist_p=(),
               prediction_type="epsilon", out=None):
    """UniPCMultistepScheduler.step (b200mix_unipc_step, see include/b200mix.h). coeffs: dict of the fp32 scalars of
    `b200mix_unipc_coeffs` (rc / rk_c / rp / rk_p: one value per history term); last_sample and m_prev (both or neither)
    switch the corrector on; hist_c / hist_p: at most two x0 tensors each, most recent first. m_out receives x0 and
    x_corr the corrected sample. Every tensor but the model outputs is fp32 with x's element count."""
    hist_c, hist_p = list(hist_c), list(hist_p)
    if len(hist_c) > 2 or len(hist_p) > 2:
        raise ValueError("unipc_step: at most two history terms each for the corrector and the predictor (order <= 3)")
    if (last_sample is None) != (m_prev is None) or (hist_c and last_sample is None):
        raise ValueError("unipc_step: last_sample, m_prev and the corrector history go together")
    bufs = dict(m_out=m_out, x_corr=x_corr, last_sample=last_sample, m_prev=m_prev)
    bufs.update({f"corrector history {k}": t for k, t in enumerate(hist_c)})
    bufs.update({f"predictor history {k}": t for k, t in enumerate(hist_p)})
    if m_out is None or x_corr is None:
        raise ValueError("unipc_step: m_out and x_corr are required")
    fp32, out = _step_tensors("unipc_step", x, m_u, m_c, out, **bufs)
    k = _lib.UnipcCoeffs()
    for name in ("alpha_t", "sigma_t", "A_c", "K_c", "E_c", "rc_last", "A_p", "K_p", "E_p"):
        setattr(k, name, float(coeffs.get(name, 0.0)))
    for name in ("rc", "rk_c", "rp", "rk_p"):
        vals = [float(v) for v in coeffs.get(name, ())]
        getattr(k, name)[:len(vals)] = vals
    hc, hp = hist_c + [None] * (2 - len(hist_c)), hist_p + [None] * (2 - len(hist_p))
    _launch("b200mix_unipc_step", m_u, m_c, fp32, float(guidance), x, last_sample, m_prev, *hc, *hp, out, x_corr, m_out,
            x.numel(), PRED_TYPES[prediction_type], ctypes.byref(k))
    return out


def scale_model_input(x: torch.Tensor, denom: float, out=None) -> torch.Tensor:
    """EulerDiscreteScheduler.scale_model_input: x / denom in fp32 (IEEE division)."""
    c = _Args("scale_model_input")
    c("x", x, F32), c("out", out, F32, numel=x.numel())
    c.on_cuda()
    if out is None:
        out = torch.empty_like(x)
    _launch("b200mix_scale_model_input", x, out, x.numel(), float(denom))
    return out


def cast(x: torch.Tensor, dtype):
    c = _Args("cast")
    c("x", x, FLOAT)
    out = torch.empty_like(x, dtype=dtype)
    c("out", out, FLOAT)
    c.on_cuda()
    _launch("b200mix_cast", x, out, x.numel(), 1 if x.dtype == torch.float32 else 0, 1 if dtype == torch.float32 else 0)
    return out


def rope_inplace(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, rot_dim: Optional[int] = None):
    """x: bf16 [T, H, Dpad] view (last dim contiguous); cos/sin fp32 [T, rot_dim]."""
    c = _Args("rope_inplace")
    T, H, Dp = c("x", x, BF16, (None, None, None), STRIDED)
    D = rot_dim or Dp
    if D > Dp:
        raise ValueError(f"rope_inplace: rot_dim {D} is wider than the {Dp} channels of a head")
    c("cos", cos, F32, (T, D)), c("sin", sin, F32, (T, D))
    c.on_cuda()
    _launch("b200mix_rope_inplace", x, T, H, D, x.stride(0), x.stride(1), cos, sin)
    return x


def decode_rope_cache(qkv: torch.Tensor, heads: int, kv_heads: int, head_dim: int, cos: torch.Tensor, sin: torch.Tensor,
                      rows: torch.Tensor, cache_k: torch.Tensor, cache_v: torch.Tensor):
    """qkv bf16 [B, (heads + 2*kv_heads) * head_dim] of a single-token step: RoPE on the q heads in place, RoPE'd k heads and
    the v heads written into row rows[b] (int64, device) of the flattened caches [*, kv_heads * head_dim]."""
    c = _Args("decode_rope_cache")
    B = c("qkv", qkv, BF16, (None, (heads + 2 * kv_heads) * head_dim), ROWS)[0]
    c("cos", cos, F32, (B, head_dim)), c("sin", sin, F32, (B, head_dim)), c("rows", rows, I64, numel=B)
    c("cache_k", cache_k, BF16, (None, kv_heads * head_dim)), c("cache_v", cache_v, BF16, (None, kv_heads * head_dim))
    c.on_cuda()
    _launch("b200mix_decode_rope_cache", qkv, qkv.stride(0), B, heads, kv_heads, head_dim, cos, sin, rows, cache_k,
            cache_v)


def sample_tokens(logits: torch.Tensor, presence: torch.Tensor, finished: torch.Tensor, state: torch.Tensor,
                  out: torch.Tensor, next_ids: torch.Tensor, eos_ids: Optional[torch.Tensor] = None, pad_token_id=0, *,
                  do_sample=False, temperature=1.0, top_k=0, top_p=1.0, repetition_penalty=1.0, seed=0):
    """One generation step (b200mix_sample_tokens, see include/b200mix.h): logits fp32 [B, V] view with a contiguous
    vocabulary axis (any row stride: logits[:, -1] of prefill logits [B, S, V] is read in place); presence int32
    [B, ceil(V/32)] bitmap of the ids seen so far; finished int32 [B]; state int64 [4] (step, arrivals, all finished,
    step of the last finish; zero before the first step); out int64 [B, max_new]; next_ids int64 [B]; eos_ids int64
    [n] on the device or None. Every buffer except logits is updated on the device."""
    c = _Args("sample_tokens")
    B, V = c("logits", logits, F32, (None, None), STRIDED)
    c("presence", presence, I32, (B, (V + 31) // 32)), c("finished", finished, I32, numel=B)
    c("state", state, I64, numel=4), c("out", out, I64, (B, None), STRIDED), c("next_ids", next_ids, I64, numel=B)
    c("eos_ids", eos_ids, I64)
    c.on_cuda()
    with _Timed("sampling", 4.0 * B * V, "byte", lambda: f"sample {B}x{V}"):
        _launch("b200mix_sample_tokens", logits, logits.stride(0), B, V, presence, finished, state, out, out.stride(0),
                out.shape[1], next_ids, eos_ids, 0 if eos_ids is None else eos_ids.numel(), int(pad_token_id),
                1 if do_sample else 0, float(temperature), int(top_k), float(top_p), float(repetition_penalty),
                int(seed) & (2 ** 64 - 1))


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
    c = _Args("beam_search_step")
    rows, V = c("logits", logits, F32, (None, None), STRIDED)
    nb = int(num_beams)
    if rows % nb:
        raise ValueError(f"beam_search_step: logits must be [B * {nb}, V], got {tuple(logits.shape)}")
    B = rows // nb
    for name, t, dt, n in (("state", state, I64, 4), ("next_ids", next_ids, I64, rows),
                           ("beam_scores", beam_scores, F32, rows), ("hyp_score", hyp_score, (torch.float64,), rows),
                           ("hyp_step", hyp_step, I32, rows), ("hyp_slot", hyp_slot, I32, rows),
                           ("hyp_count", hyp_count, I32, B), ("hyp_worst", hyp_worst, (torch.float64,), B),
                           ("done", done, I32, B)):
        c(name, t, dt, numel=n)
    max_new = c("tokens", tokens, I64, (None, rows))[0]
    c("parents", parents, I32, (max_new, rows)), c("workspace", workspace, (torch.uint8,))
    c("presence", presence, I32, (2, rows, (V + 31) // 32))
    c.on_cuda()
    st = _lib.BeamState(*(t.data_ptr() for t in (state, next_ids, beam_scores, tokens, parents, hyp_score, hyp_step,
                                                 hyp_slot, hyp_count, hyp_worst, done)),
                        None if presence is None else presence.data_ptr())
    with _Timed("beam_search", 4.0 * rows * V, "byte", lambda: f"beam {B}x{nb}x{V}"):
        _launch("b200mix_beam_search_step", logits, logits.stride(0), B, nb, V, ctypes.byref(st), workspace,
                workspace.numel(), max_new, int(eos_token_id), int(pad_token_id), float(repetition_penalty),
                float(diversity_rate), float(length_penalty), 1 if early_stopping else 0, kernels=3)


def kv_reorder(layer_kv: torch.Tensor, cache_k, num_beams: int, prompt_len: int, parents: torch.Tensor,
               state: torch.Tensor, done: torch.Tensor):
    """b200mix_kv_reorder: layer_kv int64 [2 * L] device table of the K / V base pointers (K_0, V_0, K_1, ...) of caches
    shaped like cache_k (bf16 [B * nb, max_len, kv_heads, head_dim], contiguous); moves the generated positions
    [prompt_len, prompt_len + state[3]) from parent beam to child (parents int32 [max_new, B * nb], column state[0] - 1)
    for every item whose done flag is 0."""
    c = _Args("kv_reorder")
    rows, max_len = c("cache_k", cache_k, BF16, (None, None, ...))[:2]
    nb = int(num_beams)
    if rows % nb or layer_kv.numel() % 2:
        raise ValueError(f"kv_reorder: {rows} cache rows are not a multiple of {nb} beams, or layer_kv holds an odd "
                         f"number of caches")
    c("layer_kv", layer_kv, I64), c("parents", parents, I32, (None, rows)), c("state", state, I64, numel=4)
    c("done", done, I32, numel=rows // nb)
    c.on_cuda()
    _launch("b200mix_kv_reorder", layer_kv, layer_kv.numel() // 2, rows // nb, nb, max_len, cache_k[0, 0].numel(),
            int(prompt_len), parents.shape[0], parents, state, done)


def gather_rows(table: torch.Tensor, ids: torch.Tensor) -> torch.Tensor:
    """table bf16 [V, D], ids int64 [n] (device) -> bf16 [n, D]."""
    c = _Args("gather_rows")
    D = c("table", table, BF16, (None, None))[1]
    c("ids", ids, I64)
    c.on_cuda()
    out = torch.empty(ids.numel(), D, device=table.device, dtype=bf16)
    _launch("b200mix_gather_rows", table, ids, out, ids.numel(), D)
    return out


def scatter_rows(src: torch.Tensor, idx: torch.Tensor, dst: torch.Tensor) -> torch.Tensor:
    """dst[idx[i]] = src[i]; src bf16 [n, D], idx int64 [n] (device), dst bf16 [*, D] (in place)."""
    c = _Args("scatter_rows")
    n, D = c("src", src, BF16, (None, None))
    c("idx", idx, I64, numel=n), c("dst", dst, BF16, (None, D))
    c.on_cuda()
    _launch("b200mix_scatter_rows", src, idx, dst, n, D)
    return dst


def broadcast_add(x: torch.Tensor, table: torch.Tensor) -> torch.Tensor:
    """x fp32 [B, N], table fp32 [G, N] -> fp32 [B, G, N]."""
    c = _Args("broadcast_add")
    B, N = c("x", x, F32, (None, None))
    G = c("table", table, F32, (None, N))[0]
    c.on_cuda()
    out = torch.empty(B, G, N, device=x.device, dtype=torch.float32)
    _launch("b200mix_broadcast_add", x, table, out, B, G, N)
    return out


def head_rmsnorm_inplace(x: torch.Tensor, weight: torch.Tensor, d: int, eps: float = 1e-6) -> torch.Tensor:
    """x bf16 [rows, H, Dpad] view (last dim contiguous): RMSNorm over the first d channels of every head."""
    c = _Args("head_rmsnorm_inplace")
    rows, H, Dp = c("x", x, BF16, (None, None, None), STRIDED)
    if d > Dp:
        raise ValueError(f"head_rmsnorm_inplace: d = {d} is wider than the {Dp} channels of a head")
    c("weight", weight, F32, numel=d)
    c.on_cuda()
    _launch("b200mix_head_rmsnorm_inplace", x, rows, H, d, x.stride(0), x.stride(1), weight, float(eps))
    return x


def small_attention(qkv: torch.Tensor, B: int, T: int, S: int, H: int, d: int, *, scale: float, rope_cos=None,
                    rope_sin=None, q_norm_w=None, k_norm_w=None, eps: float = 1e-6, out=None) -> torch.Tensor:
    """qkv bf16 [B*T*S, 3*H*d] (row = (b*T+t)*S+s) -> bf16 [B*T*S, H*d]; attention along the T axis. qkv and out may
    be row-strided views (last dim contiguous)."""
    c = _Args("small_attention")
    rows = B * T * S
    for name, t, width in (("qkv", qkv, 3 * H * d), ("out", out, H * d)):
        if c(name, t, BF16, (rows, None), STRIDED) is not None and t.shape[1] < width:
            raise ValueError(f"small_attention: {name} has {t.shape[1]} columns, fewer than {width}")
    c("rope_cos", rope_cos, F32, (T, d // 2)), c("rope_sin", rope_sin, F32, (T, d // 2))
    c("q_norm_w", q_norm_w, F32, numel=d), c("k_norm_w", k_norm_w, F32, numel=d)
    c.on_cuda()
    if out is None:
        out = torch.empty(rows, H * d, device=qkv.device, dtype=bf16)
    with _Timed("small_attention", 2.0 * 2 * rows * 4 * H * d, "byte"):
        _launch("b200mix_small_attention", qkv, out, B, T, S, H, d, qkv.stride(0), out.stride(0), rope_cos, rope_sin,
                q_norm_w, k_norm_w, float(eps), float(scale))
    return out


def patchify3d(x: torch.Tensor, p: int) -> torch.Tensor:
    c = _Args("patchify3d")
    B, C, T, H, W = c("x", x, FLOAT, (None,) * 5)
    c.on_cuda()
    out = torch.empty(B, T * (H // p) * (W // p), C * p * p, device=x.device, dtype=bf16)
    _launch("b200mix_patchify3d", x, 1 if x.dtype == torch.float32 else 0, out, B, C, T, H, W, p)
    return out


def unpatchify3d(x: torch.Tensor, C: int, T: int, h: int, w: int, p: int) -> torch.Tensor:
    c = _Args("unpatchify3d")
    B = x.shape[0]
    c("x", x, BF16, numel=B * T * h * w * p * p * C)
    c.on_cuda()
    out = torch.empty(B, C, T, h * p, w * p, device=x.device, dtype=torch.float32)
    _launch("b200mix_unpatchify3d", x, out, B, C, T, h, w, p)
    return out
