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


def linear(a: torch.Tensor, w: torch.Tensor, bias=None, *, act=ACT_NONE, glu=GLU_NONE, residual=None, row_add=None,
           row_gate=None, rows_per_group=0, out_fp32=False, out=None, out_scale=1.0, residual_row_mod=0, stats=False,
           ln=None):
    """out[M, N(/2)] = epilogue(a[M, K] @ w[N, K]^T). a: bf16 [..., K] (last dim contiguous), w: bf16 [N, K].
    stats=True or a ZEROED int64 [M, 2] tensor (RowStats.arena): also returns the RowStats of the output rows
    (-> (out, RowStats)); ln=(RowStats of a's rows, colsum, eps[, rms]): a is the UN-normalised tensor and w / bias carry
    the folded affine (fold_layernorm_into_linear)."""
    _req(a, bf16, "a"), _req(w, bf16, "w")
    K = a.shape[-1]
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
    assert a.stride(-1) == 1 and out.stride(-1) == 1 and out.shape[0] == B and out.shape[1] == rows
    mod = row_add if row_add is not None else row_gate
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


def ddim_step(eps_u, eps_c, guidance, x, sa_t, sb_t, sa_p, sb_p, out=None):
    _req(x, torch.float32, "x")
    if out is None:
        out = torch.empty_like(x)
    check(lib.b200mix_ddim_step(_p(eps_u), _p(eps_c), 1 if eps_u.dtype == torch.float32 else 0, float(guidance), _p(x),
                                _p(out), x.numel(), float(sa_t), float(sb_t), float(sa_p), float(sb_p), _stream()),
          "b200mix_ddim_step")
    _count()
    return out


PRED_TYPES = {"epsilon": 0, "sample": 1, "v_prediction": 2}


def ddim_step_ex(m_u, m_c, guidance, x, sa_t, sb_t, sa_p, sb_p, prediction_type="epsilon", clip_sample_range=0.0, out=None):
    """DDIM step for any prediction_type, optional x0 clipping (clip_sample_range > 0), fused CFG combine."""
    _req(x, torch.float32, "x")
    if out is None:
        out = torch.empty_like(x)
    check(lib.b200mix_ddim_step_ex(_p(m_u), _p(m_c), 1 if m_u.dtype == torch.float32 else 0, float(guidance), _p(x), _p(out),
                                   x.numel(), float(sa_t), float(sb_t), float(sa_p), float(sb_p),
                                   PRED_TYPES[prediction_type], float(clip_sample_range), _stream()), "b200mix_ddim_step_ex")
    _count()
    return out


def lcm_step(m_u, m_c, guidance, x, noise, sa_t, sb_t, c_skip, c_out, sa_p, sb_p, prediction_type="epsilon",
             clip_sample_range=0.0, out=None, denoised=None):
    """LCMScheduler.step; noise None = final step (x_prev = denoised)."""
    _req(x, torch.float32, "x")
    if noise is not None:
        _req(noise, torch.float32, "noise")
    if out is None:
        out = torch.empty_like(x)
    check(lib.b200mix_lcm_step(_p(m_u), _p(m_c), 1 if m_u.dtype == torch.float32 else 0, float(guidance), _p(x), _p(noise),
                               _p(out), _p(denoised), x.numel(), float(sa_t), float(sb_t), float(c_skip), float(c_out),
                               float(sa_p), float(sb_p), PRED_TYPES[prediction_type], float(clip_sample_range), _stream()),
          "b200mix_lcm_step")
    _count()
    return out


def cfg_combine(eps_u, eps_c, guidance, guidance_rescale=0.0, out=None):
    """noise_pred_uncond + g * (noise_pred_text - noise_pred_uncond), then rescale_noise_cfg when guidance_rescale > 0
    (pipeline_stable_diffusion.py:69-80, :882-888). eps_*: [B, ...] bf16 / fp32 contiguous. Returns fp32."""
    assert eps_u.shape == eps_c.shape and eps_u.dtype == eps_c.dtype and eps_u.is_contiguous() and eps_c.is_contiguous()
    B = eps_u.shape[0]
    nps = eps_u.numel() // B
    fp32 = 1 if eps_u.dtype == torch.float32 else 0
    if out is None:
        out = torch.empty(eps_u.shape, device=eps_u.device, dtype=torch.float32)
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
    _req(x, torch.float32, "x")
    if out is None:
        out = torch.empty_like(x)
    check(lib.b200mix_euler_step(_p(v_u), _p(v_c), 1 if v_u.dtype == torch.float32 else 0, float(guidance), _p(x),
                                 _p(out), x.numel(), float(sigma), float(dt), _stream()), "b200mix_euler_step")
    _count()
    return out


def dpmpp_2m_step(eps_u, eps_c, guidance, x, m_prev, m_out, sigma_cur, alpha_cur, A, C, halfC, inv_r0, out=None):
    """DPM-Solver++ 2M update (see include/b200mix.h); m_prev None = first-order step; m_out receives x0."""
    _req(x, torch.float32, "x"), _req(m_out, torch.float32, "m_out")
    if out is None:
        out = torch.empty_like(x)
    check(lib.b200mix_dpmpp_2m_step(_p(eps_u), _p(eps_c), 1 if eps_u.dtype == torch.float32 else 0, float(guidance), _p(x),
                                    _p(m_prev), _p(out), _p(m_out), x.numel(), float(sigma_cur), float(alpha_cur), float(A),
                                    float(C), float(halfC), float(inv_r0), _stream()), "b200mix_dpmpp_2m_step")
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
                    rope_sin=None, q_norm_w=None, k_norm_w=None, eps: float = 1e-6) -> torch.Tensor:
    """qkv bf16 [B*T*S, 3*H*d] (row = (b*T+t)*S+s) -> bf16 [B*T*S, H*d]; attention along the T axis."""
    _req(qkv, bf16, "qkv")
    out = torch.empty(qkv.shape[0], H * d, device=qkv.device, dtype=bf16)
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
