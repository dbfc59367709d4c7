// Small HBM-/latency-bound kernels around the denoiser: timestep embedding, activation, nearest upsample, channel
// concat, NCHW<->NHWC, conv_in (tiny C_in), fused CFG + DDIM / flow-match Euler step, casts, rotary embedding.
// Reference call sites are cited per function in include/b200mix.h.
#include "common.cuh"
#include "ptx.cuh"

namespace b200 {

__device__ __forceinline__ float ew_act(float v, int act) {
  switch (act) {
    case B200MIX_ACT_SILU: return v / (1.0f + expf(-v));
    case B200MIX_ACT_GELU_ERF: return 0.5f * v * (1.0f + erff(v * 0.70710678118654752f));
    case B200MIX_ACT_GELU_TANH: {
      float u = 0.7978845608028654f * (v + 0.044715f * v * v * v);
      return 0.5f * v * (1.0f + tanhf(u));
    }
    case B200MIX_ACT_QUICK_GELU: return v / (1.0f + expf(-1.702f * v));
    default: return v;
  }
}

__device__ __forceinline__ float load_any(const void* p, long long i, int fp32) {
  return fp32 ? reinterpret_cast<const float*>(p)[i] : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[i]);
}

// embeddings.py:26-64 — exponent = -ln(max_period) * i / (half - shift); emb = scale * t * exp(exponent);
// [sin | cos], swapped to [cos | sin] when flip_sin_to_cos.
__global__ void timestep_embedding_kernel(const float* __restrict__ t, void* __restrict__ out, int out_fp32, int B,
                                          int dim, long long ld_out, long long col0, int flip, float shift, float scale,
                                          float max_period) {
  const int half = dim / 2;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * half) return;
  const int b = idx / half, i = idx % half;
  const float exponent = -logf(max_period) * static_cast<float>(i) / (static_cast<float>(half) - shift);
  const float arg = scale * (t[b] * expf(exponent));
  const float s = sinf(arg), c = cosf(arg);
  const long long base = b * ld_out + col0;
  const long long i_sin = flip ? half + i : i;
  const long long i_cos = flip ? i : half + i;
  if (out_fp32) {
    float* o = reinterpret_cast<float*>(out);
    o[base + i_sin] = s;
    o[base + i_cos] = c;
    if ((dim & 1) && i == 0) o[base + dim - 1] = 0.0f;
  } else {
    __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(out);
    o[base + i_sin] = __float2bfloat16(s);
    o[base + i_cos] = __float2bfloat16(c);
    if ((dim & 1) && i == 0) o[base + dim - 1] = __float2bfloat16(0.0f);
  }
}

__global__ void activation_kernel(const void* __restrict__ x, void* __restrict__ y, long long n, int act, int x_fp32,
                                  int y_fp32) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float v = x_fp32 ? reinterpret_cast<const float*>(x)[i]
                     : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(x)[i]);
    v = ew_act(v, act);
    if (y_fp32) reinterpret_cast<float*>(y)[i] = v;
    else reinterpret_cast<__nv_bfloat16*>(y)[i] = __float2bfloat16(v);
  }
}

// y[b, 2h+dy, 2w+dx, :] = x[b, h, w, :]; one thread per 16-byte channel vector of an OUTPUT pixel (coalesced writes).
__global__ void upsample2x_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, long long total, int H, int W,
                                  int CV) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(i % CV);
    long long pix = i / CV;
    const int ow = (int)(pix % (2 * W));
    pix /= (2 * W);
    const int oh = (int)(pix % (2 * H));
    const long long b = pix / (2 * H);
    y[i] = __ldg(x + ((b * H + (oh >> 1)) * W + (ow >> 1)) * CV + cv);
  }
}

__global__ void concat_channels_kernel(const uint4* __restrict__ x1, int CV1, const uint4* __restrict__ x2, int CV2,
                                       uint4* __restrict__ y, long long total) {
  const int CV = CV1 + CV2;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(i % CV);
    const long long row = i / CV;
    y[i] = cv < CV1 ? __ldg(x1 + row * CV1 + cv) : __ldg(x2 + row * CV2 + (cv - CV1));
  }
}

__global__ void nchw_to_nhwc_kernel(const void* __restrict__ x, int x_fp32, __nv_bfloat16* __restrict__ y, int B, int C,
                                    int H, int W) {
  const long long total = (long long)B * C * H * W;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    long long r = i / C;
    const int w = (int)(r % W);
    r /= W;
    const int h = (int)(r % H);
    const long long b = r / H;
    const long long src = ((b * C + c) * H + h) * W + w;
    float v = x_fp32 ? reinterpret_cast<const float*>(x)[src]
                     : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(x)[src]);
    y[i] = __float2bfloat16(v);
  }
}

__global__ void nhwc_to_nchw_kernel(const __nv_bfloat16* __restrict__ x, void* __restrict__ y, int y_fp32, int B, int C,
                                    int H, int W) {
  const long long total = (long long)B * C * H * W;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int w = (int)(i % W);
    long long r = i / W;
    const int h = (int)(r % H);
    r /= H;
    const int c = (int)(r % C);
    const long long b = r / C;
    const float v = __bfloat162float(x[((b * H + h) * W + w) * C + c]);
    if (y_fp32) reinterpret_cast<float*>(y)[i] = v;
    else reinterpret_cast<__nv_bfloat16*>(y)[i] = __float2bfloat16(v);
  }
}

// y = a + r on an NHWC bf16 activation, r either NHWC (bf16) or NCHW (fp32 | bf16): the ControlNet / T2I-Adapter
// residuals of UNet2DConditionModel.forward (unet_2d_condition.py:1109-1155) arrive in the caller's NCHW layout.
__global__ void add_residual_nhwc_kernel(const __nv_bfloat16* __restrict__ a, const void* __restrict__ r, int r_fp32,
                                         int r_nchw, __nv_bfloat16* __restrict__ y, int B, int C, int H, int W) {
  const long long total = (long long)B * C * H * W;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    long long src = i;
    if (r_nchw) {
      const int c = (int)(i % C);
      long long q = i / C;
      const int w = (int)(q % W);
      q /= W;
      const int h = (int)(q % H);
      const long long b = q / H;
      src = ((b * C + c) * H + h) * W + w;
    }
    const float rv = r_fp32 ? reinterpret_cast<const float*>(r)[src]
                            : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(r)[src]);
    y[i] = __float2bfloat16(__bfloat162float(a[i]) + rv);
  }
}

// conv_in with Cin == 4 (SD / SDXL latents): one thread = one output pixel. Its 3x3x4 input patch is read once into
// registers (bf16-rounded, zero outside the image) and reused for every output channel; the filter bank sits in shared
// memory as fp32 [36][Cout] and is read as warp-wide broadcasts (all lanes want the same 8 output channels), so the
// kernel runs at the FP32 FMA rate: 8 x 128 x 128 x 320 in ~60 us instead of 1.4 ms for the generic kernel below.
// Same accumulation order as the generic kernel (taps outside the image contribute fma(0, w, acc) == acc).
__global__ void __launch_bounds__(256) conv3x3_cin4_kernel(const void* __restrict__ x, int x_fp32,
                                                           const __nv_bfloat16* __restrict__ w,
                                                           const float* __restrict__ bias, __nv_bfloat16* __restrict__ y,
                                                           int B, int H, int W, int Cout) {
  extern __shared__ float sw[];  // [36][Cout] then bias [Cout]
  float* sb = sw + 36 * Cout;
  for (int i = threadIdx.x; i < 36 * Cout; i += blockDim.x) {
    const int co = i / 36, k = i - co * 36;  // w is [Cout][36]
    sw[k * Cout + co] = __bfloat162float(w[i]);
  }
  for (int i = threadIdx.x; i < Cout; i += blockDim.x) sb[i] = bias ? bias[i] : 0.0f;
  __syncthreads();
  const long long npix = static_cast<long long>(B) * H * W;
  for (long long pix = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; pix < npix;
       pix += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int ow = static_cast<int>(pix % W);
    const int oh = static_cast<int>((pix / W) % H);
    const long long b = pix / (static_cast<long long>(W) * H);
    float xr[36];
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int ih = oh + t / 3 - 1, iw = ow + t % 3 - 1;
      float4 v = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
      if (ih >= 0 && ih < H && iw >= 0 && iw < W) {
        const long long src = ((b * H + ih) * W + iw) * 4;
        if (x_fp32) {
          const float4 f = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(x) + src);
          // rounded to bf16 first: the tensor-core path of every other conv sees bf16 activations
          v = make_float4(__bfloat162float(__float2bfloat16(f.x)), __bfloat162float(__float2bfloat16(f.y)),
                          __bfloat162float(__float2bfloat16(f.z)), __bfloat162float(__float2bfloat16(f.w)));
        } else {
          const uint2 u = *reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(x) + src);
          v = make_float4(bf16_lo(u.x), bf16_hi(u.x), bf16_lo(u.y), bf16_hi(u.y));
        }
      }
      xr[4 * t + 0] = v.x, xr[4 * t + 1] = v.y, xr[4 * t + 2] = v.z, xr[4 * t + 3] = v.w;
    }
    __nv_bfloat16* dst = y + pix * Cout;
#pragma unroll 1
    for (int g = 0; g < (Cout >> 3); ++g) {
      const float4 b0 = *reinterpret_cast<const float4*>(sb + g * 8), b1 = *reinterpret_cast<const float4*>(sb + g * 8 + 4);
      float acc[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int k = 0; k < 36; ++k) {
        const float4 w0 = *reinterpret_cast<const float4*>(sw + k * Cout + g * 8);
        const float4 w1 = *reinterpret_cast<const float4*>(sw + k * Cout + g * 8 + 4);
        acc[0] = fmaf(xr[k], w0.x, acc[0]), acc[1] = fmaf(xr[k], w0.y, acc[1]);
        acc[2] = fmaf(xr[k], w0.z, acc[2]), acc[3] = fmaf(xr[k], w0.w, acc[3]);
        acc[4] = fmaf(xr[k], w1.x, acc[4]), acc[5] = fmaf(xr[k], w1.y, acc[5]);
        acc[6] = fmaf(xr[k], w1.z, acc[6]), acc[7] = fmaf(xr[k], w1.w, acc[7]);
      }
      *reinterpret_cast<uint4*>(dst + g * 8) = make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]),
                                                           pack_bf16x2(acc[4], acc[5]), pack_bf16x2(acc[6], acc[7]));
    }
  }
}

// conv_in: Cin <= 8. Thread = (pixel, 8 output channels); weights staged in smem as fp32 [9*Cin][Cout].
__global__ void conv3x3_small_cin_kernel(const void* __restrict__ x, int x_fp32, const __nv_bfloat16* __restrict__ w,
                                         const float* __restrict__ bias, __nv_bfloat16* __restrict__ y, int B, int H,
                                         int W, int Cin, int Cout) {
  extern __shared__ float sw[];  // [9*Cin][Cout]
  const int K = 9 * Cin;
  for (int i = threadIdx.x; i < K * Cout; i += blockDim.x) {
    const int co = i / K, k = i % K;  // w is [Cout][9*Cin]
    sw[k * Cout + co] = __bfloat162float(w[i]);
  }
  __syncthreads();
  const int CV = Cout >> 3;
  const long long total = (long long)B * H * W * CV;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(i % CV);
    long long pix = i / CV;
    const int ow = (int)(pix % W);
    const int oh = (int)((pix / W) % H);
    const long long b = pix / ((long long)W * H);
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = bias ? bias[cv * 8 + j] : 0.0f;
    for (int kh = 0; kh < 3; ++kh) {
      const int ih = oh + kh - 1;
      if (ih < 0 || ih >= H) continue;
      for (int kw = 0; kw < 3; ++kw) {
        const int iw = ow + kw - 1;
        if (iw < 0 || iw >= W) continue;
        const long long src = ((b * H + ih) * W + iw) * Cin;
        for (int c = 0; c < Cin; ++c) {
          // inputs are rounded to bf16 first: the tensor-core path of every other conv sees bf16 activations
          float xv = x_fp32 ? __bfloat162float(__float2bfloat16(reinterpret_cast<const float*>(x)[src + c]))
                            : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(x)[src + c]);
          const float* wr = sw + ((kh * 3 + kw) * Cin + c) * Cout + cv * 8;
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] = fmaf(xv, wr[j], acc[j]);
        }
      }
    }
    uint4 o = make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]), pack_bf16x2(acc[4], acc[5]),
                         pack_bf16x2(acc[6], acc[7]));
    *reinterpret_cast<uint4*>(y + pix * Cout + cv * 8) = o;
  }
}


// scheduling_ddim.py:410-457 with eta = 0, epsilon prediction, no clipping; every operation individually rounded
// (no FMA contraction) so the result is bit-identical to the fp32 CPU evaluation of the same expression.
__global__ void ddim_step_kernel(const void* __restrict__ eps_u, const void* __restrict__ eps_c, int eps_fp32,
                                 float guidance, const float* __restrict__ x, float* __restrict__ x_prev, long long n,
                                 float sa_t, float sb_t, float sa_p, float sb_p) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float e = load_any(eps_u, i, eps_fp32);
    if (eps_c) {
      const float ec = load_any(eps_c, i, eps_fp32);
      e = __fadd_rn(e, __fmul_rn(guidance, __fsub_rn(ec, e)));
    }
    const float x0 = __fdiv_rn(__fsub_rn(x[i], __fmul_rn(sb_t, e)), sa_t);
    x_prev[i] = __fadd_rn(__fmul_rn(sa_p, x0), __fmul_rn(sb_p, e));
  }
}

// DDIM step for every prediction type (scheduling_ddim.py:424-443) with optional clipping of the predicted x0
// (:446-452), eta = 0; same operation order as the reference, every operation rounded individually.
//   epsilon      x0 = (x - sb_t*m) / sa_t            eps = m
//   sample       x0 = m                               eps = (x - sa_t*x0) / sb_t
//   v_prediction x0 = sa_t*x - sb_t*m                 eps = sa_t*m + sb_t*x
//   x_prev = sa_p * clip(x0) + sb_p * eps            (use_clipped_model_output = False: eps is NOT re-derived)
__global__ void ddim_step_ex_kernel(const void* __restrict__ m_u, const void* __restrict__ m_c, int m_fp32, float guidance,
                                    const float* __restrict__ x, float* __restrict__ x_prev, long long n, float sa_t,
                                    float sb_t, float sa_p, float sb_p, int pred_type, float clip) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float m = load_any(m_u, i, m_fp32);
    if (m_c) {
      const float mc = load_any(m_c, i, m_fp32);
      m = __fadd_rn(m, __fmul_rn(guidance, __fsub_rn(mc, m)));
    }
    const float xi = x[i];
    float x0, e;
    if (pred_type == 0) {
      x0 = __fdiv_rn(__fsub_rn(xi, __fmul_rn(sb_t, m)), sa_t);
      e = m;
    } else if (pred_type == 1) {
      x0 = m;
      e = __fdiv_rn(__fsub_rn(xi, __fmul_rn(sa_t, x0)), sb_t);
    } else {
      x0 = __fsub_rn(__fmul_rn(sa_t, xi), __fmul_rn(sb_t, m));
      e = __fadd_rn(__fmul_rn(sa_t, m), __fmul_rn(sb_t, xi));
    }
    if (clip > 0.0f) x0 = fminf(fmaxf(x0, -clip), clip);
    x_prev[i] = __fadd_rn(__fmul_rn(sa_p, x0), __fmul_rn(sb_p, e));
  }
}

// LCMScheduler.step (scheduling_lcm.py:468-545): x0 from the model output (as above), optional clip,
// denoised = c_out*x0 + c_skip*x, then x_prev = sa_p*denoised + sb_p*noise (multi-step; the noise tensor is the
// caller's randn) or x_prev = denoised on the final step (noise == NULL).
__global__ void lcm_step_kernel(const void* __restrict__ m_u, const void* __restrict__ m_c, int m_fp32, float guidance,
                                const float* __restrict__ x, const float* __restrict__ noise, float* __restrict__ x_prev,
                                float* __restrict__ denoised_out, long long n, float sa_t, float sb_t, float c_skip,
                                float c_out, float sa_p, float sb_p, int pred_type, float clip) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float m = load_any(m_u, i, m_fp32);
    if (m_c) {
      const float mc = load_any(m_c, i, m_fp32);
      m = __fadd_rn(m, __fmul_rn(guidance, __fsub_rn(mc, m)));
    }
    const float xi = x[i];
    float x0;
    if (pred_type == 0) x0 = __fdiv_rn(__fsub_rn(xi, __fmul_rn(sb_t, m)), sa_t);
    else if (pred_type == 1) x0 = m;
    else x0 = __fsub_rn(__fmul_rn(sa_t, xi), __fmul_rn(sb_t, m));
    if (clip > 0.0f) x0 = fminf(fmaxf(x0, -clip), clip);
    const float den = __fadd_rn(__fmul_rn(c_out, x0), __fmul_rn(c_skip, xi));
    if (denoised_out) denoised_out[i] = den;
    x_prev[i] = noise ? __fadd_rn(__fmul_rn(sa_p, den), __fmul_rn(sb_p, noise[i])) : den;
  }
}

// rescale_noise_cfg (pipeline_stable_diffusion.py:69-80; SDXL pipeline_stable_diffusion_xl.py:1061-1067), first half:
// per sample b, ratio[b] = std(noise_pred_text[b]) / std(noise_cfg[b]) over all non-batch axes (unbiased std, Paddle's
// default), with noise_cfg = u + g*(c - u). One CTA per sample, double accumulators, fixed reduction order.
__global__ void __launch_bounds__(256) cfg_rescale_ratio_kernel(const void* __restrict__ e_u, const void* __restrict__ e_c,
                                                               int fp32, float guidance, float* __restrict__ ratio,
                                                               long long nps) {
  __shared__ double sh[4][256];
  const long long base = static_cast<long long>(blockIdx.x) * nps;
  double st = 0.0, qt = 0.0, sc = 0.0, qc = 0.0;
  for (long long i = threadIdx.x; i < nps; i += blockDim.x) {
    const float u = load_any(e_u, base + i, fp32), c = load_any(e_c, base + i, fp32);
    const float cfg = __fadd_rn(u, __fmul_rn(guidance, __fsub_rn(c, u)));
    st += c, qt += (double)c * c, sc += cfg, qc += (double)cfg * cfg;
  }
  sh[0][threadIdx.x] = st, sh[1][threadIdx.x] = qt, sh[2][threadIdx.x] = sc, sh[3][threadIdx.x] = qc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o)
      for (int k = 0; k < 4; ++k) sh[k][threadIdx.x] += sh[k][threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double n = (double)nps;
    const double vt = (sh[1][0] - sh[0][0] * sh[0][0] / n) / (n - 1.0);
    const double vc = (sh[3][0] - sh[2][0] * sh[2][0] / n) / (n - 1.0);
    ratio[blockIdx.x] = (float)(sqrt(vt > 0.0 ? vt : 0.0) / sqrt(vc > 0.0 ? vc : 0.0));
  }
}

// second half: out = u + g*(c - u), then (ratio given) out = gr * (out * ratio[b]) + (1 - gr) * out   (fp32 output)
__global__ void cfg_combine_kernel(const void* __restrict__ e_u, const void* __restrict__ e_c, int fp32, float guidance,
                                   const float* __restrict__ ratio, float gr, long long nps, float* __restrict__ out,
                                   long long n) {
  const float one_minus = __fsub_rn(1.0f, gr);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float u = load_any(e_u, i, fp32), c = load_any(e_c, i, fp32);
    float cfg = __fadd_rn(u, __fmul_rn(guidance, __fsub_rn(c, u)));
    if (ratio) {
      const float resc = __fmul_rn(cfg, __ldg(ratio + i / nps));
      cfg = __fadd_rn(__fmul_rn(gr, resc), __fmul_rn(one_minus, cfg));
    }
    out[i] = cfg;
  }
}

// EulerDiscreteScheduler.scale_model_input (scheduling_euler_discrete.py:218-241): sample / ((sigma^2 + 1) ** 0.5), the
// denominator computed on the host in fp32; an IEEE division here, like the reference's tensor / 0-d tensor.
__global__ void scale_model_input_kernel(const float* __restrict__ x, float* __restrict__ y, long long n, float denom) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = __fdiv_rn(x[i], denom);
}

__global__ void euler_step_kernel(const void* __restrict__ v_u, const void* __restrict__ v_c, int v_fp32, float guidance,
                                  const float* __restrict__ x, float* __restrict__ x_prev, long long n, float sigma,
                                  float dt) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float v = load_any(v_u, i, v_fp32);
    if (v_c) {
      const float vc = load_any(v_c, i, v_fp32);
      v = __fadd_rn(v, __fmul_rn(guidance, __fsub_rn(vc, v)));
    }
    // scheduling_flow_match_euler_discrete.py:262-270: denoised = x - v*sigma; derivative = (x - denoised)/sigma_hat
    const float xi = x[i];
    const float den = __fsub_rn(xi, __fmul_rn(v, sigma));
    const float der = __fdiv_rn(__fsub_rn(xi, den), sigma);
    x_prev[i] = __fadd_rn(xi, __fmul_rn(der, dt));
  }
}

__global__ void cast_kernel(const void* __restrict__ x, void* __restrict__ y, long long n, int x_fp32, int y_fp32) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = load_any(x, i, x_fp32);
    if (y_fp32) reinterpret_cast<float*>(y)[i] = v;
    else reinterpret_cast<__nv_bfloat16*>(y)[i] = __float2bfloat16(v);
  }
}

// rotate_half RoPE in place, fp32 math: o[i] = x[i]*cos[i] - x[i+D/2]*sin[i]; o[i+D/2] = x[i+D/2]*cos[i+D/2] + x[i]*sin[i+D/2]
__global__ void rope_kernel(__nv_bfloat16* __restrict__ x, long long T, int H, int D, long long ld_tok, long long ld_head,
                            const float* __restrict__ cs, const float* __restrict__ sn) {
  const int half = D >> 1;
  const long long total = T * H * half;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(idx % half);
    const int h = (int)((idx / half) % H);
    const long long t = idx / ((long long)half * H);
    __nv_bfloat16* p = x + t * ld_tok + h * ld_head;
    const float x1 = __bfloat162float(p[i]), x2 = __bfloat162float(p[i + half]);
    const float c1 = cs[t * D + i], c2 = cs[t * D + i + half];
    const float s1 = sn[t * D + i], s2 = sn[t * D + i + half];
    p[i] = __float2bfloat16(x1 * c1 - x2 * s1);
    p[i + half] = __float2bfloat16(x2 * c2 + x1 * s2);
  }
}

// Decode-step glue in one launch (was: RoPE(q), RoPE(k), two staging copies, two cache scatters): for every sequence b of
// a single-token step, rotate the q heads of the fused qkv row in place, rotate the k heads INTO the cache row rows[b],
// copy the v heads into the cache row. grid (heads + 2 * kv_heads, B); same fp32 expression as rope_kernel.
__global__ void decode_rope_cache_kernel(__nv_bfloat16* __restrict__ qkv, long long ld_row, int nh, int nkv, int D,
                                         const float* __restrict__ cs, const float* __restrict__ sn,
                                         const long long* __restrict__ rows, __nv_bfloat16* __restrict__ cache_k,
                                         __nv_bfloat16* __restrict__ cache_v) {
  const int b = blockIdx.y, hh = blockIdx.x, half = D >> 1;
  const long long kvd = (long long)nkv * D;
  __nv_bfloat16* src = qkv + b * ld_row + (long long)hh * D;  // q heads, then k heads, then v heads, all D wide
  if (hh >= nh + nkv) {
    __nv_bfloat16* dst = cache_v + rows[b] * kvd + (long long)(hh - nh - nkv) * D;
    for (int i = threadIdx.x; i < D / 8; i += blockDim.x)
      reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(src)[i];
    return;
  }
  __nv_bfloat16* dst = hh < nh ? src : cache_k + rows[b] * kvd + (long long)(hh - nh) * D;
  const float* c = cs + (long long)b * D;
  const float* s = sn + (long long)b * D;
  for (int i = threadIdx.x; i < half; i += blockDim.x) {
    const float x1 = __bfloat162float(src[i]), x2 = __bfloat162float(src[i + half]);
    dst[i] = __float2bfloat16(x1 * c[i] - x2 * s[i]);
    dst[i + half] = __float2bfloat16(x2 * c[i + half] + x1 * s[i + half]);
  }
}

__global__ void patchify_kernel(const void* __restrict__ x, int x_fp32, __nv_bfloat16* __restrict__ y, int B, int C,
                                int H, int W, int p) {
  const int h = H / p, w = W / p, K = C * p * p;
  const long long total = (long long)B * h * w * K;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(i % K);
    long long r = i / K;
    const int pw = k % p, ph = (k / p) % p, c = k / (p * p);
    const int ww = (int)(r % w);
    r /= w;
    const int hh = (int)(r % h);
    const long long b = r / h;
    const long long src = ((b * C + c) * H + hh * p + ph) * W + ww * p + pw;
    y[i] = __float2bfloat16(load_any(x, src, x_fp32));
  }
}

__global__ void unpatchify_kernel(const __nv_bfloat16* __restrict__ x, void* __restrict__ y, int y_fp32, int B, int C,
                                  int h, int w, int p) {
  const int H = h * p, W = w * p;
  const long long total = (long long)B * C * H * W;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int X = (int)(i % W);
    long long r = i / W;
    const int Y = (int)(r % H);
    r /= H;
    const int c = (int)(r % C);
    const long long b = r / C;
    const int hh = Y / p, ph = Y % p, ww = X / p, pw = X % p;
    const float v = __bfloat162float(x[((b * h + hh) * w + ww) * (long long)(p * p * C) + (ph * p + pw) * C + c]);
    if (y_fp32) reinterpret_cast<float*>(y)[i] = v;
    else reinterpret_cast<__nv_bfloat16*>(y)[i] = __float2bfloat16(v);
  }
}

// out[i, :] = table[ids[i], :]   (nn.Embedding lookup, modeling_qwen2_vl.py:1443) — 16-byte vectors
__global__ void gather_rows_kernel(const uint4* __restrict__ table, const long long* __restrict__ ids,
                                   uint4* __restrict__ out, long long n, int DV) {
  const long long total = n * DV;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / DV;
    out[i] = __ldg(table + ids[r] * DV + (i - r * DV));
  }
}
// dst[idx[i], :] = src[i, :]   (inputs_embeds[image_mask] = image_embeds, modeling_qwen2_vl.py:1449-1452)
__global__ void scatter_rows_kernel(const uint4* __restrict__ src, const long long* __restrict__ idx,
                                    uint4* __restrict__ dst, long long n, int DV) {
  const long long total = n * DV;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / DV;
    dst[idx[r] * DV + (i - r * DV)] = __ldg(src + i);
  }
}

static inline unsigned ew_grid(long long n, int threads) {
  long long g = (n + threads - 1) / threads;
  const long long cap = (long long)num_sms() * 16;
  return (unsigned)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace b200

using namespace b200;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int b200mix_timestep_embedding(const float* t, void* out, int32_t out_fp32, int64_t B, int64_t dim,
                                          int64_t ld_out, int64_t col0, int32_t flip_sin_to_cos,
                                          float downscale_freq_shift, float scale, float max_period, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(t && out && B > 0 && dim >= 2, "timestep_embedding: bad arguments");
  const int half = (int)(dim / 2);
  const long long n = B * half;
  timestep_embedding_kernel<<<(unsigned)((n + 127) / 128), 128, 0, ST(stream)>>>(
      t, out, out_fp32, (int)B, (int)dim, ld_out, col0, flip_sin_to_cos, downscale_freq_shift, scale, max_period);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_activation(const void* x, void* y, int64_t n, int32_t act, int32_t x_fp32, int32_t y_fp32,
                                  void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(x && y && n > 0, "activation: bad arguments");
  activation_kernel<<<ew_grid(n, 256), 256, 0, ST(stream)>>>(x, y, n, act, x_fp32, y_fp32);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_upsample_nearest2x_nhwc(const void* x, void* y, int64_t B, int64_t H, int64_t W, int64_t C,
                                               void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(x && y && C % 8 == 0, "upsample: C must be a multiple of 8");
  const long long total = B * 4 * H * W * (C / 8);
  upsample2x_kernel<<<ew_grid(total, 256), 256, 0, ST(stream)>>>(reinterpret_cast<const uint4*>(x),
                                                                 reinterpret_cast<uint4*>(y), total, (int)H, (int)W,
                                                                 (int)(C / 8));
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_concat_channels(const void* x1, int64_t C1, const void* x2, int64_t C2, void* y, int64_t rows,
                                       void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(x1 && x2 && y && C1 % 8 == 0 && C2 % 8 == 0, "concat: channel counts must be multiples of 8");
  const long long total = rows * ((C1 + C2) / 8);
  concat_channels_kernel<<<ew_grid(total, 256), 256, 0, ST(stream)>>>(
      reinterpret_cast<const uint4*>(x1), (int)(C1 / 8), reinterpret_cast<const uint4*>(x2), (int)(C2 / 8),
      reinterpret_cast<uint4*>(y), total);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_nchw_to_nhwc(const void* x, int32_t x_fp32, void* y, int64_t B, int64_t C, int64_t H, int64_t W,
                                    void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(x && y, "nchw_to_nhwc: null pointer");
  nchw_to_nhwc_kernel<<<ew_grid(B * C * H * W, 256), 256, 0, ST(stream)>>>(x, x_fp32,
                                                                           reinterpret_cast<__nv_bfloat16*>(y), (int)B,
                                                                           (int)C, (int)H, (int)W);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_add_residual_nhwc(const void* a, const void* r, int32_t r_fp32, int32_t r_nchw, void* y, int64_t B,
                                         int64_t C, int64_t H, int64_t W, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(a && r && y && B > 0 && C > 0 && H > 0 && W > 0, "add_residual_nhwc: bad arguments");
  add_residual_nhwc_kernel<<<ew_grid(B * C * H * W, 256), 256, 0, ST(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(a), r, r_fp32, r_nchw, reinterpret_cast<__nv_bfloat16*>(y), (int)B, (int)C,
      (int)H, (int)W);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_nhwc_to_nchw(const void* x, void* y, int32_t y_fp32, int64_t B, int64_t C, int64_t H, int64_t W,
                                    void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(x && y, "nhwc_to_nchw: null pointer");
  nhwc_to_nchw_kernel<<<ew_grid(B * C * H * W, 256), 256, 0, ST(stream)>>>(reinterpret_cast<const __nv_bfloat16*>(x),
                                                                           y, y_fp32, (int)B, (int)C, (int)H, (int)W);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_conv3x3_small_cin(const void* x, int32_t x_fp32, const void* w, const float* bias, void* y,
                                         int64_t B, int64_t H, int64_t W, int64_t Cin, int64_t Cout, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(x && w && y, "conv3x3_small_cin: null pointer");
  B200_CHECK_ARG(Cin >= 1 && Cin <= 16 && Cout % 8 == 0, "conv3x3_small_cin: Cin in [1,16], Cout %% 8 == 0");
  const size_t smem = (size_t)9 * Cin * Cout * sizeof(float);
  B200_CHECK_ARG(smem <= 200 * 1024, "conv3x3_small_cin: weights do not fit shared memory");
  static bool configured = false;
  if (!configured) {
    B200_CUDA(cudaFuncSetAttribute(conv3x3_small_cin_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    configured = true;
  }
  if (Cin == 4 && (9 * 4 + 1) * Cout * sizeof(float) <= 200 * 1024 && reinterpret_cast<uintptr_t>(x) % 16 == 0) {
    static bool configured4 = false;
    if (!configured4) {
      B200_CUDA(cudaFuncSetAttribute(conv3x3_cin4_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
      configured4 = true;
    }
    const size_t smem4 = (size_t)(36 + 1) * Cout * sizeof(float);
    unsigned grid4 = ew_grid(B * H * W, 256);
    if (grid4 > 4u * (unsigned)num_sms()) grid4 = 4u * (unsigned)num_sms();
    conv3x3_cin4_kernel<<<grid4, 256, smem4, ST(stream)>>>(x, x_fp32, reinterpret_cast<const __nv_bfloat16*>(w), bias,
                                                          reinterpret_cast<__nv_bfloat16*>(y), (int)B, (int)H, (int)W,
                                                          (int)Cout);
    B200_LAUNCH_CHECK();
    return 0;
  }
  const long long total = B * H * W * (Cout / 8);
  // every block first stages the whole filter bank in shared memory: keep the grid at ~2 blocks per SM
  unsigned grid = ew_grid(total, 256);
  if (grid > 2u * (unsigned)num_sms()) grid = 2u * (unsigned)num_sms();
  conv3x3_small_cin_kernel<<<grid, 256, smem, ST(stream)>>>(
      x, x_fp32, reinterpret_cast<const __nv_bfloat16*>(w), bias, reinterpret_cast<__nv_bfloat16*>(y), (int)B, (int)H,
      (int)W, (int)Cin, (int)Cout);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_ddim_step(const void* eps_u, const void* eps_c, int32_t eps_fp32, float guidance, const float* x,
                                 float* x_prev, int64_t n, float sqrt_alpha_t, float sqrt_beta_t,
                                 float sqrt_alpha_prev, float sqrt_beta_prev, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(eps_u && x && x_prev && n > 0, "ddim_step: bad arguments");
  ddim_step_kernel<<<ew_grid(n, 256), 256, 0, ST(stream)>>>(eps_u, eps_c, eps_fp32, guidance, x, x_prev, n,
                                                           sqrt_alpha_t, sqrt_beta_t, sqrt_alpha_prev, sqrt_beta_prev);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_ddim_step_ex(const void* m_u, const void* m_c, int32_t m_fp32, float guidance, const float* x,
                                    float* x_prev, int64_t n, float sqrt_alpha_t, float sqrt_beta_t,
                                    float sqrt_alpha_prev, float sqrt_beta_prev, int32_t prediction_type,
                                    float clip_sample_range, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(m_u && x && x_prev && n > 0, "ddim_step_ex: bad arguments");
  B200_CHECK_ARG(prediction_type >= 0 && prediction_type <= 2, "ddim_step_ex: prediction_type must be 0 (epsilon), 1 "
                 "(sample) or 2 (v_prediction)");
  ddim_step_ex_kernel<<<ew_grid(n, 256), 256, 0, ST(stream)>>>(m_u, m_c, m_fp32, guidance, x, x_prev, n, sqrt_alpha_t,
                                                              sqrt_beta_t, sqrt_alpha_prev, sqrt_beta_prev,
                                                              prediction_type, clip_sample_range);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_lcm_step(const void* m_u, const void* m_c, int32_t m_fp32, float guidance, const float* x,
                                const float* noise, float* x_prev, float* denoised, int64_t n, float sqrt_alpha_t,
                                float sqrt_beta_t, float c_skip, float c_out, float sqrt_alpha_prev, float sqrt_beta_prev,
                                int32_t prediction_type, float clip_sample_range, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(m_u && x && x_prev && n > 0, "lcm_step: bad arguments");
  B200_CHECK_ARG(prediction_type >= 0 && prediction_type <= 2, "lcm_step: prediction_type must be 0, 1 or 2");
  lcm_step_kernel<<<ew_grid(n, 256), 256, 0, ST(stream)>>>(m_u, m_c, m_fp32, guidance, x, noise, x_prev, denoised, n,
                                                          sqrt_alpha_t, sqrt_beta_t, c_skip, c_out, sqrt_alpha_prev,
                                                          sqrt_beta_prev, prediction_type, clip_sample_range);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_cfg_rescale_ratio(const void* eps_u, const void* eps_c, int32_t eps_fp32, float guidance,
                                         float* ratio, int64_t B, int64_t n_per_sample, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(eps_u && eps_c && ratio && B > 0 && n_per_sample > 1, "cfg_rescale_ratio: bad arguments");
  cfg_rescale_ratio_kernel<<<(unsigned)B, 256, 0, ST(stream)>>>(eps_u, eps_c, eps_fp32, guidance, ratio, n_per_sample);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_cfg_combine(const void* eps_u, const void* eps_c, int32_t eps_fp32, float guidance,
                                   const float* ratio, float guidance_rescale, int64_t n_per_sample, float* out, int64_t n,
                                   void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(eps_u && eps_c && out && n > 0 && n_per_sample > 0, "cfg_combine: bad arguments");
  cfg_combine_kernel<<<ew_grid(n, 256), 256, 0, ST(stream)>>>(eps_u, eps_c, eps_fp32, guidance, ratio, guidance_rescale,
                                                             n_per_sample, out, n);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_euler_step(const void* v_u, const void* v_c, int32_t v_fp32, float guidance, const float* x,
                                  float* x_prev, int64_t n, float sigma, float dt, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(v_u && x && x_prev && n > 0, "euler_step: bad arguments");
  euler_step_kernel<<<ew_grid(n, 256), 256, 0, ST(stream)>>>(v_u, v_c, v_fp32, guidance, x, x_prev, n, sigma, dt);
  B200_LAUNCH_CHECK();
  return 0;
}

// DPM-Solver++ (2M) step, scheduling_dpmsolver_multistep.py:446-453 (x0 from epsilon), :548-553 (first order) and
// :633-640 (second order, midpoint), every operation individually rounded in the reference's order.
__global__ void dpmpp_2m_step_kernel(const void* __restrict__ eps_u, const void* __restrict__ eps_c, int eps_fp32,
                                     float guidance, const float* __restrict__ x, const float* __restrict__ m_prev,
                                     float* __restrict__ x_next, float* __restrict__ m_out, long long n, float sigma_cur,
                                     float alpha_cur, float A, float C, float halfC, float inv_r0) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float e = load_any(eps_u, i, eps_fp32);
    if (eps_c) {
      const float ec = load_any(eps_c, i, eps_fp32);
      e = __fadd_rn(e, __fmul_rn(guidance, __fsub_rn(ec, e)));
    }
    const float xv = x[i];
    const float m0 = __fdiv_rn(__fsub_rn(xv, __fmul_rn(sigma_cur, e)), alpha_cur);
    float r = __fsub_rn(__fmul_rn(A, xv), __fmul_rn(C, m0));
    if (m_prev) {
      const float d1 = __fmul_rn(inv_r0, __fsub_rn(m0, m_prev[i]));
      r = __fsub_rn(r, __fmul_rn(halfC, d1));
    }
    m_out[i] = m0;
    x_next[i] = r;
  }
}

extern "C" int b200mix_dpmpp_2m_step(const void* eps_u, const void* eps_c, int32_t eps_fp32, float guidance, const float* x,
                                     const float* m_prev, float* x_next, float* m_out, int64_t n, float sigma_cur,
                                     float alpha_cur, float A, float C, float halfC, float inv_r0, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(eps_u && x && x_next && m_out && n > 0 && alpha_cur != 0.0f, "dpmpp_2m_step: bad arguments");
  dpmpp_2m_step_kernel<<<ew_grid(n, 256), 256, 0, ST(stream)>>>(eps_u, eps_c, eps_fp32, guidance, x, m_prev, x_next, m_out, n,
                                                               sigma_cur, alpha_cur, A, C, halfC, inv_r0);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_scale_model_input(const float* x, float* y, int64_t n, float denom, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(x && y && n > 0 && denom > 0.0f, "scale_model_input: bad arguments");
  scale_model_input_kernel<<<ew_grid(n, 256), 256, 0, ST(stream)>>>(x, y, n, denom);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_patchify(const void* x, int32_t x_fp32, void* y, int64_t B, int64_t C, int64_t H, int64_t W,
                                int32_t p, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(x && y && p > 0 && H % p == 0 && W % p == 0, "patchify: bad arguments");
  patchify_kernel<<<ew_grid(B * C * H * W, 256), 256, 0, ST(stream)>>>(x, x_fp32, reinterpret_cast<__nv_bfloat16*>(y),
                                                                       (int)B, (int)C, (int)H, (int)W, p);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_unpatchify(const void* x, void* y, int32_t y_fp32, int64_t B, int64_t C, int64_t h, int64_t w,
                                  int32_t p, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(x && y && p > 0, "unpatchify: bad arguments");
  unpatchify_kernel<<<ew_grid(B * C * h * w * p * p, 256), 256, 0, ST(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), y, y_fp32, (int)B, (int)C, (int)h, (int)w, p);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_gather_rows(const void* table, const int64_t* ids, void* out, int64_t n, int64_t dim,
                                   void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(table && ids && out && n > 0 && dim % 8 == 0, "gather_rows: bad arguments (dim %% 8 == 0)");
  gather_rows_kernel<<<ew_grid(n * (dim / 8), 256), 256, 0, ST(stream)>>>(
      reinterpret_cast<const uint4*>(table), reinterpret_cast<const long long*>(ids), reinterpret_cast<uint4*>(out), n,
      (int)(dim / 8));
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_scatter_rows(const void* src, const int64_t* idx, void* dst, int64_t n, int64_t dim,
                                    void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(src && idx && dst && n > 0 && dim % 8 == 0, "scatter_rows: bad arguments (dim %% 8 == 0)");
  scatter_rows_kernel<<<ew_grid(n * (dim / 8), 256), 256, 0, ST(stream)>>>(
      reinterpret_cast<const uint4*>(src), reinterpret_cast<const long long*>(idx), reinterpret_cast<uint4*>(dst), n,
      (int)(dim / 8));
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_cast(const void* x, void* y, int64_t n, int32_t x_fp32, int32_t y_fp32, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(x && y && n > 0, "cast: bad arguments");
  cast_kernel<<<ew_grid(n, 256), 256, 0, ST(stream)>>>(x, y, n, x_fp32, y_fp32);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_rope_inplace(void* x, int64_t T, int64_t H, int64_t D, int64_t ld_tok, int64_t ld_head,
                                    const float* cos, const float* sin, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(x && cos && sin && D % 2 == 0, "rope: bad arguments");
  rope_kernel<<<ew_grid(T * H * (D / 2), 256), 256, 0, ST(stream)>>>(reinterpret_cast<__nv_bfloat16*>(x), T, (int)H,
                                                                     (int)D, ld_tok, ld_head, cos, sin);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_decode_rope_cache(void* qkv, int64_t ld_row, int64_t B, int64_t heads, int64_t kv_heads, int64_t D,
                                         const float* cos, const float* sin, const int64_t* rows, void* cache_k,
                                         void* cache_v, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(qkv && cos && sin && rows && cache_k && cache_v, "decode_rope_cache: null pointer");
  B200_CHECK_ARG(B > 0 && heads > 0 && kv_heads > 0 && D % 8 == 0 && ld_row % 8 == 0 && B < 65536,
                 "decode_rope_cache: bad shape (head_dim and the row stride must be multiples of 8)");
  static_assert(sizeof(long long) == sizeof(int64_t), "int64 layout");
  decode_rope_cache_kernel<<<dim3((unsigned)(heads + 2 * kv_heads), (unsigned)B), 64, 0, ST(stream)>>>(
      reinterpret_cast<__nv_bfloat16*>(qkv), ld_row, (int)heads, (int)kv_heads, (int)D, cos, sin,
      reinterpret_cast<const long long*>(rows), reinterpret_cast<__nv_bfloat16*>(cache_k),
      reinterpret_cast<__nv_bfloat16*>(cache_v));
  B200_LAUNCH_CHECK();
  return 0;
}

// ================================================================================================================
// STDiT2 helpers (Open-Sora): short-sequence temporal attention, per-head RMSNorm, table broadcast, 3-D (un)patchify
// ================================================================================================================
namespace b200 {

// out[b, g, n] = x[b, n] + table[g, n]   (scale_shift_table[None] + t.reshape(B, 6, C), stdit2.py:121-126)
__global__ void broadcast_add_kernel(const float* __restrict__ x, const float* __restrict__ table,
                                     float* __restrict__ out, int B, int G, int N) {
  const long long total = (long long)B * G * N;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(i % N);
    const long long r = i / N;
    const int g = (int)(r % G);
    const long long b = r / G;
    out[i] = x[b * N + n] + table[(long long)g * N + n];
  }
}

// In-place RMSNorm over the first d channels of every head (LlamaRMSNorm as q_norm / k_norm, blocks.py:62-68,214):
// one warp per (row, head).
__global__ void head_rmsnorm_kernel(__nv_bfloat16* __restrict__ x, long long rows, int H, int d, long long ld_row,
                                    long long ld_head, const float* __restrict__ w, float eps) {
  const int lane = threadIdx.x & 31;
  const long long wid = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  if (wid >= rows * H) return;
  const long long r = wid / H;
  const int h = (int)(wid % H);
  __nv_bfloat16* p = x + r * ld_row + h * ld_head;
  float v[4];
  float ss = 0.0f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = lane + 32 * i;
    v[i] = c < d ? __bfloat162float(p[c]) : 0.0f;
    ss += v[i] * v[i];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float rs = rsqrtf(ss / d + eps);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = lane + 32 * i;
    // hidden_states.to(input_dtype) then * weight (blocks.py:67-68)
    if (c < d) p[c] = __float2bfloat16(__bfloat162float(__float2bfloat16(v[i] * rs)) * w[c]);
  }
}

// Temporal self-attention of STDiT2 (stdit2.py:160-171): sequences of length T <= 32 taken along the frame axis of a
// token-major [B, T, S, 3, H, d] qkv buffer (row = (b*T + t)*S + s), with interleaved-pair RoPE (blocks.py:566-591)
// and optional q/k RMSNorm applied in the reference order (rope, then norm). One CTA (128 threads) per (b, s, head):
// the work per sequence (16x16x72) is far below one tensor-core tile, so this is a plain fp32 CUDA-core kernel bound
// by the qkv / output traffic.
__global__ void __launch_bounds__(128) small_attention_kernel(
    const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out, int T, int S, int H, int d,
    long long ld_row, long long ld_out, const float* __restrict__ rope_cos, const float* __restrict__ rope_sin,
    const float* __restrict__ qw, const float* __restrict__ kw, float eps, float scale) {
  extern __shared__ float sm[];  // q[T][d] k[T][d] v[T][d] p[T][T]
  float* sq = sm;
  float* sk = sq + T * d;
  float* sv = sk + T * d;
  float* sp = sv + T * d;
  const int h = blockIdx.x % H;
  const long long bs = blockIdx.x / H;  // b*S + s
  const long long b = bs / S, s = bs % S;
  const int tid = threadIdx.x;
  const int half = d >> 1;
  // load with RoPE on pairs (2i, 2i+1)
  for (int idx = tid; idx < T * half; idx += blockDim.x) {
    const int t = idx / half, i = idx % half;
    const __nv_bfloat16* row = qkv + ((b * T + t) * S + s) * ld_row + h * d;
    const __nv_bfloat162 q2 = *reinterpret_cast<const __nv_bfloat162*>(row + 2 * i);
    const __nv_bfloat162 k2 = *reinterpret_cast<const __nv_bfloat162*>(row + (long long)H * d + 2 * i);
    const __nv_bfloat162 v2 = *reinterpret_cast<const __nv_bfloat162*>(row + 2LL * H * d + 2 * i);
    float q0 = __low2float(q2), q1 = __high2float(q2), k0 = __low2float(k2), k1 = __high2float(k2);
    if (rope_cos) {
      const float c = rope_cos[t * half + i], sn = rope_sin[t * half + i];
      const float a0 = q0 * c - q1 * sn, a1 = q1 * c + q0 * sn;
      const float b0 = k0 * c - k1 * sn, b1 = k1 * c + k0 * sn;
      // apply_rotary_emb runs with autocast off but returns the input dtype: round to bf16 like the reference
      q0 = __bfloat162float(__float2bfloat16(a0)), q1 = __bfloat162float(__float2bfloat16(a1));
      k0 = __bfloat162float(__float2bfloat16(b0)), k1 = __bfloat162float(__float2bfloat16(b1));
    }
    sq[t * d + 2 * i] = q0, sq[t * d + 2 * i + 1] = q1;
    sk[t * d + 2 * i] = k0, sk[t * d + 2 * i + 1] = k1;
    sv[t * d + 2 * i] = __low2float(v2), sv[t * d + 2 * i + 1] = __high2float(v2);
  }
  __syncthreads();
  if (qw) {  // q_norm / k_norm: one warp per row, rows 0..T-1 = q, T..2T-1 = k
    const int warp = tid >> 5, lane = tid & 31;
    for (int r = warp; r < 2 * T; r += (blockDim.x >> 5)) {
      float* rowp = (r < T ? sq + r * d : sk + (r - T) * d);
      const float* w = r < T ? qw : kw;
      float ss = 0.0f;
      for (int c = lane; c < d; c += 32) ss += rowp[c] * rowp[c];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
      const float rs = rsqrtf(ss / d + eps);
      for (int c = lane; c < d; c += 32) rowp[c] = __bfloat162float(__float2bfloat16(rowp[c] * rs)) * w[c];
    }
    __syncthreads();
  }
  for (int idx = tid; idx < T * T; idx += blockDim.x) {
    const int i = idx / T, j = idx % T;
    float acc = 0.0f;
    for (int c = 0; c < d; ++c) acc = fmaf(sq[i * d + c], sk[j * d + c], acc);
    sp[idx] = acc * scale;
  }
  __syncthreads();
  if (tid < T) {  // softmax of row tid
    float m = -INFINITY;
    for (int j = 0; j < T; ++j) m = fmaxf(m, sp[tid * T + j]);
    float l = 0.0f;
    for (int j = 0; j < T; ++j) {
      const float e = __expf(sp[tid * T + j] - m);
      sp[tid * T + j] = e;
      l += e;
    }
    const float inv = 1.0f / l;
    for (int j = 0; j < T; ++j) sp[tid * T + j] *= inv;
  }
  __syncthreads();
  for (int idx = tid; idx < T * half; idx += blockDim.x) {
    const int t = idx / half, i = idx % half;
    float o0 = 0.0f, o1 = 0.0f;
    for (int j = 0; j < T; ++j) {
      const float pj = sp[t * T + j];
      o0 = fmaf(pj, sv[j * d + 2 * i], o0);
      o1 = fmaf(pj, sv[j * d + 2 * i + 1], o1);
    }
    __nv_bfloat16* orow = out + ((b * T + t) * S + s) * ld_out + h * d;
    *reinterpret_cast<__nv_bfloat162*>(orow + 2 * i) = __floats2bfloat162_rn(o0, o1);
  }
}

// x NCTHW (fp32|bf16) -> rows [B*T*(H/p)*(W/p), C*p*p] bf16, column order (c, ph, pw): PatchEmbed3D with patch
// (1, p, p) (blocks.py:94-164); and the inverse head: rows [B*T*h*w, p*p*C] in (ph, pw, c) order -> [B,C,T,h*p,w*p].
__global__ void patchify3d_kernel(const void* __restrict__ x, int x_fp32, __nv_bfloat16* __restrict__ y, int B, int C,
                                  int T, int H, int W, int p) {
  const int h = H / p, w = W / p, K = C * p * p;
  const long long total = (long long)B * T * h * w * K;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(i % K);
    long long r = i / K;
    const int pw = k % p, ph = (k / p) % p, c = k / (p * p);
    const int ww = (int)(r % w);
    r /= w;
    const int hh = (int)(r % h);
    r /= h;
    const int t = (int)(r % T);
    const long long b = r / T;
    const long long src = (((b * C + c) * T + t) * H + hh * p + ph) * W + ww * p + pw;
    y[i] = __float2bfloat16(load_any(x, src, x_fp32));
  }
}
__global__ void unpatchify3d_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ y, int B, int C, int T,
                                    int h, int w, int p) {
  const int H = h * p, W = w * p;
  const long long total = (long long)B * C * T * H * W;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int X = (int)(i % W);
    long long r = i / W;
    const int Y = (int)(r % H);
    r /= H;
    const int t = (int)(r % T);
    r /= T;
    const int c = (int)(r % C);
    const long long b = r / C;
    const int hh = Y / p, ph = Y % p, ww = X / p, pw = X % p;
    y[i] = __bfloat162float(x[(((b * T + t) * h + hh) * w + ww) * (long long)(p * p * C) + (ph * p + pw) * C + c]);
  }
}

}  // namespace b200

extern "C" int b200mix_broadcast_add(const float* x, const float* table, float* out, int64_t B, int64_t G, int64_t N,
                                     void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(x && table && out && B > 0 && G > 0 && N > 0, "broadcast_add: bad arguments");
  broadcast_add_kernel<<<ew_grid(B * G * N, 256), 256, 0, ST(stream)>>>(x, table, out, (int)B, (int)G, (int)N);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_head_rmsnorm_inplace(void* x, int64_t rows, int64_t H, int64_t d, int64_t ld_row, int64_t ld_head,
                                            const float* weight, float eps, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(x && weight && d > 0 && d <= 128, "head_rmsnorm: d must be in (0, 128]");
  const long long warps = rows * H;
  head_rmsnorm_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, ST(stream)>>>(
      reinterpret_cast<__nv_bfloat16*>(x), rows, (int)H, (int)d, ld_row, ld_head, weight, eps);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_small_attention(const void* qkv, void* out, int64_t B, int64_t T, int64_t S, int64_t H, int64_t d,
                                       int64_t ld_row, int64_t ld_out, const float* rope_cos, const float* rope_sin,
                                       const float* q_norm_w, const float* k_norm_w, float eps, float scale,
                                       void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(qkv && out, "small_attention: null pointer");
  B200_CHECK_ARG(T > 0 && T <= 32 && d > 0 && d <= 128 && d % 2 == 0, "small_attention: T <= 32, even d <= 128");
  B200_CHECK_ARG((rope_cos == nullptr) == (rope_sin == nullptr) && (q_norm_w == nullptr) == (k_norm_w == nullptr),
                 "small_attention: rope / norm tables come in pairs");
  const size_t smem = (size_t)(3 * T * d + T * T) * sizeof(float);
  const long long ctas = B * S * H;
  B200_CHECK_ARG(ctas < (1ll << 31), "small_attention: too many sequences");
  small_attention_kernel<<<(unsigned)ctas, 128, smem, ST(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(qkv), reinterpret_cast<__nv_bfloat16*>(out), (int)T, (int)S, (int)H, (int)d,
      ld_row, ld_out, rope_cos, rope_sin, q_norm_w, k_norm_w, eps, scale);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_patchify3d(const void* x, int32_t x_fp32, void* y, int64_t B, int64_t C, int64_t T, int64_t H,
                                  int64_t W, int32_t p, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(x && y && p > 0 && H % p == 0 && W % p == 0, "patchify3d: bad arguments");
  patchify3d_kernel<<<ew_grid(B * C * T * H * W, 256), 256, 0, ST(stream)>>>(
      x, x_fp32, reinterpret_cast<__nv_bfloat16*>(y), (int)B, (int)C, (int)T, (int)H, (int)W, p);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_unpatchify3d(const void* x, float* y, int64_t B, int64_t C, int64_t T, int64_t h, int64_t w,
                                    int32_t p, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(x && y && p > 0, "unpatchify3d: bad arguments");
  unpatchify3d_kernel<<<ew_grid(B * C * T * h * w * p * p, 256), 256, 0, ST(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), y, (int)B, (int)C, (int)T, (int)h, (int)w, p);
  B200_LAUNCH_CHECK();
  return 0;
}

