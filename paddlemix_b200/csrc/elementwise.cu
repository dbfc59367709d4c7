// Small HBM-/latency-bound kernels around the denoiser: timestep embedding, activation, nearest upsample, channel
// concat, NCHW<->NHWC, conv_in (tiny C_in), fused CFG + DDIM / LCM / Euler / Euler-ancestral / DPM-Solver++ / UniPC /
// IDDPM step, casts, rotary embedding.
// Reference call sites are cited per function in include/b200mix.h.
#include "common.cuh"
#include "philox.cuh"
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
    case B200MIX_ACT_RELU: return v < 0.0f ? 0.0f : v;  // NaN passes through, as in max(x, 0) on the host
    default: return v;
  }
}

__device__ __forceinline__ float load_any(const void* p, long long i, int fp32) {
  return fp32 ? reinterpret_cast<const float*>(p)[i] : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[i]);
}

// Classifier-free guidance, u + g*(c - u) (pipeline_stable_diffusion.py:882-884), every operation rounded on its own
// so that every sampler step matches the fp32 CPU evaluation of the same expression bit for bit.
__device__ __forceinline__ float cfg_mix(float u, float c, float g) {
  return __fadd_rn(u, __fmul_rn(g, __fsub_rn(c, u)));
}

// Element i of the model output, guided: m_c == NULL means no guidance (the output is m_u itself).
__device__ __forceinline__ float load_guided(const void* m_u, const void* m_c, long long i, int fp32, float g) {
  const float u = load_any(m_u, i, fp32);
  return m_c ? cfg_mix(u, load_any(m_c, i, fp32), g) : u;
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


// x0 and eps from the model output m for each prediction_type (scheduling_ddim.py:424-443, scheduling_lcm.py:530-535),
// in the reference's operation order:
//   epsilon      x0 = (x - sb_t*m) / sa_t            eps = m
//   sample       x0 = m                               eps = (x - sa_t*x0) / sb_t
//   v_prediction x0 = sa_t*x - sb_t*m                 eps = sa_t*m + sb_t*x
__device__ __forceinline__ void predict_x0_eps(int pred_type, float m, float x, float sa_t, float sb_t, float& x0,
                                               float& eps) {
  if (pred_type == 0) {
    x0 = __fdiv_rn(__fsub_rn(x, __fmul_rn(sb_t, m)), sa_t);
    eps = m;
  } else if (pred_type == 1) {
    x0 = m;
    eps = __fdiv_rn(__fsub_rn(x, __fmul_rn(sa_t, x0)), sb_t);
  } else {
    x0 = __fsub_rn(__fmul_rn(sa_t, x), __fmul_rn(sb_t, m));
    eps = __fadd_rn(__fmul_rn(sa_t, m), __fmul_rn(sb_t, x));
  }
}

// DDIM step (scheduling_ddim.py:410-457), eta = 0, with optional clipping of the predicted x0 (:446-452):
//   x_prev = sa_p * clip(x0) + sb_p * eps            (use_clipped_model_output = False: eps is NOT re-derived)
__global__ void ddim_step_ex_kernel(const void* __restrict__ m_u, const void* __restrict__ m_c, int m_fp32, float guidance,
                                    const float* __restrict__ x, float* __restrict__ x_prev, long long n, float sa_t,
                                    float sb_t, float sa_p, float sb_p, int pred_type, float clip) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float x0, e;
    predict_x0_eps(pred_type, load_guided(m_u, m_c, i, m_fp32, guidance), x[i], sa_t, sb_t, x0, e);
    if (clip > 0.0f) x0 = fminf(fmaxf(x0, -clip), clip);
    x_prev[i] = __fadd_rn(__fmul_rn(sa_p, x0), __fmul_rn(sb_p, e));
  }
}

// LCMScheduler.step (scheduling_lcm.py:468-545): x0 from the model output (as above; eps unused), optional clip,
// denoised = c_out*x0 + c_skip*x, then x_prev = sa_p*denoised + sb_p*noise (multi-step; the noise tensor is the
// caller's randn) or x_prev = denoised on the final step (noise == NULL).
__global__ void lcm_step_kernel(const void* __restrict__ m_u, const void* __restrict__ m_c, int m_fp32, float guidance,
                                const float* __restrict__ x, const float* __restrict__ noise, float* __restrict__ x_prev,
                                float* __restrict__ denoised_out, long long n, float sa_t, float sb_t, float c_skip,
                                float c_out, float sa_p, float sb_p, int pred_type, float clip) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float xi = x[i];
    float x0, unused;
    predict_x0_eps(pred_type, load_guided(m_u, m_c, i, m_fp32, guidance), xi, sa_t, sb_t, x0, unused);
    if (clip > 0.0f) x0 = fminf(fmaxf(x0, -clip), clip);
    const float den = __fadd_rn(__fmul_rn(c_out, x0), __fmul_rn(c_skip, xi));
    if (denoised_out) denoised_out[i] = den;
    x_prev[i] = noise ? __fadd_rn(__fmul_rn(sa_p, den), __fmul_rn(sb_p, noise[i])) : den;
  }
}

// Open-Sora IDDPM p_sample with learned-range variance (gaussian_diffusion.py:278-372, 409-485) behind forward_with_cfg
// (schedulers/iddpm/__init__.py:97-114). One thread per group of 4 consecutive state elements, which is one Philox
// call (philox_normal4). Output channel k of the 2C model channels is guided when k < cfg_channel; the rest are read
// from the conditional rows [0, B). Every operation is rounded on its own, in the reference's order; exp is the fp32
// rounding of the fp64 exp.
struct IddpmArgs {
  const void* m;           // [2B, 2C, N], conditional rows first
  const float* x;          // [B, C, N]; may alias x_prev
  const float* noise;      // [B, C, N] or NULL (Philox)
  float* x_prev;           // [B, C, N]
  float* x_dup;            // optional second copy of x_prev (the unconditional half of the model input)
  long long B, C, N;
  int m_fp32, cfg_channel, add_noise;
  float cfg_scale, sqrt_recip, sqrt_recipm1, coef1, coef2, max_log, min_log;
  unsigned long long seed;
  uint32_t step;
};

__global__ void __launch_bounds__(256) iddpm_step_kernel(IddpmArgs a) {
  pdl_wait();
  pdl_launch_dependents();
  const long long n = a.B * a.C * a.N, CN = a.C * a.N;
  const long long groups = (n + 3) >> 2;
  for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < groups; g += (long long)gridDim.x * blockDim.x) {
    float z[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    if (a.add_noise && !a.noise) philox_normal4(a.seed, a.step, (unsigned long long)g, z);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const long long i = 4 * g + k;
      if (i >= n) break;
      const long long b = i / CN, r = i - b * CN;
      const long long c = r / a.N, j = r - c * a.N;
      const long long ec = (b * 2 * a.C + c) * a.N + j;          // eps channel c, conditional row b
      const long long vc = ec + CN;                                // variance channel C + c
      const long long off_u = a.B * 2 * CN;                        // unconditional row B + b
      float e = load_any(a.m, ec, a.m_fp32);
      if (c < a.cfg_channel) e = cfg_mix(load_any(a.m, ec + off_u, a.m_fp32), e, a.cfg_scale);
      float v = load_any(a.m, vc, a.m_fp32);
      if (a.C + c < a.cfg_channel) v = cfg_mix(load_any(a.m, vc + off_u, a.m_fp32), v, a.cfg_scale);
      const float xi = a.x[i];
      const float frac = __fdiv_rn(__fadd_rn(v, 1.0f), 2.0f);
      const float logvar = __fadd_rn(__fmul_rn(frac, a.max_log), __fmul_rn(__fsub_rn(1.0f, frac), a.min_log));
      const float x0 = __fsub_rn(__fmul_rn(a.sqrt_recip, xi), __fmul_rn(a.sqrt_recipm1, e));
      float out = __fadd_rn(__fmul_rn(a.coef1, x0), __fmul_rn(a.coef2, xi));
      if (a.add_noise) {
        const float sd = (float)exp((double)__fmul_rn(0.5f, logvar));
        out = __fadd_rn(out, __fmul_rn(sd, a.noise ? a.noise[i] : z[k]));
      }
      a.x_prev[i] = out;
      if (a.x_dup) a.x_dup[i] = out;
    }
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
    const float cfg = cfg_mix(u, c, guidance);
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
    float cfg = cfg_mix(u, c, guidance);
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

// The deterministic Euler update shared by b200mix_euler_step and b200mix_euler_ancestral_step
// (scheduling_flow_match_euler_discrete.py:262-270, scheduling_euler_discrete.py:433-463,
// scheduling_euler_ancestral_discrete.py:327-349), one rounding per operation in this order:
//   v_pred == 0 (epsilon / flow):  x0 = x - m*sigma
//   v_pred != 0:                   x0 = m*c_out + x/s2p1     (c_out = -sigma/(sigma^2+1)^0.5, s2p1 = sigma^2+1: host fp32)
//   d = (x - x0)/sigma;  returns x + d*dt
__device__ __forceinline__ float euler_update(int v_pred, float m, float x, float sigma, float c_out, float s2p1,
                                              float dt) {
  const float x0 = v_pred ? __fadd_rn(__fmul_rn(m, c_out), __fdiv_rn(x, s2p1)) : __fsub_rn(x, __fmul_rn(m, sigma));
  const float d = __fdiv_rn(__fsub_rn(x, x0), sigma);
  return __fadd_rn(x, __fmul_rn(d, dt));
}

__global__ void euler_step_kernel(const void* __restrict__ v_u, const void* __restrict__ v_c, int v_fp32, float guidance,
                                  const float* __restrict__ x, float* __restrict__ x_prev, long long n, float sigma,
                                  float dt) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    x_prev[i] = euler_update(0, load_guided(v_u, v_c, i, v_fp32, guidance), x[i], sigma, 0.0f, 1.0f, dt);
}

// EulerAncestralDiscreteScheduler.step: euler_update with dt = sigma_down - sigma, then + z*sigma_up. One thread per
// group of 4 consecutive elements, which is one Philox call (philox_normal4) when noise is NULL. x_prev may alias x.
// The minimum of 4 CTAs per SM gives ptxas the registers to keep the fp64 Box-Muller out of local memory.
__global__ void __launch_bounds__(256, 4) euler_ancestral_step_kernel(
    const void* __restrict__ m_u, const void* __restrict__ m_c, int m_fp32, float guidance, const float* x,
    const float* __restrict__ noise, float* x_prev, long long n, int v_pred, float sigma, float c_out, float s2p1,
    float dt, float sigma_up, unsigned long long seed, uint32_t step) {
  const long long groups = (n + 3) >> 2;
  for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < groups; g += (long long)gridDim.x * blockDim.x) {
    float z[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    if (!noise) philox_normal4(seed, step, (unsigned long long)g, z);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const long long i = 4 * g + k;
      if (i >= n) break;
      const float xp = euler_update(v_pred, load_guided(m_u, m_c, i, m_fp32, guidance), x[i], sigma, c_out, s2p1, dt);
      x_prev[i] = __fadd_rn(xp, __fmul_rn(noise ? noise[i] : z[k], sigma_up));
    }
  }
}

// UniPCMultistepScheduler.step with predict_x0 (scheduling_unipc_multistep.py:720-804): convert_model_output
// (:368-437), the optional UniC corrector (:567-701) and the UniP predictor (:438-565), one rounding per operation in
// the order documented at b200mix_unipc_step. The pointers without __restrict__ may alias as documented there.
struct UnipcArgs {
  const void* m_u;
  const void* m_c;
  const float* x;
  const float* last;
  const float* m_prev;
  const float* hc[2];
  const float* hp[2];
  float* x_next;
  float* x_corr;
  float* m_out;
  long long n;
  int m_fp32, pred_type;
  float guidance;
  b200mix_unipc_coeffs k;
};

// sum_k r[k] * ((h[k][i] - base) / rk[k]) over the present terms in ascending k; `have` tells whether any was present
__device__ __forceinline__ float unipc_history_sum(const float* const h[2], const float r[2], const float rk[2],
                                                   long long i, float base, bool& have) {
  float acc = 0.0f;
  have = false;
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    if (!h[k]) continue;
    const float t = __fmul_rn(r[k], __fdiv_rn(__fsub_rn(h[k][i], base), rk[k]));
    acc = have ? __fadd_rn(acc, t) : t;
    have = true;
  }
  return acc;
}

__global__ void __launch_bounds__(256) unipc_step_kernel(UnipcArgs a) {
  const b200mix_unipc_coeffs& k = a.k;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < a.n; i += (long long)gridDim.x * blockDim.x) {
    const float xi = a.x[i];
    float m0, unused;
    predict_x0_eps(a.pred_type, load_guided(a.m_u, a.m_c, i, a.m_fp32, a.guidance), xi, k.alpha_t, k.sigma_t, m0,
                   unused);
    float xc = xi;
    if (a.last) {
      const float mp = a.m_prev[i];
      const float base = __fsub_rn(__fmul_rn(k.A_c, a.last[i]), __fmul_rn(k.K_c, mp));
      float res = __fmul_rn(k.rc_last, __fsub_rn(m0, mp));
      bool have;
      const float corr = unipc_history_sum(a.hc, k.rc, k.rk_c, i, mp, have);
      if (have) res = __fadd_rn(corr, res);
      xc = __fsub_rn(base, __fmul_rn(k.E_c, res));
    }
    float xn = __fsub_rn(__fmul_rn(k.A_p, xc), __fmul_rn(k.K_p, m0));
    bool have;
    const float pred = unipc_history_sum(a.hp, k.rp, k.rk_p, i, m0, have);
    if (have) xn = __fsub_rn(xn, __fmul_rn(k.E_p, pred));
    a.m_out[i] = m0;
    a.x_corr[i] = xc;
    a.x_next[i] = xn;
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

// ---- T2I-Adapter (models/adapter.py) -------------------------------------------------------------------------------
__device__ __forceinline__ void bf16x8_to_f32(const uint4& v, float* f) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int k = 0; k < 4; ++k) f[2 * k] = bf16_lo(w[k]), f[2 * k + 1] = bf16_hi(w[k]);
}
__device__ __forceinline__ uint4 f32x8_to_bf16(const float* f) {
  return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
}

// nn.PixelUnshuffle(F): y[b, ho, wo, c*F*F + i*F + j] = x[b, c, ho*F + i, wo*F + j]. One thread per 16-byte output piece:
// 8 consecutive output channels are 8 neighbouring pixels (j0 .. j0+7) of one input row, read as one or two 16-byte
// loads. Consecutive threads write consecutive pieces of one output pixel.
template <int F>
__global__ void __launch_bounds__(256) pixel_unshuffle_kernel(const void* __restrict__ x, int x_fp32,
                                                              uint4* __restrict__ y, long long total, int C, int H,
                                                              int W) {
  pdl_wait();
  pdl_launch_dependents();
  constexpr int RV = F / 8;      // pieces per input row segment
  constexpr int PV = F * RV;     // pieces per input channel
  const int Ho = H / F, Wo = W / F, pieces = C * PV;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int p = (int)(i % pieces);
    long long q = i / pieces;
    const int wo = (int)(q % Wo);
    q /= Wo;
    const int ho = (int)(q % Ho);
    const long long b = q / Ho;
    const int c = p / PV, r = p - c * PV;
    const int row = r / RV, j0 = (r - row * RV) * 8;
    const long long src = ((b * C + c) * H + (long long)ho * F + row) * W + (long long)wo * F + j0;
    uint4 out;
    if (x_fp32) {
      const float4* s = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(x) + src);
      const float4 a = __ldg(s), e = __ldg(s + 1);
      out = make_uint4(pack_bf16x2(a.x, a.y), pack_bf16x2(a.z, a.w), pack_bf16x2(e.x, e.y), pack_bf16x2(e.z, e.w));
    } else {
      out = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(x) + src));
    }
    y[i] = out;
  }
}

// nn.AvgPool2D(2, 2, ceil_mode=True, exclusive=True) on bf16 NHWC: one thread per 16-byte piece of an output pixel. The
// valid pixels of the window are summed in fp32 in row-major order and divided by their count (1, 2 or 4: exact).
__global__ void __launch_bounds__(256) avgpool2x2_nhwc_kernel(const uint4* __restrict__ x, uint4* __restrict__ y,
                                                              long long total, int H, int W, int CV) {
  pdl_wait();
  pdl_launch_dependents();
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(i % CV);
    long long q = i / CV;
    const int wo = (int)(q % Wo);
    q /= Wo;
    const int ho = (int)(q % Ho);
    const long long b = q / Ho;
    const int nh = min(2, H - 2 * ho), nw = min(2, W - 2 * wo);
    float acc[8] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
    for (int dy = 0; dy < nh; ++dy) {
      for (int dx = 0; dx < nw; ++dx) {
        float v[8];
        bf16x8_to_f32(__ldg(x + ((b * H + 2 * ho + dy) * W + 2 * wo + dx) * CV + cv), v);
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = __fadd_rn(acc[k], v[k]);
      }
    }
    const float inv = 1.0f / (float)(nh * nw);  // a power of two: the product is the exact quotient
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = __fmul_rn(acc[k], inv);
    y[i] = f32x8_to_bf16(acc);
  }
}

// y[r, :] = sum_k w[k] * x_k[r mod rows_k, :], one thread per 16-byte piece; products and sums rounded separately in k
// order, then once to bf16.
constexpr int kWsumMax = 8;
struct WsumArgs {
  const uint4* x[kWsumMax];
  long long rows[kWsumMax];
  float w[kWsumMax];
  int n;
};
__global__ void __launch_bounds__(256) weighted_sum_rows_kernel(WsumArgs a, uint4* __restrict__ y, long long total,
                                                                long long RV) {
  pdl_wait();
  pdl_launch_dependents();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / RV, v = i - r * RV;
    float acc[8] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
    for (int k = 0; k < a.n; ++k) {
      float f[8];
      bf16x8_to_f32(__ldg(a.x[k] + (r % a.rows[k]) * RV + v), f);
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] = __fadd_rn(acc[e], __fmul_rn(a.w[k], f[e]));
    }
    y[i] = f32x8_to_bf16(acc);
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
  B200_CHECK_ARG(act >= B200MIX_ACT_NONE && act <= B200MIX_ACT_RELU, "activation: unknown act %d", (int)act);
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

extern "C" int b200mix_iddpm_step(const void* model_out, int32_t m_fp32, const float* x, const float* noise, float* x_prev,
                                  float* x_dup, int64_t B, int64_t C, int64_t n_per_channel, float cfg_scale,
                                  int32_t cfg_channel, float sqrt_recip_alphas_cumprod, float sqrt_recipm1_alphas_cumprod,
                                  float posterior_mean_coef1, float posterior_mean_coef2, float max_log, float min_log,
                                  int32_t add_noise, uint64_t seed, int64_t step, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(model_out && x && x_prev && B > 0 && C > 0 && n_per_channel > 0, "iddpm_step: bad arguments");
  B200_CHECK_ARG(cfg_channel >= 0 && cfg_channel <= 2 * C, "iddpm_step: cfg_channel must lie in [0, 2C]");
  B200_CHECK_ARG(step >= 0 && step <= 0xFFFFFFFFll, "iddpm_step: step must fit 32 bits");
  IddpmArgs a;
  a.m = model_out, a.x = x, a.noise = noise, a.x_prev = x_prev, a.x_dup = x_dup;
  a.B = B, a.C = C, a.N = n_per_channel;
  a.m_fp32 = m_fp32, a.cfg_channel = cfg_channel, a.add_noise = add_noise ? 1 : 0;
  a.cfg_scale = cfg_scale, a.sqrt_recip = sqrt_recip_alphas_cumprod, a.sqrt_recipm1 = sqrt_recipm1_alphas_cumprod;
  a.coef1 = posterior_mean_coef1, a.coef2 = posterior_mean_coef2, a.max_log = max_log, a.min_log = min_log;
  a.seed = seed, a.step = (uint32_t)step;
  const long long groups = (B * C * n_per_channel + 3) / 4;
  B200_CUDA(launch_pdl(iddpm_step_kernel, dim3(ew_grid(groups, 256)), dim3(256), 0, ST(stream), 1, a));
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

extern "C" int b200mix_euler_ancestral_step(const void* m_u, const void* m_c, int32_t m_fp32, float guidance,
                                            const float* x, const float* noise, float* x_prev, int64_t n,
                                            int32_t prediction_type, float sigma, float c_out, float s2p1, float dt,
                                            float sigma_up, uint64_t seed, int64_t step, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(m_u && x && x_prev && n > 0, "euler_ancestral_step: bad arguments");
  B200_CHECK_ARG(prediction_type == 0 || prediction_type == 2,
                 "euler_ancestral_step: prediction_type must be 0 (epsilon) or 2 (v_prediction)");
  B200_CHECK_ARG(step >= 0 && step <= 0xFFFFFFFFll, "euler_ancestral_step: step must fit 32 bits");
  euler_ancestral_step_kernel<<<ew_grid((n + 3) / 4, 256), 256, 0, ST(stream)>>>(
      m_u, m_c, m_fp32, guidance, x, noise, x_prev, n, prediction_type == 2, sigma, c_out, s2p1, dt, sigma_up, seed,
      (uint32_t)step);
  B200_LAUNCH_CHECK();
  return 0;
}

extern "C" int b200mix_unipc_step(const void* m_u, const void* m_c, int32_t m_fp32, float guidance, const float* x,
                                  const float* last_sample, const float* m_prev, const float* hc0, const float* hc1,
                                  const float* hp0, const float* hp1, float* x_next, float* x_corr, float* m_out,
                                  int64_t n, int32_t prediction_type, const b200mix_unipc_coeffs* coeffs, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(m_u && x && x_next && x_corr && m_out && coeffs && n > 0, "unipc_step: bad arguments");
  B200_CHECK_ARG(prediction_type >= 0 && prediction_type <= 2, "unipc_step: prediction_type must be 0, 1 or 2");
  B200_CHECK_ARG(!last_sample == !m_prev, "unipc_step: last_sample and m_prev go together (the corrector)");
  B200_CHECK_ARG(last_sample || (!hc0 && !hc1), "unipc_step: corrector history without the corrector");
  UnipcArgs a;
  a.m_u = m_u, a.m_c = m_c, a.x = x, a.last = last_sample, a.m_prev = m_prev;
  a.hc[0] = hc0, a.hc[1] = hc1, a.hp[0] = hp0, a.hp[1] = hp1;
  a.x_next = x_next, a.x_corr = x_corr, a.m_out = m_out;
  a.n = n, a.m_fp32 = m_fp32, a.pred_type = prediction_type, a.guidance = guidance, a.k = *coeffs;
  unipc_step_kernel<<<ew_grid(n, 256), 256, 0, ST(stream)>>>(a);
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
    const float e = load_guided(eps_u, eps_c, i, eps_fp32, guidance);
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

// The two stochastic steps below take one thread per group of 4 consecutive elements, which is one Philox call
// (philox_normal4) when noise is NULL, as euler_ancestral_step_kernel does; the minimum of 4 CTAs per SM gives ptxas
// the registers to keep the fp64 Box-Muller out of local memory. x / x_prev may alias, so they are not __restrict__.

// DDIMScheduler.step with eta > 0 (scheduling_ddim.py:410-475) in the order documented at b200mix_ddim_eta_step.
__global__ void __launch_bounds__(256, 4) ddim_eta_step_kernel(
    const void* __restrict__ m_u, const void* __restrict__ m_c, int m_fp32, float guidance, const float* x,
    const float* __restrict__ noise, float* x_prev, long long n, float sa_t, float sb_t, float sa_p, float sb_p,
    float std_dev_t, int pred_type, float clip, int clipped_eps, unsigned long long seed, uint32_t step) {
  pdl_wait();
  pdl_launch_dependents();
  const long long groups = (n + 3) >> 2;
  for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < groups; g += (long long)gridDim.x * blockDim.x) {
    float z[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    if (!noise) philox_normal4(seed, step, (unsigned long long)g, z);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const long long i = 4 * g + k;
      if (i >= n) break;
      const float xi = x[i];
      float x0, e;
      predict_x0_eps(pred_type, load_guided(m_u, m_c, i, m_fp32, guidance), xi, sa_t, sb_t, x0, e);
      if (clip > 0.0f) x0 = fminf(fmaxf(x0, -clip), clip);
      if (clipped_eps) e = __fdiv_rn(__fsub_rn(xi, __fmul_rn(sa_t, x0)), sb_t);
      const float mean = __fadd_rn(__fmul_rn(sa_p, x0), __fmul_rn(sb_p, e));
      x_prev[i] = __fadd_rn(mean, __fmul_rn(std_dev_t, noise ? noise[i] : z[k]));
    }
  }
}

// DPM-Solver++ 2M SDE step (scheduling_dpmsolver_multistep.py:446-453, :561-567, :666-674) in the order documented at
// b200mix_dpmpp_2m_sde_step.
__global__ void __launch_bounds__(256, 4) dpmpp_2m_sde_step_kernel(
    const void* __restrict__ eps_u, const void* __restrict__ eps_c, int eps_fp32, float guidance, const float* x,
    const float* __restrict__ noise, const float* __restrict__ m_prev, float* x_next, float* __restrict__ m_out,
    long long n, float sigma_cur, float alpha_cur, float A, float B, float halfB, float inv_r0, float N,
    unsigned long long seed, uint32_t step) {
  pdl_wait();
  pdl_launch_dependents();
  const long long groups = (n + 3) >> 2;
  for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < groups; g += (long long)gridDim.x * blockDim.x) {
    float z[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    if (!noise) philox_normal4(seed, step, (unsigned long long)g, z);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const long long i = 4 * g + k;
      if (i >= n) break;
      const float xv = x[i];
      const float m0 = __fdiv_rn(__fsub_rn(xv, __fmul_rn(sigma_cur, load_guided(eps_u, eps_c, i, eps_fp32, guidance))),
                                 alpha_cur);
      float r = __fadd_rn(__fmul_rn(A, xv), __fmul_rn(B, m0));
      if (m_prev) r = __fadd_rn(r, __fmul_rn(halfB, __fmul_rn(inv_r0, __fsub_rn(m0, m_prev[i]))));
      m_out[i] = m0;
      x_next[i] = __fadd_rn(r, __fmul_rn(N, noise ? noise[i] : z[k]));
    }
  }
}

extern "C" int b200mix_ddim_eta_step(const void* m_u, const void* m_c, int32_t m_fp32, float guidance, const float* x,
                                     const float* noise, float* x_prev, int64_t n, float sqrt_alpha_t, float sqrt_beta_t,
                                     float sqrt_alpha_prev, float sqrt_beta_prev, float std_dev_t,
                                     int32_t prediction_type, float clip_sample_range, int32_t use_clipped_model_output,
                                     uint64_t seed, int64_t step, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(m_u && x && x_prev && n > 0, "ddim_eta_step: bad arguments");
  B200_CHECK_ARG(prediction_type >= 0 && prediction_type <= 2, "ddim_eta_step: prediction_type must be 0 (epsilon), 1 "
                 "(sample) or 2 (v_prediction)");
  B200_CHECK_ARG(step >= 0 && step <= 0xFFFFFFFFll, "ddim_eta_step: step must fit 32 bits");
  B200_CUDA(launch_pdl(ddim_eta_step_kernel, dim3(ew_grid((n + 3) / 4, 256)), dim3(256), 0, ST(stream), 1, m_u, m_c,
                       (int)m_fp32, guidance, x, noise, x_prev, (long long)n, sqrt_alpha_t, sqrt_beta_t, sqrt_alpha_prev,
                       sqrt_beta_prev, std_dev_t, (int)prediction_type, clip_sample_range,
                       (int)(use_clipped_model_output ? 1 : 0), (unsigned long long)seed, (uint32_t)step));
  return 0;
}

extern "C" int b200mix_dpmpp_2m_sde_step(const void* eps_u, const void* eps_c, int32_t eps_fp32, float guidance,
                                         const float* x, const float* noise, const float* m_prev, float* x_next,
                                         float* m_out, int64_t n, float sigma_cur, float alpha_cur, float A, float B,
                                         float halfB, float inv_r0, float N, uint64_t seed, int64_t step, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(eps_u && x && x_next && m_out && n > 0 && alpha_cur != 0.0f, "dpmpp_2m_sde_step: bad arguments");
  B200_CHECK_ARG(step >= 0 && step <= 0xFFFFFFFFll, "dpmpp_2m_sde_step: step must fit 32 bits");
  B200_CUDA(launch_pdl(dpmpp_2m_sde_step_kernel, dim3(ew_grid((n + 3) / 4, 256)), dim3(256), 0, ST(stream), 1, eps_u,
                       eps_c, (int)eps_fp32, guidance, x, noise, m_prev, x_next, m_out, (long long)n, sigma_cur,
                       alpha_cur, A, B, halfB, inv_r0, N, (unsigned long long)seed, (uint32_t)step));
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
  // the kernel reads and writes (even column) bf16 pairs
  B200_CHECK_ARG(ld_row % 2 == 0 && ld_out % 2 == 0 && ld_row >= 3 * H * d && ld_out >= H * d &&
                     reinterpret_cast<uintptr_t>(qkv) % 4 == 0 && reinterpret_cast<uintptr_t>(out) % 4 == 0,
                 "small_attention: rows must be 4-byte aligned, ld_row >= 3*H*d, ld_out >= H*d");
  const size_t smem = (size_t)(3 * T * d + T * T) * sizeof(float);
  const long long ctas = B * S * H;
  B200_CHECK_ARG(ctas < (1ll << 31), "small_attention: too many sequences");
  // T = 32, d = 128 needs 52 KB, above the 48 KB available without opting in
  constexpr int kMaxSmem = (3 * 32 * 128 + 32 * 32) * sizeof(float);
  static bool configured = false;
  if (!configured) {
    B200_CUDA(cudaFuncSetAttribute(small_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem));
    configured = true;
  }
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

static inline bool aligned16(const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 == 0; }

// nn.PixelUnshuffle + cast, models/adapter.py:306,328 (FullAdapter / FullAdapterXL / LightAdapter.forward)
extern "C" int b200mix_pixel_unshuffle(const void* x, int32_t x_fp32, void* y, int64_t B, int64_t C, int64_t H,
                                       int64_t W, int32_t f, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(x && y && aligned16(x) && aligned16(y), "pixel_unshuffle: x and y must be 16-byte aligned device pointers");
  B200_CHECK_ARG(f == 8 || f == 16, "pixel_unshuffle: downscale factor must be 8 or 16, got %d", (int)f);
  B200_CHECK_ARG(B > 0 && C > 0 && H > 0 && W > 0, "pixel_unshuffle: bad shape");
  B200_CHECK_ARG(H % f == 0 && W % f == 0, "pixel_unshuffle: H=%lld and W=%lld must be multiples of %d", (long long)H,
                 (long long)W, (int)f);
  B200_CHECK_ARG(B * C * H * W < (1ll << 40) && C * f * f < (1ll << 31) && H < (1ll << 31) && W < (1ll << 31),
                 "pixel_unshuffle: tensor too large");
  const long long total = B * C * H * W / 8;
  auto kernel = f == 8 ? pixel_unshuffle_kernel<8> : pixel_unshuffle_kernel<16>;
  B200_CUDA(launch_pdl(kernel, dim3(ew_grid(total, 256)), dim3(256), 0, ST(stream), 1, x, (int)(x_fp32 ? 1 : 0),
                       reinterpret_cast<uint4*>(y), total, (int)C, (int)H, (int)W));
  return 0;
}

// nn.AvgPool2D(kernel_size=2, stride=2, ceil_mode=True), models/adapter.py:411,537 (AdapterBlock / LightAdapterBlock)
extern "C" int b200mix_avgpool2x2_nhwc(const void* x, void* y, int64_t B, int64_t H, int64_t W, int64_t C, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(x && y && aligned16(x) && aligned16(y), "avgpool2x2_nhwc: x and y must be 16-byte aligned device pointers");
  B200_CHECK_ARG(B > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0, "avgpool2x2_nhwc: bad shape (C must be a multiple of 8)");
  B200_CHECK_ARG(H < (1ll << 30) && W < (1ll << 30) && C < (1ll << 31), "avgpool2x2_nhwc: tensor too large");
  const long long total = B * ((H + 1) / 2) * ((W + 1) / 2) * (C / 8);
  B200_CUDA(launch_pdl(avgpool2x2_nhwc_kernel, dim3(ew_grid(total, 256)), dim3(256), 0, ST(stream), 1,
                       reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(y), total, (int)H, (int)W,
                       (int)(C / 8)));
  return 0;
}

// MultiAdapter.forward's weighted sum (models/adapter.py:85-100) fused with the pipelines' scale, tile and CFG concat
// (pipeline_stable_diffusion_adapter.py:823-836)
extern "C" int b200mix_weighted_sum_rows(int32_t n, const void* const* x, const int64_t* rows_in, const float* weight,
                                         void* y, int64_t rows_out, int64_t row_elems, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(n >= 1 && n <= kWsumMax && x && rows_in && weight, "weighted_sum_rows: 1 to %d inputs", kWsumMax);
  B200_CHECK_ARG(y && aligned16(y) && rows_out > 0 && row_elems > 0 && row_elems % 8 == 0,
                 "weighted_sum_rows: y must be 16-byte aligned, rows_out > 0, row_elems a positive multiple of 8");
  const char* y0 = static_cast<const char*>(y);
  const char* y1 = y0 + rows_out * row_elems * 2;
  WsumArgs a = {};
  a.n = n;
  for (int k = 0; k < n; ++k) {
    B200_CHECK_ARG(x[k] && aligned16(x[k]) && rows_in[k] > 0, "weighted_sum_rows: input %d is null, unaligned or empty", k);
    const char* x0 = static_cast<const char*>(x[k]);
    const char* x1 = x0 + rows_in[k] * row_elems * 2;
    B200_CHECK_ARG(x1 <= y0 || y1 <= x0, "weighted_sum_rows: y overlaps input %d", k);
    a.x[k] = static_cast<const uint4*>(x[k]), a.rows[k] = rows_in[k], a.w[k] = weight[k];
  }
  const long long total = rows_out * (row_elems / 8);
  B200_CUDA(launch_pdl(weighted_sum_rows_kernel, dim3(ew_grid(total, 256)), dim3(256), 0, ST(stream), 1, a,
                       reinterpret_cast<uint4*>(y), total, (long long)(row_elems / 8)));
  return 0;
}
