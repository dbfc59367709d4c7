// HBM-bound normalisation kernels: GroupNorm(+SiLU) on NHWC with fused channel-concat input, and the row-wise
// LayerNorm / RMSNorm family with fused residual-gate and AdaLN modulation. 16-byte coalesced accesses, fp32 math.
//
// Replaces (reference): nn.GroupNorm + SiLU in ResnetBlock2D (ppdiffusers/models/resnet.py:667-692,760-786),
// Transformer2DModel.norm (transformer_2d.py:161), conv_norm_out (unet_2d_condition.py:604,1193-1195);
// nn.LayerNorm in BasicTransformerBlock (attention.py:307-350); the Triton ops fused_adaLN_scale_residual /
// adaptive_layer_norm / rms_norm (paddlemix/triton_ops/triton_ops.py:702-755, 981-1027, 1198-1232) and
// Qwen2RMSNorm (paddlemix/models/qwen2_vl/modeling_qwen2_vl.py:467-478).
#include <algorithm>

#include "common.cuh"
#include "ptx.cuh"

namespace b200 {

__device__ __forceinline__ void unpack8(const uint4& w, float (&f)[8]) {
  f[0] = bf16_lo(w.x), f[1] = bf16_hi(w.x), f[2] = bf16_lo(w.y), f[3] = bf16_hi(w.y);
  f[4] = bf16_lo(w.z), f[5] = bf16_hi(w.z), f[6] = bf16_lo(w.w), f[7] = bf16_hi(w.w);
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]),
                    pack_bf16x2(f[6], f[7]));
}
// SiLU as x * sigmoid(x) = h + h * tanh(h), h = x / 2: ONE MUFU op (tanh.approx, relative error ~2^-11, below the
// bf16 rounding of the output) and two FMA-pipe ops. The round-1 form x / (1 + __expf(-x)) compiled to two MUFU ops plus
// an IEEE division (~10 instructions) and made gn_apply issue-bound (72 registers, 45 % issue-active, 38 us for a 42 MB
// tensor against 15 us for the statistics pass over the same bytes).
__device__ __forceinline__ float silu_f(float x) {
  const float h = 0.5f * x;
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(h));
  return fmaf(h, t, h);
}

// ------------------------------------------------------------------------------------------------------------
// GroupNorm statistics: per (batch, CTA, group) partial sum / sum of squares, exchanged as FIXED-POINT int64 (sum: 2^24,
// sum of squares: 2^16) so that the cross-CTA reduction is integer adds: exact, order-independent (bit-reproducible
// without atomics-ordering concerns) and off the FP64 pipe. The first version kept the partials in double; on this
// part ~100 dependent DADDs per CTA (one warp, one group per lane) cost more than streaming the CTA's pixels
// (FP64 issues at a fraction of the FP32 rate). Only the last three operations per
// group (mean, variance from the int64 totals) are double. Block = PPB pixels x CV 8-channel vectors; each thread owns
// a fixed channel vector, so every row is read with fully coalesced 16-byte loads.
// ------------------------------------------------------------------------------------------------------------
constexpr float GN_FIX_SUM = 16777216.0f, GN_FIX_SQ = 65536.0f;
__global__ void gn_stats_kernel(const __nv_bfloat16* __restrict__ x1, int C1, const __nv_bfloat16* __restrict__ x2,
                                int C2, long long* __restrict__ partial, float* __restrict__ mr,  // n_per_group: 1 / elements per group
                                unsigned int* __restrict__ counters, long long HW, int groups, int PPB, int pix_per_cta,
                                double n_per_group, float eps) {
  extern __shared__ float sm[];  // [PPB][2][C]
  __shared__ bool is_last;
  pdl_wait();
  pdl_launch_dependents();
  const int C = C1 + C2;
  const int CV = C >> 3;
  const int cv = threadIdx.x % CV;
  const int pl = threadIdx.x / CV;
  const int b = blockIdx.y;
  const int c0 = cv * 8;
  const __nv_bfloat16* src;
  long long ld;
  int cc;
  if (c0 < C1) {
    src = x1 + static_cast<long long>(b) * HW * C1, ld = C1, cc = c0;
  } else {
    src = x2 + static_cast<long long>(b) * HW * C2, ld = C2, cc = c0 - C1;
  }
  const long long p_begin = static_cast<long long>(blockIdx.x) * pix_per_cta;
  const long long p_end = min(HW, p_begin + pix_per_cta);
  if (pl < PPB) {
    float s[8], q[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i] = 0.0f, q[i] = 0.0f;
    long long pix = p_begin + pl;
    for (; pix + 7LL * PPB < p_end; pix += 8LL * PPB) {  // 8 independent 16-byte loads in flight per thread
      uint4 w[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) w[u] = __ldg(reinterpret_cast<const uint4*>(src + (pix + (long long)u * PPB) * ld + cc));
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        float f[8];
        unpack8(w[u], f);
#pragma unroll
        for (int i = 0; i < 8; ++i) s[i] += f[i], q[i] += f[i] * f[i];
      }
    }
    for (; pix < p_end; pix += PPB) {
      const uint4 w = __ldg(reinterpret_cast<const uint4*>(src + pix * ld + cc));
      float f[8];
      unpack8(w, f);
#pragma unroll
      for (int i = 0; i < 8; ++i) s[i] += f[i], q[i] += f[i] * f[i];
    }
    float* dst = sm + static_cast<size_t>(pl) * 2 * C;
#pragma unroll
    for (int i = 0; i < 8; ++i) dst[c0 + i] = s[i], dst[C + c0 + i] = q[i];
  }
  __syncthreads();
  const int cpg = C / groups;
  // `per` threads cooperate on one group (host guarantees blockDim >= groups): strided fp32 partial sums, combined in a
  // fixed order through shared memory
  const int per = blockDim.x / groups;
  const int gq = threadIdx.x / per, jq = threadIdx.x % per;
  float ss = 0.0f, qq = 0.0f;
  if (gq < groups) {
    const int n = PPB * cpg;
    for (int e = jq; e < n; e += per) {
      const int l = e / cpg, c = gq * cpg + (e - l * cpg);
      const float* row = sm + static_cast<size_t>(l) * 2 * C;
      ss += row[c], qq += row[C + c];
    }
  }
  __syncthreads();  // everybody has read the per-thread sums: the buffer is reused for the per-group combine
  float2* comb = reinterpret_cast<float2*>(sm);  // [threads]
  comb[threadIdx.x] = make_float2(ss, qq);
  __syncthreads();
  if (gq < groups && jq == 0) {
    float a = 0.0f, c = 0.0f;
    for (int t = 0; t < per; ++t) a += comb[threadIdx.x + t].x, c += comb[threadIdx.x + t].y;
    long long* o = partial + ((static_cast<long long>(b) * gridDim.x + blockIdx.x) * groups + gq) * 2;
    o[0] = __float2ll_rn(a * GN_FIX_SUM), o[1] = __float2ll_rn(c * GN_FIX_SQ);
  }
  // ---- the last CTA of this batch element reduces the per-CTA partials in a FIXED order (bit-reproducible whichever
  // CTA happens to be last) and writes (mean, rstd) per group: no separate finalize launch. The counter is reset for
  // the next call (graph replays reuse the scratch).
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int done = atomicAdd(&counters[b], 1u);
    is_last = (done == gridDim.x - 1);
    if (is_last) counters[b] = 0u;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  long long* red = reinterpret_cast<long long*>(sm);  // [threads][2] (dynamic smem is at least threads * 16 bytes: host guarantees)
  const int gx = gridDim.x;
  const int g = gq, j = jq;
  long long su = 0, sq = 0;
  if (g < groups) {
    // L2 loads (the partials were published with __threadfence + the arrival counter), several in flight: a volatile
    // loop here would serialise one L2 round trip per partial
    const longlong2* srcp = reinterpret_cast<const longlong2*>(partial + (static_cast<long long>(b) * gx * groups + g) * 2);
#pragma unroll 4
    for (int i = j; i < gx; i += per) {
      const longlong2 t = __ldcg(srcp + static_cast<size_t>(i) * groups);
      su += t.x, sq += t.y;
    }
  }
  red[2 * threadIdx.x] = su, red[2 * threadIdx.x + 1] = sq;
  __syncthreads();
  if (g < groups && j == 0) {
    long long ai = 0, ci = 0;
    for (int t = 0; t < per; ++t) ai += red[2 * (threadIdx.x + t)], ci += red[2 * (threadIdx.x + t) + 1];
    // n_per_group arrives as its reciprocal: a double division is ~30 FP64 instructions on the kernel's critical tail
    const double mean = static_cast<double>(ai) * (1.0 / GN_FIX_SUM) * n_per_group;
    double var = static_cast<double>(ci) * (1.0 / GN_FIX_SQ) * n_per_group - mean * mean;
    if (var < 0.0) var = 0.0;
    mr[(b * groups + g) * 2 + 0] = static_cast<float>(mean);
    mr[(b * groups + g) * 2 + 1] = rsqrtf(static_cast<float>(var) + eps);
  }
}

__global__ void __launch_bounds__(1024) gn_apply_kernel(const __nv_bfloat16* __restrict__ x1, int C1, const __nv_bfloat16* __restrict__ x2,
                                int C2, const float* __restrict__ gamma, const float* __restrict__ beta,
                                __nv_bfloat16* __restrict__ y, const float* __restrict__ mr, long long HW,
                                int groups, int silu, int PPB, int pix_per_cta) {
  pdl_wait();
  pdl_launch_dependents();
  const int C = C1 + C2;
  const int CV = C >> 3;
  const int cv = threadIdx.x % CV;
  const int pl = threadIdx.x / CV;
  const int b = blockIdx.y;
  const int cpg = C / groups;
  const float* sm = mr + static_cast<long long>(b) * groups * 2;  // (mean, rstd) per group
  if (pl >= PPB) return;
  const int c0 = cv * 8;
  float a[8], sh[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = c0 + i;
    const int g = c / cpg;
    a[i] = __ldg(sm + 2 * g + 1) * gamma[c];
    sh[i] = beta[c] - __ldg(sm + 2 * g) * a[i];
  }
  const __nv_bfloat16* src;
  long long ld;
  int cc;
  if (c0 < C1) {
    src = x1 + static_cast<long long>(b) * HW * C1, ld = C1, cc = c0;
  } else {
    src = x2 + static_cast<long long>(b) * HW * C2, ld = C2, cc = c0 - C1;
  }
  __nv_bfloat16* dst = y + static_cast<long long>(b) * HW * C + c0;
  const long long p_begin = static_cast<long long>(blockIdx.x) * pix_per_cta;
  const long long p_end = min(HW, p_begin + pix_per_cta);
  long long pix = p_begin + pl;
  for (; pix + 3LL * PPB < p_end; pix += 4LL * PPB) {
    uint4 w[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) w[u] = __ldg(reinterpret_cast<const uint4*>(src + (pix + (long long)u * PPB) * ld + cc));
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      float f[8];
      unpack8(w[u], f);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float v = fmaf(f[i], a[i], sh[i]);
        f[i] = silu ? silu_f(v) : v;
      }
      *reinterpret_cast<uint4*>(dst + (pix + (long long)u * PPB) * C) = pack8(f);
    }
  }
  for (; pix < p_end; pix += PPB) {
    const uint4 w = __ldg(reinterpret_cast<const uint4*>(src + pix * ld + cc));
    float f[8];
    unpack8(w, f);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float v = fmaf(f[i], a[i], sh[i]);
      f[i] = silu ? silu_f(v) : v;
    }
    *reinterpret_cast<uint4*>(dst + pix * C) = pack8(f);
  }
}

// ------------------------------------------------------------------------------------------------------------
// Row-wise LayerNorm / RMSNorm: one warp per row, the row lives in registers (two-pass mean / variance).
// The arithmetic runs on PACKED fp32 pairs (FADD2 / FMUL2 / FFMA2: two lanes per instruction): the round-1 kernels were
// issue-bound (ncu: 57 % issue-active, ~20 instructions per element, DRAM at 21 %), not memory-bound. Both LayerNorm
// kernels share these helpers, so they accumulate in the same order and stay bit-identical to each other.
// ------------------------------------------------------------------------------------------------------------
struct P8 {
  uint64_t p[4];  // 8 fp32 values as 4 (even, odd) pairs
};
__device__ __forceinline__ P8 unpack8p(const uint4& w) {
  P8 r;
  r.p[0] = pack_f32x2(bf16_lo(w.x), bf16_hi(w.x)), r.p[1] = pack_f32x2(bf16_lo(w.y), bf16_hi(w.y));
  r.p[2] = pack_f32x2(bf16_lo(w.z), bf16_hi(w.z)), r.p[3] = pack_f32x2(bf16_lo(w.w), bf16_hi(w.w));
  return r;
}
__device__ __forceinline__ uint4 pack8p(const P8& v) {
  float a, b;
  uint4 w;
  unpack_f32x2(v.p[0], a, b), w.x = pack_bf16x2(a, b);
  unpack_f32x2(v.p[1], a, b), w.y = pack_bf16x2(a, b);
  unpack_f32x2(v.p[2], a, b), w.z = pack_bf16x2(a, b);
  unpack_f32x2(v.p[3], a, b), w.w = pack_bf16x2(a, b);
  return w;
}
__device__ __forceinline__ float pair_sum(uint64_t v) {
  float a, b;
  unpack_f32x2(v, a, b);
  return a + b;
}
// acc += the 8 values of w (as two interleaved partial sums)
__device__ __forceinline__ void ln_acc_sum(uint64_t& acc, const uint4& w) {
  const P8 v = unpack8p(w);
  acc = fadd2(fadd2(acc, v.p[0]), fadd2(v.p[1], fadd2(v.p[2], v.p[3])));
}
// acc += (v - mean)^2 over the 8 values of w
__device__ __forceinline__ void ln_acc_sq(uint64_t& acc, const uint4& w, uint64_t nmean2) {
  const P8 v = unpack8p(w);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint64_t d = fadd2(v.p[k], nmean2);
    acc = ffma2(d, d, acc);
  }
}
__device__ __forceinline__ P8 load8f(const float* ptr) {  // 8 consecutive fp32 (32-byte aligned) as pairs
  const float4 a = __ldg(reinterpret_cast<const float4*>(ptr)), b = __ldg(reinterpret_cast<const float4*>(ptr) + 1);
  P8 r;
  r.p[0] = pack_f32x2(a.x, a.y), r.p[1] = pack_f32x2(a.z, a.w), r.p[2] = pack_f32x2(b.x, b.y), r.p[3] = pack_f32x2(b.z, b.w);
  return r;
}
// Output stage for 8 channels of one row: ((x - mean) * rstd) [*w] [+b] [*(1 + scale) + shift] -> bf16. RMSNorm with a
// weight keeps Qwen2RMSNorm's cast order (normalised value rounded to the activation dtype, THEN multiplied).
__device__ __forceinline__ uint4 ln_output8(const uint4& raw, uint64_t nmean2, uint64_t rstd2, bool rms, const P8* wv,
                                            const P8* bv, const float* scale, const float* shift) {
  P8 o = unpack8p(raw);
#pragma unroll
  for (int k = 0; k < 4; ++k) o.p[k] = fmul2(fadd2(o.p[k], nmean2), rstd2);
  if (rms && wv) {
    o = unpack8p(pack8p(o));
#pragma unroll
    for (int k = 0; k < 4; ++k) o.p[k] = fmul2(o.p[k], wv->p[k]);
  } else if (wv) {
#pragma unroll
    for (int k = 0; k < 4; ++k) o.p[k] = fmul2(o.p[k], wv->p[k]);
  }
  if (bv) {
#pragma unroll
    for (int k = 0; k < 4; ++k) o.p[k] = fadd2(o.p[k], bv->p[k]);
  }
  if (scale) {
    const P8 sc = load8f(scale);
    const uint64_t one2 = pack_f32x2(1.0f, 1.0f);
#pragma unroll
    for (int k = 0; k < 4; ++k) o.p[k] = fmul2(o.p[k], fadd2(sc.p[k], one2));
  }
  if (shift) {
    const P8 sh = load8f(shift);
#pragma unroll
    for (int k = 0; k < 4; ++k) o.p[k] = fadd2(o.p[k], sh.p[k]);
  }
  return pack8p(o);
}
struct LNParams {
  const __nv_bfloat16* x;
  const __nv_bfloat16* delta;
  const float* gate;
  __nv_bfloat16* resid_out;
  __nv_bfloat16* y;
  const float* weight;
  const float* bias;
  const float* scale;
  const float* shift;
  long long ld_mod;
  long long rows_per_group;
  long long M;
  int N;
  float eps;
  int rms;
};

// Each warp normalises ROWS consecutive rows at once. The rows are kept PACKED (bf16 pairs, one uint4 per 8 channels)
// so that all ROWS*VPL 16-byte loads of a lane can be in flight together within the register budget; values are
// unpacked transiently for the two reductions and for the output.
template <int VPL, int ROWS>
__global__ void __launch_bounds__(256, (VPL * ROWS > 16) ? 1 : 2) layernorm_kernel(const LNParams p) {
  pdl_wait();
  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long row0 = (static_cast<long long>(blockIdx.x) * 8 + warp) * ROWS;
  if (row0 >= p.M) return;
  const int NV = p.N >> 3;
  uint4 raw[ROWS][VPL];
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
    const long long row = row0 + r;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int vi = lane + 32 * i;
      raw[r][i] = (row < p.M && vi < NV) ? __ldg(reinterpret_cast<const uint4*>(p.x + row * p.N) + vi)
                                          : make_uint4(0u, 0u, 0u, 0u);
    }
  }
  if (p.delta) {
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      const long long row = row0 + r;
      if (row >= p.M) continue;
      const long long g = static_cast<long long>(static_cast<unsigned>(row) / static_cast<unsigned>(p.rows_per_group));
#pragma unroll
      for (int i = 0; i < VPL; ++i) {
        const int vi = lane + 32 * i;
        if (vi >= NV) continue;
        float v[8], d[8];
        unpack8(raw[r][i], v);
        unpack8(__ldg(reinterpret_cast<const uint4*>(p.delta + row * p.N) + vi), d);
        if (p.gate) {
          const float* gp = p.gate + g * p.ld_mod + vi * 8;
#pragma unroll
          for (int k = 0; k < 8; ++k) v[k] = fmaf(__ldg(gp + k), d[k], v[k]);
        } else {
#pragma unroll
          for (int k = 0; k < 8; ++k) v[k] += d[k];
        }
        // the residual stream is stored in bf16: the rounded value is what gets normalised, so both outputs agree
        raw[r][i] = pack8(v);
        if (p.resid_out) *(reinterpret_cast<uint4*>(p.resid_out + row * p.N) + vi) = raw[r][i];
      }
    }
  }
  float mean[ROWS], rstd[ROWS];
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
    mean[r] = 0.0f;
    if (!p.rms) {
      uint64_t acc = 0ull;
#pragma unroll
      for (int i = 0; i < VPL; ++i) ln_acc_sum(acc, raw[r][i]);  // lanes past the row hold zeros
      float s = pair_sum(acc);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      mean[r] = s / p.N;
    }
  }
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
    const uint64_t nmean2 = pack_f32x2(-mean[r], -mean[r]);
    uint64_t acc = 0ull;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int vi = lane + 32 * i;
      if (vi < NV) ln_acc_sq(acc, raw[r][i], nmean2);
    }
    float sq = pair_sum(acc);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    rstd[r] = rsqrtf(sq / p.N + p.eps);
  }

  // output: columns are the same for all ROWS rows of a lane, so the affine vectors are loaded once (16-byte loads)
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int vi = lane + 32 * i;
    if (vi >= NV) continue;
    P8 wv, bv;
    if (p.weight) wv = load8f(p.weight + 8 * vi);
    if (p.bias) bv = load8f(p.bias + 8 * vi);
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      const long long row = row0 + r;
      if (row >= p.M) continue;
      const float* sc = nullptr;
      const float* sh = nullptr;
      if (p.scale || p.shift) {
        const long long g = static_cast<long long>(static_cast<unsigned>(row) / static_cast<unsigned>(p.rows_per_group));
        if (p.scale) sc = p.scale + g * p.ld_mod + 8 * vi;
        if (p.shift) sh = p.shift + g * p.ld_mod + 8 * vi;
      }
      *(reinterpret_cast<uint4*>(p.y + row * p.N) + vi) =
          ln_output8(raw[r][i], pack_f32x2(-mean[r], -mean[r]), pack_f32x2(rstd[r], rstd[r]), p.rms != 0,
                     p.weight ? &wv : nullptr, p.bias ? &bv : nullptr, sc, sh);
    }
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200mix_groupnorm_nhwc(const void* x1, int64_t C1, const void* x2, int64_t C2, const float* gamma,
                                      const float* beta, void* y, void* stats, int64_t stats_bytes, int64_t B, int64_t HW,
                                      int32_t groups, float eps, int32_t silu, void* stream) {
  if (int rc = ensure_device()) return rc;
  const int64_t C = C1 + C2;
  B200_CHECK_ARG(x1 && y && gamma && beta && stats, "groupnorm: null pointer");
  B200_CHECK_ARG(C1 % 8 == 0 && C2 % 8 == 0 && (C2 == 0 || x2), "groupnorm: channel counts must be multiples of 8");
  B200_CHECK_ARG(C % groups == 0, "groupnorm: C=%lld not divisible by groups=%d", (long long)C, groups);
  B200_CHECK_ARG(C / 8 <= 1024, "groupnorm: C too large");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int CV = (int)(C / 8);
  int PPB = 256 / CV;
  if (PPB < 1) PPB = 1;
  const int threads = ((CV * PPB + 31) / 32) * 32;
  long long ctas_per_b = (4LL * num_sms() + B - 1) / B;
  long long pix_per_cta = (HW + ctas_per_b - 1) / ctas_per_b;
  pix_per_cta = ((pix_per_cta + PPB - 1) / PPB) * PPB;
  if (pix_per_cta < PPB) pix_per_cta = PPB;
  const unsigned gx = (unsigned)((HW + pix_per_cta - 1) / pix_per_cta);
  // scratch layout: [1024] uint32 arrival counters at a FIXED offset | [gx*B*groups*2] double partials | [B*groups*2]
  // float (mean, rstd). The counters must be ZERO before the first call and are left at zero by every call (the caller
  // zero-fills the scratch once when it allocates it); they sit in front because gx - and with it the size of the
  // partial region - changes from call to call.
  B200_CHECK_ARG(B <= 1024, "groupnorm: at most 1024 batch elements");
  unsigned int* counters = reinterpret_cast<unsigned int*>(stats);
  long long* dstats = reinterpret_cast<long long*>(reinterpret_cast<char*>(stats) + 4096);
  const long long need = 4096 + (long long)gx * B * groups * 16 + (long long)B * groups * 8;
  B200_CHECK_ARG(need <= stats_bytes, "groupnorm: stats scratch too small (%lld bytes needed)", need);
  B200_CHECK_ARG(groups <= 256 && groups <= threads, "groupnorm: at most min(256, block size) groups");
  float* mr = reinterpret_cast<float*>(dstats + (long long)gx * B * groups * 2);
  dim3 grid(gx, (unsigned)B);
  const size_t smem = std::max((size_t)PPB * 2 * C * sizeof(float), (size_t)threads * 2 * sizeof(double));
  B200_CUDA(launch_pdl(gn_stats_kernel, grid, dim3(threads), smem, st, 1, reinterpret_cast<const __nv_bfloat16*>(x1),
                       (int)C1, reinterpret_cast<const __nv_bfloat16*>(x2), (int)C2, dstats, mr, counters, (long long)HW,
                       (int)groups, PPB, (int)pix_per_cta, 1.0 / (static_cast<double>(HW) * (double)(C / groups)), eps));
  B200_CUDA(launch_pdl(gn_apply_kernel, grid, dim3(threads), 0, st, 1, reinterpret_cast<const __nv_bfloat16*>(x1),
                       (int)C1, reinterpret_cast<const __nv_bfloat16*>(x2), (int)C2, gamma, beta,
                       reinterpret_cast<__nv_bfloat16*>(y), (const float*)mr, (long long)HW, (int)groups, (int)silu, PPB,
                       (int)pix_per_cta));
  return 0;
}

// Row softmax y = softmax(x * scale) for fp32 scores [M, N] -> bf16 probabilities: the attention of the VAE decoder's
// mid block (ONE 512-wide head over H*W tokens, ppdiffusers/models/vae.py:232-241, attention_processor.py:673-735 with
// upcast_softmax) runs as two GEMMs around this kernel because a 512-wide head does not fit the flash kernel's register /
// shared-memory budget. One CTA per row; the row is staged in shared memory (read once), fp32 math, exp2.
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                                          long long N, long long ldx, long long ldy, float scale_log2) {
  extern __shared__ float srow[];
  __shared__ float red[8];
  const float* xr = x + static_cast<long long>(blockIdx.x) * ldx;
  __nv_bfloat16* yr = y + static_cast<long long>(blockIdx.x) * ldy;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float mx = -INFINITY;
  for (long long i = threadIdx.x * 4; i < N; i += blockDim.x * 4) {
    const float4 v = *reinterpret_cast<const float4*>(xr + i);
    *reinterpret_cast<float4*>(srow + i) = v;
    mx = fmaxf(fmaxf(mx, fmaxf(v.x, v.y)), fmaxf(v.z, v.w));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) mx = fmaxf(mx, red[w]);
  __syncthreads();
  const float ms = (mx == -INFINITY) ? 0.0f : mx * scale_log2;
  float sum = 0.0f;
  for (long long i = threadIdx.x * 4; i < N; i += blockDim.x * 4) {
    float4 v = *reinterpret_cast<const float4*>(srow + i);
    v.x = exp2f(fmaf(v.x, scale_log2, -ms)), v.y = exp2f(fmaf(v.y, scale_log2, -ms));
    v.z = exp2f(fmaf(v.z, scale_log2, -ms)), v.w = exp2f(fmaf(v.w, scale_log2, -ms));
    sum += (v.x + v.y) + (v.z + v.w);
    *reinterpret_cast<float4*>(srow + i) = v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  sum = 0.0f;
#pragma unroll
  for (int w = 0; w < 8; ++w) sum += red[w];  // fixed order: bit-reproducible
  const float inv = 1.0f / sum;
  for (long long i = threadIdx.x * 4; i < N; i += blockDim.x * 4) {
    const float4 v = *reinterpret_cast<const float4*>(srow + i);
    uint2 o;
    o.x = pack_bf16x2(v.x * inv, v.y * inv), o.y = pack_bf16x2(v.z * inv, v.w * inv);
    *reinterpret_cast<uint2*>(yr + i) = o;
  }
}

extern "C" int b200mix_softmax_rows(const float* x, void* y, int64_t M, int64_t N, int64_t ldx, int64_t ldy, float scale,
                                    void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(x && y && M > 0 && N > 0, "softmax_rows: bad arguments");
  B200_CHECK_ARG(N % 4 == 0 && ldx % 4 == 0 && ldy % 4 == 0 && N * 4 <= 200 * 1024,
                 "softmax_rows: N, ldx, ldy must be multiples of 4 and N <= 51200");
  B200_CHECK_ARG(reinterpret_cast<uintptr_t>(x) % 16 == 0 && reinterpret_cast<uintptr_t>(y) % 8 == 0,
                 "softmax_rows: pointers must be 16- / 8-byte aligned");
  static bool configured = false;
  if (!configured) {
    B200_CUDA(cudaFuncSetAttribute(softmax_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    configured = true;
  }
  softmax_rows_kernel<<<(unsigned)M, 256, (size_t)N * 4, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, reinterpret_cast<__nv_bfloat16*>(y), N, ldx, ldy, scale * 1.4426950408889634f);
  B200_LAUNCH_CHECK();
  return 0;
}

// Large inputs: block-resident variant. Each CTA owns a contiguous block of rows, fetched into shared memory by four
// 1-D bulk copies (one mbarrier each) so the whole block is in flight at once and no registers hold row data: the grid
// is sized to exactly fill the machine (2 CTAs per SM, a whole number of waves). Each warp then normalises two rows
// per iteration out of shared memory with the same per-lane accumulation order as layernorm_kernel (bit-identical).
constexpr int LN_BLOCK_SMEM_CAP = 104 * 1024;

__global__ void __launch_bounds__(512, 2) layernorm_block_kernel(const LNParams p, int rows_per_cta, int rows_per_chunk) {
  extern __shared__ __align__(128) uint8_t ln_smem[];
  __shared__ uint64_t bars[4];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long r0 = static_cast<long long>(blockIdx.x) * rows_per_cta;
  const int nrows = static_cast<int>(min(static_cast<long long>(rows_per_cta), p.M - r0));
  const uint32_t row_bytes = static_cast<uint32_t>(p.N) * 2u;
  uint8_t* sx = ln_smem;
  uint8_t* sd = ln_smem + static_cast<size_t>(rows_per_cta) * row_bytes;
  if (threadIdx.x == 0) {
#pragma unroll
    for (int c = 0; c < 4; ++c) mbar_init(&bars[c], 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    for (int c = 0; c < 4; ++c) {
      const int cr0 = c * rows_per_chunk;
      if (cr0 >= nrows) break;
      const uint32_t bytes = static_cast<uint32_t>(min(rows_per_chunk, nrows - cr0)) * row_bytes;
      mbar_expect_tx(&bars[c], p.delta ? 2 * bytes : bytes);
      bulk_load_1d(sx + static_cast<size_t>(cr0) * row_bytes, p.x + (r0 + cr0) * p.N, bytes, &bars[c]);
      if (p.delta) bulk_load_1d(sd + static_cast<size_t>(cr0) * row_bytes, p.delta + (r0 + cr0) * p.N, bytes, &bars[c]);
    }
  }
  const int NV = p.N >> 3;
  for (int r = 2 * warp; r < nrows; r += 32) {  // rows_per_chunk is even: a row pair never straddles two chunks
    mbar_wait(&bars[r / rows_per_chunk], 0);
    const int nr = (r + 1 < nrows) ? 2 : 1;
    uint4* srow[2] = {reinterpret_cast<uint4*>(sx + static_cast<size_t>(r) * row_bytes),
                      reinterpret_cast<uint4*>(sx + static_cast<size_t>(r + 1) * row_bytes)};
    float mean[2] = {0.0f, 0.0f}, rstd[2] = {0.0f, 0.0f};
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      if (rr >= nr) break;
      const long long row = r0 + r + rr;
      if (p.delta) {
        const uint4* drow = reinterpret_cast<const uint4*>(sd + static_cast<size_t>(r + rr) * row_bytes);
        const long long g = static_cast<long long>(static_cast<unsigned>(row) / static_cast<unsigned>(p.rows_per_group));
        for (int vi = lane; vi < NV; vi += 32) {
          float v[8], d[8];
          unpack8(srow[rr][vi], v);
          unpack8(drow[vi], d);
          if (p.gate) {
            const float* gp = p.gate + g * p.ld_mod + vi * 8;
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] = fmaf(__ldg(gp + k), d[k], v[k]);
          } else {
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] += d[k];
          }
          const uint4 packed = pack8(v);  // bf16 residual stream: the rounded value is what gets normalised
          srow[rr][vi] = packed;          // only this lane reads these 16 bytes again
          if (p.resid_out) *(reinterpret_cast<uint4*>(p.resid_out + row * p.N) + vi) = packed;
        }
      }
      if (!p.rms) {
        uint64_t acc = 0ull;
        for (int vi = lane; vi < NV; vi += 32) ln_acc_sum(acc, srow[rr][vi]);
        float s = pair_sum(acc);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        mean[rr] = s / p.N;
      }
      const uint64_t nmean2 = pack_f32x2(-mean[rr], -mean[rr]);
      uint64_t acc = 0ull;
      for (int vi = lane; vi < NV; vi += 32) ln_acc_sq(acc, srow[rr][vi], nmean2);
      float sq = pair_sum(acc);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
      rstd[rr] = rsqrtf(sq / p.N + p.eps);
    }
    for (int vi = lane; vi < NV; vi += 32) {
      P8 wv, bv;
      if (p.weight) wv = load8f(p.weight + 8 * vi);
      if (p.bias) bv = load8f(p.bias + 8 * vi);
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        if (rr >= nr) break;
        const long long row = r0 + r + rr;
        const float* sc = nullptr;
        const float* sh = nullptr;
        if (p.scale || p.shift) {
          const long long g = static_cast<long long>(static_cast<unsigned>(row) / static_cast<unsigned>(p.rows_per_group));
          if (p.scale) sc = p.scale + g * p.ld_mod + 8 * vi;
          if (p.shift) sh = p.shift + g * p.ld_mod + 8 * vi;
        }
        *(reinterpret_cast<uint4*>(p.y + row * p.N) + vi) =
            ln_output8(srow[rr][vi], pack_f32x2(-mean[rr], -mean[rr]), pack_f32x2(rstd[rr], rstd[rr]), p.rms != 0,
                       p.weight ? &wv : nullptr, p.bias ? &bv : nullptr, sc, sh);
      }
    }
  }
}

// Test hook (not part of the public header): 1 = always use the register-resident kernel.
static int g_ln_register_only = 0;
extern "C" void b200mix_debug_ln_register_only(int on) { g_ln_register_only = on; }

extern "C" int b200mix_layernorm(const void* x, const void* delta, const float* gate, void* resid_out, void* y,
                                 const float* weight, const float* bias, const float* scale, const float* shift,
                                 int64_t ld_mod, int64_t rows_per_group, int64_t M, int64_t N, float eps, int32_t rms,
                                 void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(x && y, "layernorm: null pointer");
  B200_CHECK_ARG(N % 8 == 0 && N > 0 && N <= 8192, "layernorm: N=%lld must be a multiple of 8 and <= 8192",
                 (long long)N);
  B200_CHECK_ARG(M > 0, "layernorm: M must be positive");
  LNParams p;
  p.x = reinterpret_cast<const __nv_bfloat16*>(x);
  p.delta = reinterpret_cast<const __nv_bfloat16*>(delta);
  p.gate = gate;
  p.resid_out = reinterpret_cast<__nv_bfloat16*>(resid_out);
  p.y = reinterpret_cast<__nv_bfloat16*>(y);
  p.weight = weight, p.bias = bias, p.scale = scale, p.shift = shift;
  p.ld_mod = ld_mod;
  p.rows_per_group = rows_per_group > 0 ? rows_per_group : M;
  p.M = M, p.N = (int)N, p.eps = eps, p.rms = rms;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int nv = (int)(N / 8);
  {
    // block-resident kernel for inputs big enough to fill the machine (same results bit for bit)
    const long long row_bytes = N * 2 * (delta ? 2 : 1);
    const bool aligned = (reinterpret_cast<uintptr_t>(x) % 16 == 0) && (!delta || reinterpret_cast<uintptr_t>(delta) % 16 == 0);
    const long long slots = 2ll * num_sms();
    // only when the whole input is resident in one wave: with several waves the register kernel overlaps better
    if (!g_ln_register_only && aligned && M * row_bytes >= (4ll << 20) && M * row_bytes <= slots * LN_BLOCK_SMEM_CAP) {
      const long long waves = 1;
      long long rpc = (M + slots * waves - 1) / (slots * waves);
      rpc = (rpc + 1) & ~1ll;
      if (rpc * row_bytes > LN_BLOCK_SMEM_CAP) rpc = (LN_BLOCK_SMEM_CAP / row_bytes) & ~1ll;
      long long rchunk = (((rpc + 3) / 4) + 1) & ~1ll;
      const size_t smem = (size_t)(rpc * row_bytes);
      static bool configured = false;
      if (!configured) {
        B200_CUDA(cudaFuncSetAttribute(layernorm_block_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       LN_BLOCK_SMEM_CAP));
        configured = true;
      }
      B200_CUDA(launch_pdl(layernorm_block_kernel, dim3((unsigned)((M + rpc - 1) / rpc)), dim3(512), smem, st, 1, p,
                           (int)rpc, (int)rchunk));
      return 0;
    }
  }
#define LN_LAUNCH(VPL, ROWS)                                                                                      \
  B200_CUDA(launch_pdl(layernorm_kernel<VPL, ROWS>, dim3((unsigned)((M + 8 * ROWS - 1) / (8 * ROWS))), dim3(256), 0, \
                       st, 1, p))
  if (nv <= 32) LN_LAUNCH(1, 8);
  else if (nv <= 64) LN_LAUNCH(2, 8);
  else if (nv <= 96) LN_LAUNCH(3, 4);
  else if (nv <= 128) LN_LAUNCH(4, 4);
  else if (nv <= 160) LN_LAUNCH(5, 3);
  else if (nv <= 192) LN_LAUNCH(6, 2);
  else if (nv <= 256) LN_LAUNCH(8, 2);
  else if (nv <= 512) LN_LAUNCH(16, 1);
  else LN_LAUNCH(32, 1);
#undef LN_LAUNCH
  return 0;
}
