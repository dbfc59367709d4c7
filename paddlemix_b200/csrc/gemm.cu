// Implicit-GEMM on Hopper tensor cores: one persistent, warp-specialised kernel that serves
//   * Linear / 1x1 conv        C[M,N] = A[M,K] W[N,K]^T                       (1 tap)
//   * conv3x3 NHWC, stride 1|2 y = sum_taps shift(x) W_tap^T                  (9 taps, im2col-free)
// Data path: TMA (cp.async.bulk.tensor, 128B swizzle, hardware zero fill for halos / ragged edges) -> shared memory
// ring -> wgmma (bf16 x bf16 -> fp32 register accumulators, 64 x BN x 16 per instruction and consumer warpgroup) ->
// fused epilogue (bias / temb row-add / activation / GEGLU|SwiGLU / AdaLN gate / residual) -> HBM.
//
// CTAs run as clusters of 2 along M: both CTAs of a cluster work on the same n-tile, and each loads one half of the
// weight tile with TMA multicast into both CTAs' shared memory, so the L2 -> SM traffic per MAC drops from
// (128+BN)/(128*BN) to (128+BN/2)/(128*BN). A stage goes back to the producers when every consumer warp of both CTAs
// has arrived on its empty barrier (local arrive + remote arrive through the cluster's shared-memory window).
//
// Replaces (reference): F.linear / F.conv2d call sites ppdiffusers/models/lora.py:365-377,453-459,
// resnet.py:728-808, attention.py:623-677 (FeedForward/GEGLU), and their cuBLASLt / cuDNN kernels inside Paddle.
#include "common.cuh"
#include "ptx.cuh"

#include <algorithm>
#include <cstdlib>
#include <mutex>

namespace b200 {

struct IGemmParams {
  int N;        // accumulator columns (before GLU halving)
  int Kc;       // reduction length per tap (C_in or K)
  int ntaps;    // 1 or 9
  int kchunks;  // ceil(Kc / 64)
  int TW, TH, TB;  // tile box in (x, y, b); TW*TH*TB == 128
  int Wo, Ho, Bn;  // output extents in (x, y, b); plain GEMM: Wo = M, Ho = Bn = 1
  int tiles_x, tiles_y, tiles_b, tiles_n;
  int tap_dc[16], tap_dx[16], tap_p[16], tap_dy[16];
  // fused nearest-2x upsample (b200mix_conv3x3_up2x): m-tiles enumerate (output parity, low-resolution tile); tile
  // `mt` has parity mt / par_tiles and uses taps [4 * parity, 4 * parity + 4); its rows land on output pixels
  // (2y + parity / 2, 2x + parity % 2). par_tiles = tiles per parity rounded up to even (the two CTAs of a cluster share one n-tile).
  int up, par_tiles;
  // epilogue
  const float* bias;
  const float* row_add;
  const float* row_gate;
  long long ld_row;
  int rows_per_group;
  const __nv_bfloat16* residual;
  long long ldr;
  void* C;
  long long ldc;
  int act, glu, out_fp32, vec_ok;
  float out_scale;
  // batched-strided mode (b200mix_linear_batched): row (b, x) of the output lives at C + b*c_bstride + x*ldc and the
  // residual at residual + b*r_bstride + x*ldr; plain mode (c_bstride == 0) uses the flat row index for both.
  long long c_bstride, r_bstride;
  long long res_row_mod;  // > 0: residual row = flat row % res_row_mod (a [rows, N] table shared by all groups)
  // LayerNorm folded into the GEMMs either side of it (b200mix_epilogue: stats_out / ln_stats), see fill_epilogue
  long long* stats_out;       // producer: [M][2] fixed-point (sum, sum of squares) of the bf16 output rows, += by atomics
  const long long* ln_stats;  // consumer: the same table for this GEMM's input rows
  const float* ln_colsum;     // consumer: [N] sum_k W'[n, k]
  int ln_rms;
  float ln_eps;
  float ln_inv_k;             // 2^-24 / K
  // stream-K head (see SegIter): the first sk_tiles super-tiles are cut into equal k-block ranges, one per cluster
  int sk_tiles;
  float4* sk_ws;          // [cluster][cta rank][chunk][8][128 rows] fp32 partial accumulators
  unsigned int* sk_flags; // [cluster][cta rank]: 1 = the partial of that CTA's tail piece is in sk_ws
};

// ---- work schedule -------------------------------------------------------------------------------------------------
// A problem of T super-tiles (256 x BN) on C clusters needs ceil(T / C) rounds; SDXL's 8192 x 1280 projections have
// T = 160 on C = 74: 2.16 rounds of work in 3 rounds of time. The schedule therefore starts with a STREAM-K head: the
// first sk_tiles = C + (T mod C) tiles are laid end to end in units of one 64-deep k-block and cluster c takes the
// contiguous unit range [c, c+1) * units / C (>= one whole tile, so a tile is shared by at most two clusters: its k
// range splits into a HEAD piece = the last piece of cluster c and a TAIL piece = the first piece of cluster c + 1).
// The tail piece's fp32 accumulators go to a per-cluster workspace slot right after that cluster's first few k-blocks;
// the head piece's epilogue - which runs (1 + T mod C / C) tiles later - adds them to its own accumulators and finishes
// the tile (fixed split and fixed order: results are reproducible run to run). The remaining T - sk_tiles tiles (a
// multiple of C) follow round-robin as before. Every cluster thus gets T / C tiles' worth of k-blocks.
constexpr int SK_WS_FLOAT4_PER_CTA = 8 * 8 * 128;  // 8 chunks x 8 float4 x 128 rows = 128 KB
enum { SEG_FULL = 0, SEG_TAIL = 1, SEG_HEAD = 2 };
struct SegIter {
  int u, u1;        // stream-K unit range still to do
  int st_rr, step, total, kblocks;
  int st, kb0, kb1;  // current piece: super-tile and k-block range
  __device__ __forceinline__ SegIter(int sk_tiles, int total_super, int kblocks_, int cluster_id, int num_clusters) {
    const int units = sk_tiles * kblocks_;
    u = static_cast<int>(static_cast<long long>(cluster_id) * units / num_clusters);
    u1 = static_cast<int>(static_cast<long long>(cluster_id + 1) * units / num_clusters);
    st_rr = sk_tiles + cluster_id, step = num_clusters, total = total_super, kblocks = kblocks_;
    st = 0, kb0 = 0, kb1 = 0;
  }
  __device__ __forceinline__ bool next() {
    if (u < u1) {
      st = u / kblocks;
      kb0 = u - st * kblocks;
      kb1 = min(kblocks, kb0 + (u1 - u));
      u += kb1 - kb0;
      return true;
    }
    if (st_rr < total) {
      st = st_rr, kb0 = 0, kb1 = kblocks;
      st_rr += step;
      return true;
    }
    return false;
  }
  __device__ __forceinline__ int mode() const { return kb0 > 0 ? SEG_TAIL : (kb1 < kblocks ? SEG_HEAD : SEG_FULL); }
};
__device__ __forceinline__ unsigned int ld_acquire_gpu(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_gpu(unsigned int* p, unsigned int v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Epilogue activations. All are of the form x * sigmoid(q(x)) and cost one ex2 + one rcp on the MUFU pipe, so a
// GEGLU / SiLU epilogue stays well inside the tensor-core time of its tile.
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float x_sigmoid_neg_log2(float x, float neg_q_log2e) {  // x / (1 + 2^neg_q_log2e)
  return __fdividef(x, 1.0f + ex2_approx(neg_q_log2e));
}
__device__ __forceinline__ float act_silu(float x) { return x_sigmoid_neg_log2(x, -1.4426950408889634f * x); }
// Exact-erf GELU  x * Phi(x)  with  Phi(x) = sigmoid(2 x (c0 + c1 x^2 + c2 x^4)),  coefficients fitted (minimax over
// [-7,7]) so that |gelu_fast - gelu_erf| <= 3.1e-5 absolute: 250x below the bf16 rounding of the output. The quartic
// coefficient is negative, so the polynomial is only evaluated for x^2 <= 49 (ACT_X2_MAX): beyond |x| = 7 the exponent
// continues linearly (slope 2 * 1.788), where both Phi and the sigmoid differ from 0 / 1 by < 1e-12, and it
// saturates to exactly x (x -> +inf) and exactly 0 (x -> -inf: 2^(+big) = inf, x / inf = 0) like erf-GELU does
// (the reference asserts gelu(-100) == 0 and gelu(20) == 20, ppdiffusers/tests/models/test_activations.py:55-63).
constexpr float ACT_X2_MAX = 49.0f;
__device__ __forceinline__ float act_gelu_erf(float x) {
  const float k = -2.0f * 1.4426950408889634f;
  const float c0 = 7.97627599e-01f * k, c1 = 3.69255429e-02f * k, c2 = -3.41174308e-04f * k;
  const float x2 = fminf(x * x, ACT_X2_MAX);
  return x_sigmoid_neg_log2(x, x * fmaf(fmaf(c2, x2, c1), x2, c0));
}
// tanh-GELU: 0.5 x (1 + tanh(u)) == x * sigmoid(2u), u = sqrt(2/pi) (x + 0.044715 x^3)   (identity, not an approximation)
__device__ __forceinline__ float act_gelu_tanh(float x) {
  const float k = -2.0f * 1.4426950408889634f * 0.7978845608028654f;
  return x_sigmoid_neg_log2(x, x * fmaf(k * 0.044715f, x * x, k));
}
__device__ __forceinline__ float act_quick_gelu(float x) { return x_sigmoid_neg_log2(x, -1.702f * 1.4426950408889634f * x); }

// All four share the form x / (1 + 2^(x (c0 + c1 x^2 + c2 x^4))); the coefficients are picked ONCE per kernel so the
// unrolled per-element code is branch-free (a switch per element serialises the 32 MUFU chains of a chunk: measured
// 16 us instead of 5 us per 128x256 tile). With c1 = c2 = 0 the polynomial is exactly c0, so every activation keeps the
// bits of its dedicated function above.
struct ActCoef {
  float c0, c1, c2;
};
__device__ __forceinline__ ActCoef act_coef(int act, int glu) {
  const float l2e = 1.4426950408889634f;
  if (glu == B200MIX_GLU_GEGLU) act = B200MIX_ACT_GELU_ERF;
  else if (glu) act = B200MIX_ACT_SILU;
  ActCoef a = {0.0f, 0.0f, 0.0f};
  switch (act) {
    case B200MIX_ACT_SILU: a.c0 = -l2e; break;
    case B200MIX_ACT_GELU_ERF: {
      const float k = -2.0f * l2e;
      a.c0 = 7.97627599e-01f * k, a.c1 = 3.69255429e-02f * k, a.c2 = -3.41174308e-04f * k;
      break;
    }
    case B200MIX_ACT_GELU_TANH: {
      const float k = -2.0f * l2e * 0.7978845608028654f;
      a.c0 = k, a.c1 = k * 0.044715f;
      break;
    }
    case B200MIX_ACT_QUICK_GELU: a.c0 = -1.702f * l2e; break;
    default: break;
  }
  return a;
}
__device__ __forceinline__ float act_eval(float x, const ActCoef& a) {
  // x^2 is clamped to the range the erf-GELU polynomial was fitted on (see act_gelu_erf); SiLU / quick-GELU have
  // c1 = c2 = 0 and tanh-GELU is saturated to 1 ulp long before |x| = 7, so the clamp changes none of them
  const float x2 = fminf(x * x, ACT_X2_MAX);
  return x_sigmoid_neg_log2(x, x * fmaf(fmaf(a.c2, x2, a.c1), x2, a.c0));
}

// Global-memory operands of one 32-column chunk of one accumulator row.
struct EpiOperands {  // direct (row-per-thread) path: GLU / fp32 output / unaligned or partial chunks
  float4 bias[8];
  bool vec;
};

__device__ __forceinline__ void epilogue_prefetch(const IGemmParams& p, EpiOperands& eo, const float* bias_c, int n_abs) {
  eo.vec = (n_abs + 32 <= p.N) && p.vec_ok;
  if (p.bias) {  // staged in shared memory by this warp (zeros past N)
    const float4* b4 = reinterpret_cast<const float4*>(bias_c);
#pragma unroll
    for (int j = 0; j < 8; ++j) eo.bias[j] = b4[j];
  }
}

// One 32-column chunk of one accumulator row -> global memory.
__device__ __forceinline__ void epilogue_chunk(const IGemmParams& p, const ActCoef& ac, const uint32_t (&r)[32],
                                               const EpiOperands& eo, long long c_off, long long r_off, long long g,
                                               int n_abs) {
  float v[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(r[j]);
  const bool full = (n_abs + 32 <= p.N);
  const bool vec = eo.vec;

  if (p.bias) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      v[4 * j + 0] += eo.bias[j].x, v[4 * j + 1] += eo.bias[j].y, v[4 * j + 2] += eo.bias[j].z,
          v[4 * j + 3] += eo.bias[j].w;
    }
  }
  if (p.row_add) {
    const float* ra = p.row_add + g * p.ld_row + n_abs;
#pragma unroll
    for (int j = 0; j < 32; ++j)
      if (full || n_abs + j < p.N) v[j] += __ldg(ra + j);
  }
  if (p.act != B200MIX_ACT_NONE && !p.glu) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = act_eval(v[j], ac);
  }

  if (p.glu) {
    float o[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) o[j] = v[2 * j] * act_eval(v[2 * j + 1], ac);
    const int ncol = n_abs >> 1;
    const int nout = p.N >> 1;
    if (p.out_fp32) {
      float* dst = reinterpret_cast<float*>(p.C) + c_off + ncol;
#pragma unroll
      for (int j = 0; j < 16; ++j)
        if (ncol + j < nout) dst[j] = o[j];
    } else {
      __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(p.C) + c_off + ncol;
      if (vec) {
        uint4 w0 = make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]),
                              pack_bf16x2(o[6], o[7]));
        uint4 w1 = make_uint4(pack_bf16x2(o[8], o[9]), pack_bf16x2(o[10], o[11]), pack_bf16x2(o[12], o[13]),
                              pack_bf16x2(o[14], o[15]));
        reinterpret_cast<uint4*>(dst)[0] = w0;
        reinterpret_cast<uint4*>(dst)[1] = w1;
      } else {
#pragma unroll
        for (int j = 0; j < 16; ++j)
          if (ncol + j < nout) dst[j] = __float2bfloat16(o[j]);
      }
    }
    return;
  }

  if (p.row_gate) {
    const float* rg = p.row_gate + g * p.ld_row + n_abs;
#pragma unroll
    for (int j = 0; j < 32; ++j)
      if (full || n_abs + j < p.N) v[j] *= __ldg(rg + j);
  }
  if (p.residual) {
    if (vec) {
      const uint4* rs4 = reinterpret_cast<const uint4*>(p.residual + r_off + n_abs);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint4 w = __ldg(rs4 + j);
        v[8 * j + 0] += bf16_lo(w.x), v[8 * j + 1] += bf16_hi(w.x);
        v[8 * j + 2] += bf16_lo(w.y), v[8 * j + 3] += bf16_hi(w.y);
        v[8 * j + 4] += bf16_lo(w.z), v[8 * j + 5] += bf16_hi(w.z);
        v[8 * j + 6] += bf16_lo(w.w), v[8 * j + 7] += bf16_hi(w.w);
      }
    } else {
      const __nv_bfloat16* rs = p.residual + r_off + n_abs;
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (n_abs + j < p.N) v[j] += __bfloat162float(rs[j]);
    }
  }
  if (p.out_scale != 1.0f) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] *= p.out_scale;
  }

  if (p.out_fp32) {
    float* dst = reinterpret_cast<float*>(p.C) + c_off + n_abs;
    if (vec) {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        reinterpret_cast<float4*>(dst)[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (n_abs + j < p.N) dst[j] = v[j];
    }
  } else {
    __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(p.C) + c_off + n_abs;
    if (vec) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        uint4 w = make_uint4(pack_bf16x2(v[8 * j], v[8 * j + 1]), pack_bf16x2(v[8 * j + 2], v[8 * j + 3]),
                             pack_bf16x2(v[8 * j + 4], v[8 * j + 5]), pack_bf16x2(v[8 * j + 6], v[8 * j + 7]));
        reinterpret_cast<uint4*>(dst)[j] = w;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (n_abs + j < p.N) dst[j] = __float2bfloat16(v[j]);
    }
  }
}

// ---- coalesced epilogue (bf16 output, no GLU, aligned full chunk) -------------------------------------------------
// The epilogue hands every thread one accumulator ROW (32 consecutive columns = 64 bytes of bf16). Writing / reading
// global memory in that shape makes each lane of a 16-byte access hit a different 128-byte line (32 L1 wavefronts per
// instruction). The chunk is therefore transposed through a 2 KB per-warp shared-memory buffer so that a warp's
// global access covers 8 rows x 64 contiguous bytes (8 wavefronts): 4 lanes per row, lane L -> row s*8 + L/4,
// 16-byte piece L%4. The buffer is XOR-swizzled (piece ^ ((row >> 1) & 3)) so both access patterns are conflict-free.
struct RowMap {          // global offsets (16-byte units) of the 4 rows this lane touches in the transposed pattern
  uint32_t c16[4];
  uint32_t r16[4];
  uint32_t valid;        // bit s4 set = row s4 exists
};

__device__ __forceinline__ uint32_t stage_addr(int row, int piece) {
  return static_cast<uint32_t>(row * 64 + ((piece ^ ((row >> 1) & 3)) << 4));
}

__device__ __forceinline__ void epilogue_prefetch_staged(const IGemmParams& p, uint4 (&resv)[4], const RowMap& rm,
                                                         int lane, int n_abs) {
  if (p.residual) {
    const uint4* base = reinterpret_cast<const uint4*>(p.residual + n_abs) + (lane & 3);
#pragma unroll
    for (int s4 = 0; s4 < 4; ++s4)
      resv[s4] = ((rm.valid >> s4) & 1u) ? __ldg(base + rm.r16[s4]) : make_uint4(0u, 0u, 0u, 0u);
  }
}

template <bool STATS>
__device__ __forceinline__ void epilogue_chunk_staged(const IGemmParams& p, const ActCoef& ac, const uint32_t (&r)[32],
                                                      const uint4 (&resv)[4], const float* bias_c, const RowMap& rm,
                                                      uint8_t* stage, int lane, long long g, int n_abs, uint64_t (&st)[2]) {
  float v[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(r[j]);
  if (p.bias) {
    const float4* b4 = reinterpret_cast<const float4*>(bias_c);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float4 a = b4[j];
      v[4 * j + 0] += a.x, v[4 * j + 1] += a.y, v[4 * j + 2] += a.z, v[4 * j + 3] += a.w;
    }
  }
  if (p.row_add) {
    const float4* ra = reinterpret_cast<const float4*>(p.row_add + g * p.ld_row + n_abs);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float4 a = __ldg(ra + j);
      v[4 * j + 0] += a.x, v[4 * j + 1] += a.y, v[4 * j + 2] += a.z, v[4 * j + 3] += a.w;
    }
  }
  if (p.act != B200MIX_ACT_NONE) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = act_eval(v[j], ac);
  }
  if (p.row_gate) {
    const float4* rg = reinterpret_cast<const float4*>(p.row_gate + g * p.ld_row + n_abs);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float4 a = __ldg(rg + j);
      v[4 * j + 0] *= a.x, v[4 * j + 1] *= a.y, v[4 * j + 2] *= a.z, v[4 * j + 3] *= a.w;
    }
  }
  const int piece = lane & 3;
  if (p.residual) {
    // transposed (coalesced) residual pieces -> smem -> this thread's own row
#pragma unroll
    for (int s4 = 0; s4 < 4; ++s4)
      *reinterpret_cast<uint4*>(stage + stage_addr(s4 * 8 + (lane >> 2), piece)) = resv[s4];
    __syncwarp();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint4 w = *reinterpret_cast<const uint4*>(stage + stage_addr(lane, j));
      v[8 * j + 0] += bf16_lo(w.x), v[8 * j + 1] += bf16_hi(w.x);
      v[8 * j + 2] += bf16_lo(w.y), v[8 * j + 3] += bf16_hi(w.y);
      v[8 * j + 4] += bf16_lo(w.z), v[8 * j + 5] += bf16_hi(w.z);
      v[8 * j + 6] += bf16_lo(w.w), v[8 * j + 7] += bf16_hi(w.w);
    }
    __syncwarp();
  }
  if (p.out_scale != 1.0f) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] *= p.out_scale;
  }
  // own row -> smem -> transposed (coalesced) global stores
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint4 w = make_uint4(pack_bf16x2(v[8 * j], v[8 * j + 1]), pack_bf16x2(v[8 * j + 2], v[8 * j + 3]),
                               pack_bf16x2(v[8 * j + 4], v[8 * j + 5]), pack_bf16x2(v[8 * j + 6], v[8 * j + 7]));
    *reinterpret_cast<uint4*>(stage + stage_addr(lane, j)) = w;
    if (STATS) {  // row statistics of the ROUNDED values (what the consumer of this tensor reads), packed fp32 pairs
      const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const uint64_t ab = pack_f32x2(bf16_lo(ww[u]), bf16_hi(ww[u]));
        st[0] = fadd2(st[0], ab);
        st[1] = ffma2(ab, ab, st[1]);
      }
    }
  }
  __syncwarp();
  uint4* cbase = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.C) + n_abs) + piece;
#pragma unroll
  for (int s4 = 0; s4 < 4; ++s4) {
    const uint4 w = *reinterpret_cast<const uint4*>(stage + stage_addr(s4 * 8 + (lane >> 2), piece));
    if ((rm.valid >> s4) & 1u) cbase[rm.c16[s4]] = w;
  }
  __syncwarp();
}

// MCAST = the two CTAs of a cluster work on the same n-tile and each loads one half of the B tile with TMA multicast into
// both CTAs' shared memory, so the L2 -> SM traffic per MAC drops from (128+BN)/(128*BN) to (128+BN/2)/(128*BN).
// !MCAST = every CTA loads its whole B tile itself (no cluster); the tile schedule is the same.
template <int BN>
struct IGemmCfg {
  static constexpr int A_BYTES = 128 * 128;  // 128 rows x 64 bf16 (128 B per row, SW128)
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  // fp32 staging of 64 accumulator columns of one warpgroup's 64 rows; the row stride of 68 floats makes the row-wise
  // float4 reads of the epilogue conflict-free
  static constexpr int ACC_LD = 68;
  static constexpr int ACC_BYTES = 2 * 64 * ACC_LD * 4;
  // barriers | accumulator staging | 8 epilogue warps x 2 KB transpose buffers | 8 x 128 bias + 8 x 128 column sums
  static constexpr int EXTRA_BYTES = 1024 + 256 + ACC_BYTES + 8 * 2048 + 2 * 8 * 512;
};

// Roles (288 threads): warps 0-7 = two consumer warpgroups, warp 8 = TMA producer (one elected lane). Consumer
// warpgroup g multiplies rows [64 g, 64 g + 64) of the 128-row tile (wgmma m64 x BN x k16, accumulators in registers)
// and then runs the epilogue of those rows: 64 accumulator columns at a time go through shared memory so that every
// thread owns 32 consecutive columns of one row (warp w of the group: rows 32 (w & 1) + lane, chunk parity w >> 1).
constexpr int IG_THREADS = 288;
constexpr int IG_WARP_TMA = 8;

// LNM: the folded-LayerNorm epilogues are separate instantiations - the plain kernel carries none of their code.
enum { LNM_NONE = 0, LNM_CONSUMER = 1, LNM_PRODUCER = 2 };
template <int BN, int STAGES, bool MCAST, int LNM>
__global__ void __launch_bounds__(IG_THREADS, 1)
    igemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ IGemmParams p) {
  using Cfg = IGemmCfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  float* acc_all = reinterpret_cast<float*>(smem + STAGES * Cfg::STAGE_BYTES + 256);
  uint8_t* stage_all = reinterpret_cast<uint8_t*>(acc_all) + Cfg::ACC_BYTES;
  float* bias_all = reinterpret_cast<float*>(stage_all + 8 * 2048);  // 8 epilogue warps x 128 floats (their 4 chunks)
  float* colsum_all = bias_all + 8 * 128;                            // same layout: folded-LayerNorm column sums

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], MCAST ? 16 : 8);  // every consumer warp of every CTA that reads the stage
    }
    fence_barrier_init();
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
  }
  __syncthreads();
  if (MCAST) cluster_sync_all();  // barrier inits of both CTAs visible before any multicast TMA / remote arrival
  // everything above overlapped the tail of the previous kernel; from here on we touch its outputs
  pdl_wait();
  pdl_launch_dependents();

  const uint32_t cta_rank = MCAST ? cluster_ctarank() : (blockIdx.x & 1u);
  const int cluster_id = blockIdx.x >> 1;
  const int num_clusters = gridDim.x >> 1;
  const int tiles_m = p.up ? 4 * p.par_tiles : p.tiles_x * p.tiles_y * p.tiles_b;
  const int tiles_m2 = (tiles_m + 1) >> 1;            // pairs of m-tiles (the odd one out pairs with a phantom)
  const int total_super = tiles_m2 * p.tiles_n;
  const int kblocks = p.ntaps * p.kchunks;

  if (warp == IG_WARP_TMA) {
    // ===== TMA producer (whole warp runs the loop, one elected lane issues: see elect_one_sync) =====
    int stage = 0;
    uint32_t phase = 0;
    for (SegIter seg(p.sk_tiles, total_super, kblocks, cluster_id, num_clusters); seg.next();) {
      const int st = seg.st;
      const int mp = st / p.tiles_n, nt = st - mp * p.tiles_n;
      int mt = mp * 2 + (int)cta_rank;  // may be == tiles_m (phantom): its A box is out of bounds -> zeros
      int tap_base = 0;
      if (p.up) {  // phantom tiles of a parity (index >= tiles of the grid) get b0 >= Bn: zeros as well
        const int par = mt / p.par_tiles;
        mt -= par * p.par_tiles, tap_base = par * 4;
      }
      const int tx = mt % p.tiles_x;
      const int ty = (mt / p.tiles_x) % p.tiles_y;
      const int tb = mt / (p.tiles_x * p.tiles_y);
      const int x0 = tx * p.TW, y0 = ty * p.TH, b0 = tb * p.TB, n0 = nt * BN;
      int tap = seg.kb0 / p.kchunks, kc = seg.kb0 - tap * p.kchunks;
      for (int kb = seg.kb0; kb < seg.kb1; ++kb) {
        const int tg = tap_base + tap;
        const int dc = p.tap_dc[tg], dx = p.tap_dx[tg], pp = p.tap_p[tg], dy = p.tap_dy[tg];
        // MCAST: the peer CTA's consumers release this stage too (remote arrivals)
        if (MCAST) mbar_wait_cluster(&empty_bar[stage], phase ^ 1);
        else mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* sA = smem + stage * Cfg::STAGE_BYTES;
        uint8_t* sB = sA + Cfg::A_BYTES;
        if (elect_one_sync()) {
          mbar_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
          tma_load_5d(sA, &tmA, &full_bar[stage], kc * 64 + dc, x0 + dx, pp, y0 + dy, b0);
          if (MCAST) {
            // my half of the weight tile, delivered to both CTAs of the cluster
            tma_load_2d_mcast(sB + cta_rank * (Cfg::B_BYTES / 2), &tmB, &full_bar[stage], tg * p.Kc + kc * 64,
                              n0 + (int)cta_rank * (BN / 2), (uint16_t)0x3);
          } else {
            tma_load_2d(sB, &tmB, &full_bar[stage], tg * p.Kc + kc * 64, n0);
            tma_load_2d(sB + Cfg::B_BYTES / 2, &tmB, &full_bar[stage], tg * p.Kc + kc * 64, n0 + BN / 2);
          }
        }
        __syncwarp();
        if (++stage == STAGES) stage = 0, phase ^= 1;
        if (++kc == p.kchunks) kc = 0, ++tap;
      }
    }
  } else {
    // ===== consumers: MMA of 64 rows, then their epilogue =====
    const int grp = warp >> 2, w = warp & 3;
    const int q = 2 * grp + (w & 1);  // 32-row quarter of the tile this warp's epilogue owns
    const int wg = w >> 1;            // its 32-column chunks are c == wg (mod 2)
    uint8_t* stage = stage_all + warp * 2048;
    float* bias_s = bias_all + warp * 128;
    float* colsum_s = colsum_all + warp * 128;
    float* sacc = acc_all + grp * 64 * Cfg::ACC_LD;
    const ActCoef ac = act_coef(p.act, p.glu);
    const bool staged_ok = p.vec_ok && !p.glu && !p.out_fp32 && ((p.c_bstride | p.r_bstride) & 7) == 0;
    const int row = q * 32 + lane;
    const int tw = row % p.TW;
    const int th = (row / p.TW) % p.TH;
    const int tbb = row / (p.TW * p.TH);
    const uint32_t peer_empty = MCAST ? mapa_smem(&empty_bar[0], cta_rank ^ 1u) : 0u;
    int kstage = 0;
    uint32_t kphase = 0;
    const int epi_tid = warp * 32 + lane;
    auto release = [&](int s) {  // this warp's wgmma reads of stage s are complete
      if (lane == 0) {
        mbar_arrive(&empty_bar[s]);
        if (MCAST) mbar_arrive_cluster(peer_empty + 8u * s);
      }
    };
    for (SegIter seg(p.sk_tiles, total_super, kblocks, cluster_id, num_clusters); seg.next();) {
      float acc[BN / 2];
      {
        int prev = -1;
        for (int kb = seg.kb0; kb < seg.kb1; ++kb) {
          mbar_wait(&full_bar[kstage], kphase);
          const uint32_t a_addr = smem_u32(smem + kstage * Cfg::STAGE_BYTES) + grp * 64 * 128;
          const uint32_t b_addr = smem_u32(smem + kstage * Cfg::STAGE_BYTES + Cfg::A_BYTES);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k)  // a piece starts from zero
            wgmma_ss(acc, make_wgmma_desc_sw128(a_addr + k * 32, 16, 1024), make_wgmma_desc_sw128(b_addr + k * 32, 16, 1024),
                     (kb != seg.kb0 || k != 0) ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<1>();  // the previous k-block's MMAs are done: its stage goes back to the producer(s)
          wgmma_fence_operands(acc);
          if (prev >= 0) release(prev);
          prev = kstage;
          if (++kstage == STAGES) kstage = 0, kphase ^= 1;
        }
        wgmma_wait<0>();
        wgmma_fence_operands(acc);
        release(prev);
      }

      const int st = seg.st;
      const int seg_mode = seg.mode();
      // stream-K pieces: the tail piece (my first) goes to MY workspace slot; the head piece (my last) is completed with
      // the tail piece of the same tile, which the NEXT cluster produced at its very start
      const int sk_slot = (seg_mode == SEG_TAIL ? cluster_id : cluster_id + 1) * 2 + (int)cta_rank;
      float4* sk_ws = p.sk_ws + static_cast<size_t>(sk_slot) * SK_WS_FLOAT4_PER_CTA + (q * 32 + lane);
      const int mp = st / p.tiles_n, nt = st - mp * p.tiles_n;
      int mt = mp * 2 + (int)cta_rank;
      const bool in_range = mt < tiles_m;
      int par = 0;
      if (p.up) par = mt / p.par_tiles, mt -= par * p.par_tiles;
      const int tx = mt % p.tiles_x;
      const int ty = (mt / p.tiles_x) % p.tiles_y;
      const int tb = mt / (p.tiles_x * p.tiles_y);
      const int x = tx * p.TW + tw, y = ty * p.TH + th, b = tb * p.TB + tbb;
      const bool valid = in_range && (x < p.Wo) && (y < p.Ho) && (b < p.Bn);
      const long long gm = p.up ? (static_cast<long long>(b) * (2 * p.Ho) + (2 * y + (par >> 1))) * (2 * p.Wo) + (2 * x + (par & 1))
                                : (static_cast<long long>(b) * p.Ho + y) * p.Wo + x;
      long long g, c_off, r_off;
      if (p.c_bstride) {  // batched-strided: group == batch
        g = b;
        c_off = static_cast<long long>(b) * p.c_bstride + static_cast<long long>(x) * p.ldc;
        r_off = static_cast<long long>(b) * p.r_bstride + static_cast<long long>(x) * p.ldr;
      } else {
        g = gm / p.rows_per_group;
        c_off = gm * p.ldc;
        r_off = (p.res_row_mod > 0 ? gm % p.res_row_mod : gm) * p.ldr;
      }
      // rows outside the problem (phantom m-tile of an odd pair, rows past M) still run the warp-collective epilogue:
      // give them group 0 so their row_add / row_gate reads stay inside the [groups, N] tables (nothing is stored)
      if (!valid) g = 0;
      const int n0 = nt * BN;
      RowMap rm;  // offsets are multiples of 8 elements whenever staged_ok (vec_ok: 16-byte aligned rows)
      rm.valid = 0;
#pragma unroll
      for (int s4 = 0; s4 < 4; ++s4) {
        const int src = s4 * 8 + (lane >> 2);
        rm.c16[s4] = __shfl_sync(0xffffffffu, static_cast<uint32_t>(c_off >> 3), src);
        rm.r16[s4] = __shfl_sync(0xffffffffu, static_cast<uint32_t>(r_off >> 3), src);
        rm.valid |= (__shfl_sync(0xffffffffu, valid ? 1u : 0u, src) & 1u) << s4;
      }
      // this warp's bias values (its <= 4 chunks of the tile) go to shared memory, read back as broadcast float4s.
      // Folded LayerNorm (consumer side): y = rstd * (acc - mean * colsum[n]) + bias'[n] needs the column sums the same
      // way plus this row's fixed-point totals. ALL of these loads are issued before any of them is consumed, so a tile's
      // preparation costs one L2 round trip, not three.
      constexpr int NI = (BN / 32 + 1) / 2;
      float bias_r[NI], cs_r[NI];
      longlong2 t_stats = make_longlong2(0ll, 0ll);
      if (p.bias) {
#pragma unroll
        for (int i = 0; i < NI; ++i) {
          const int col = n0 + (wg + 2 * i) * 32 + lane;
          bias_r[i] = (wg + 2 * i < BN / 32 && col < p.N) ? __ldg(p.bias + col) : 0.0f;
        }
      }
      if (LNM == LNM_CONSUMER) {
#pragma unroll
        for (int i = 0; i < NI; ++i) {
          const int col = n0 + (wg + 2 * i) * 32 + lane;
          cs_r[i] = (wg + 2 * i < BN / 32 && col < p.N) ? __ldg(p.ln_colsum + col) : 0.0f;
        }
        t_stats = __ldg(reinterpret_cast<const longlong2*>(p.ln_stats) + (valid ? gm : 0ll));
      }
      if (p.bias) {
#pragma unroll
        for (int i = 0; i < NI; ++i) bias_s[i * 32 + lane] = bias_r[i];
      }
      if (LNM == LNM_CONSUMER) {
#pragma unroll
        for (int i = 0; i < NI; ++i) colsum_s[i * 32 + lane] = cs_r[i];
      }
      __syncwarp();
      float ln_rstd = 1.0f, ln_shift = 0.0f;
      if (LNM == LNM_CONSUMER) {  // mean / rstd of my row from the totals the producing GEMM's epilogues accumulated
        // fp32 on purpose (FP64 is slow on the epilogue's critical path). E[x^2] - mean^2 in fp32 is good to
        // ~1e-7 * mean^2 / var relative: below the bf16 resolution of the inputs themselves for any row bf16 can
        // represent (|mean| / std < 2^8).
        const float mean = p.ln_rms ? 0.0f : __ll2float_rn(t_stats.x) * p.ln_inv_k;
        const float var = fmaxf(fmaf(-mean, mean, __ll2float_rn(t_stats.y) * p.ln_inv_k), 0.0f);
        ln_rstd = rsqrtf(var + p.ln_eps);
        ln_shift = -ln_rstd * mean;
      }
      uint64_t st_acc[2] = {0ull, 0ull};  // producer side: packed (even, odd column) sum / sum of squares of my row over my chunks
      uint4 res_cur[4];
      bool st_cur = staged_ok && n0 + wg * 32 + 32 <= p.N;
      if (seg_mode == SEG_HEAD) {
        // the partner's partial was published ~a tile ago; a bounded spin (2^35 cycles, ~18 s: far beyond any time slice
        // the context can lose) turns a scheduling accident (the partner cluster never resident) into an error instead
        // of a hang
        const unsigned int* flag = p.sk_flags + sk_slot;
        const long long t_start = clock64();
        while (ld_acquire_gpu(flag) == 0u) {
          if (clock64() - t_start > (1ll << 35)) __trap();
        }
      }
      const int l4 = lane >> 2, lm = lane & 3;
#pragma unroll
      for (int i = 0; i < (BN + 63) / 64; ++i) {
        // columns [64 i, 64 i + 64) of the warpgroup's 64 rows: fragments -> shared memory -> one row per thread
        named_bar_sync(2 + grp, 128);  // the previous pair of chunks has been read
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int j = 8 * i + jj;  // n8 block of the accumulator fragment
          if (j < BN / 8) {
            float* d0 = sacc + (w * 16 + l4) * Cfg::ACC_LD + jj * 8 + 2 * lm;
            *reinterpret_cast<float2*>(d0) = make_float2(acc[4 * j], acc[4 * j + 1]);
            *reinterpret_cast<float2*>(d0 + 8 * Cfg::ACC_LD) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
          }
        }
        named_bar_sync(2 + grp, 128);
        const int c = 2 * i + wg;
        if (c >= BN / 32) continue;
        uint32_t r[32];
        {
          const float4* src = reinterpret_cast<const float4*>(sacc + (32 * (w & 1) + lane) * Cfg::ACC_LD + wg * 32);
#pragma unroll
          for (int t = 0; t < 8; ++t) {
            const float4 v4 = src[t];
            r[4 * t] = __float_as_uint(v4.x), r[4 * t + 1] = __float_as_uint(v4.y);
            r[4 * t + 2] = __float_as_uint(v4.z), r[4 * t + 3] = __float_as_uint(v4.w);
          }
        }
        const int n_abs = n0 + c * 32;
        if (seg_mode == SEG_TAIL) {  // partial accumulators -> workspace (512 contiguous bytes per warp and store)
#pragma unroll
          for (int j = 0; j < 8; ++j)
            __stcg(sk_ws + (c * 8 + j) * 128, make_float4(__uint_as_float(r[4 * j]), __uint_as_float(r[4 * j + 1]),
                                                          __uint_as_float(r[4 * j + 2]), __uint_as_float(r[4 * j + 3])));
          continue;
        }
        if (seg_mode == SEG_HEAD) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float4 part = __ldcg(sk_ws + (c * 8 + j) * 128);
            r[4 * j + 0] = __float_as_uint(__uint_as_float(r[4 * j + 0]) + part.x);
            r[4 * j + 1] = __float_as_uint(__uint_as_float(r[4 * j + 1]) + part.y);
            r[4 * j + 2] = __float_as_uint(__uint_as_float(r[4 * j + 2]) + part.z);
            r[4 * j + 3] = __float_as_uint(__uint_as_float(r[4 * j + 3]) + part.w);
          }
        }
        if (LNM == LNM_CONSUMER) {
          const float4* c4 = reinterpret_cast<const float4*>(colsum_s + (c >> 1) * 32);
          const uint64_t rstd2 = pack_f32x2(ln_rstd, ln_rstd), shift2 = pack_f32x2(ln_shift, ln_shift);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float4 cs = c4[j];
            float a, bb;
            unpack_f32x2(ffma2(pack_f32x2(__uint_as_float(r[4 * j + 0]), __uint_as_float(r[4 * j + 1])), rstd2,
                               fmul2(shift2, pack_f32x2(cs.x, cs.y))), a, bb);
            r[4 * j + 0] = __float_as_uint(a), r[4 * j + 1] = __float_as_uint(bb);
            unpack_f32x2(ffma2(pack_f32x2(__uint_as_float(r[4 * j + 2]), __uint_as_float(r[4 * j + 3])), rstd2,
                               fmul2(shift2, pack_f32x2(cs.z, cs.w))), a, bb);
            r[4 * j + 2] = __float_as_uint(a), r[4 * j + 3] = __float_as_uint(bb);
          }
        }
        if (st_cur) {  // warp-uniform: coalesced path through the transpose buffer
          epilogue_prefetch_staged(p, res_cur, rm, lane, n_abs);
          epilogue_chunk_staged<LNM == LNM_PRODUCER>(p, ac, r, res_cur, bias_s + (c >> 1) * 32, rm, stage, lane, g, n_abs, st_acc);
          st_cur = (c + 2 < BN / 32) && (n_abs + 96 <= p.N);
        } else {
          const bool active = valid && n_abs < p.N;
          EpiOperands eo;
          if (active) epilogue_prefetch(p, eo, bias_s + (c >> 1) * 32, n_abs);
          if (active) epilogue_chunk(p, ac, r, eo, c_off, r_off, g, n_abs);
        }
      }
      if (LNM == LNM_PRODUCER && seg_mode != SEG_TAIL && valid) {
        // 2^24 fixed point: integer adds commute, so the row totals are the same bits whatever order the tiles finish in
        float s0, s1, q0, q1;
        unpack_f32x2(st_acc[0], s0, s1);
        unpack_f32x2(st_acc[1], q0, q1);
        unsigned long long* dst = reinterpret_cast<unsigned long long*>(p.stats_out + 2 * gm);
        atomicAdd(dst, static_cast<unsigned long long>(__float2ll_rn((s0 + s1) * 16777216.0f)));
        atomicAdd(dst + 1, static_cast<unsigned long long>(__float2ll_rn((q0 + q1) * 16777216.0f)));
      }
      if (seg_mode != SEG_FULL) {
        // tail: all 256 consumer threads' partials are visible device-wide before the flag goes up;
        // head: everybody has read the partial before the flag is lowered for the next launch
        if (seg_mode == SEG_TAIL) __threadfence();
        named_bar_sync(1, 256);
        if (epi_tid == 0) {
          if (seg_mode == SEG_TAIL) st_release_gpu(p.sk_flags + sk_slot, 1u);
          else p.sk_flags[sk_slot] = 0u;
        }
      }
    }
  }

  __syncthreads();
  if (MCAST) cluster_sync_all();  // the peer may still multicast into my smem / arrive on my barriers until it is done too
}

// ------------------------------------------------------------------------------------------------------------
// Skinny-M Linear (M <= 8 activation rows: single-token decode steps, the UNet's time / text-time embedding MLPs):
// the work is streaming W once from HBM, so this is a CUDA-core weight-streaming kernel, not a tensor-core tile (a
// 256-row MMA tile would spend 97 % of its rows on zeros: round 1 measured 1.2 TB/s of weight reads through igemm).
//   * one warp owns SK_R = 4 consecutive output rows (two GLU pairs when the rows are interleaved value / gate); every
//     lane streams 16-byte pieces of the four weight rows (512 coalesced bytes per warp and row, the next k-step's
//     loads are issued before the current one is consumed: 8 x 16 B in flight per lane);
//   * the CTA's K range of the activations is staged ONCE in shared memory as fp32, laid out so that a warp's
//     LDS.128 is conflict-free ([k-step][half][lane][4]); one shared-memory read feeds four weight rows;
//   * K is split over the CTAs of a thread-block cluster (1-8) when the N direction alone cannot fill the machine or
//     the K range does not fit shared memory; the partial sums travel to the cluster's first CTA through distributed
//     shared memory and are added in rank order (deterministic, no workspace, no atomics);
//   * products accumulate on packed fp32 pairs (FFMA2), one butterfly reduction per (row, activation row) at the end.
// Bound: HBM (N * K * 2 bytes of weights); epilogue = bias / activation / GLU / residual / fp32 output.
// ------------------------------------------------------------------------------------------------------------
constexpr int SK_R = 4;                 // output rows per warp
constexpr int SK_ROWS_PER_CTA = 8 * SK_R;
constexpr int SK_SMEM_FLOATS = 24576;   // 96 KB of staged activations per CTA (two CTAs per SM)
constexpr int SK_MAX_SPLITS = 8;

__device__ __forceinline__ void sk_unpack8(const uint4& w, uint64_t (&p)[4]) {
  p[0] = pack_f32x2(bf16_lo(w.x), bf16_hi(w.x)), p[1] = pack_f32x2(bf16_lo(w.y), bf16_hi(w.y));
  p[2] = pack_f32x2(bf16_lo(w.z), bf16_hi(w.z)), p[3] = pack_f32x2(bf16_lo(w.w), bf16_hi(w.w));
}
#ifndef SK_PREFETCH
#define SK_PREFETCH 4  // k-steps (of 256 elements per row) the L2 prefetch window runs ahead of the register loads
#endif
// weights are read exactly once: no L1 allocation
__device__ __forceinline__ uint4 ldg_stream(const __nv_bfloat16* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ void st_shared_cluster_f32(uint32_t cluster_addr, float v) {
  asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(cluster_addr), "f"(v) : "memory");
}

template <int M>
__global__ void __launch_bounds__(256, M <= 4 ? 2 : 1)
    skinny_linear_kernel(const __nv_bfloat16* __restrict__ A, long long lda, const __nv_bfloat16* __restrict__ W,
                         long long ldw, void* __restrict__ C, long long ldc, int N, int K, const float* __restrict__ bias,
                         const __nv_bfloat16* __restrict__ residual, long long ldr, int act, int glu, int out_fp32,
                         int rows,     // rows <= M: the template rounds the row count up (zero rows are staged for the rest)
                         int splits,   // cluster size = number of K ranges
                         int kpart,    // K elements per cluster rank (multiple of 256)
                         int ksm) {    // K elements staged per pass (multiple of 256, <= SK_SMEM_FLOATS / M)
  extern __shared__ __align__(16) float sA[];  // [M][ksm], element (step, lane, j) at step * 256 + (j / 4) * 128 + lane * 4 + j % 4
  __shared__ float red[SK_MAX_SPLITS][8][M * SK_R];
  pdl_wait();
  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rank = splits > 1 ? (int)cluster_ctarank() : 0;
  const int n0 = ((int)(blockIdx.x / splits) * 8 + warp) * SK_R;
  const __nv_bfloat16* w[SK_R];
#pragma unroll
  for (int r = 0; r < SK_R; ++r) w[r] = W + static_cast<long long>(min(n0 + r, N - 1)) * ldw;  // clamped: results of rows >= N are dropped
  uint64_t acc[M][SK_R];
#pragma unroll
  for (int m = 0; m < M; ++m)
#pragma unroll
    for (int r = 0; r < SK_R; ++r) acc[m][r] = 0ull;
  const int kend = min(K, (rank + 1) * kpart);
  for (int k0 = rank * kpart; k0 < kend; k0 += ksm) {
    const int kc = min(ksm, kend - k0);
    // the weight stream does not depend on the staged activations: first loads and the L2 prefetch window go out first
    int kk = lane * 8;
    uint4 cur[SK_R];
    if (kk < kc) {
#pragma unroll
      for (int r = 0; r < SK_R; ++r) cur[r] = ldg_stream(w[r] + k0 + kk);
    }
#pragma unroll
    for (int d = 1; d <= SK_PREFETCH; ++d)
      if (kk + 256 * d < kc) {
#pragma unroll
        for (int r = 0; r < SK_R; ++r) prefetch_l2(w[r] + k0 + kk + 256 * d);
      }
    __syncthreads();
    for (int i = threadIdx.x * 8; i < M * kc; i += 256 * 8) {  // stage A[:, k0 : k0 + kc] as fp32 (kc % 8 == 0)
      const int m = i / kc, k = i - m * kc;
      const uint4 v = m < rows ? __ldg(reinterpret_cast<const uint4*>(A + m * lda + k0 + k)) : make_uint4(0u, 0u, 0u, 0u);
      float* d = sA + m * ksm + (k >> 8) * 256 + ((k & 255) >> 3) * 4;
      *reinterpret_cast<float4*>(d) = make_float4(bf16_lo(v.x), bf16_hi(v.x), bf16_lo(v.y), bf16_hi(v.y));
      *reinterpret_cast<float4*>(d + 128) = make_float4(bf16_lo(v.z), bf16_hi(v.z), bf16_lo(v.w), bf16_hi(v.w));
    }
    __syncthreads();
    for (; kk < kc; kk += 256) {
      uint4 nxt[SK_R];
      if (kk + 256 < kc) {
#pragma unroll
        for (int r = 0; r < SK_R; ++r) nxt[r] = ldg_stream(w[r] + k0 + kk + 256);
      }
      if (kk + 256 * (SK_PREFETCH + 1) < kc) {
#pragma unroll
        for (int r = 0; r < SK_R; ++r) prefetch_l2(w[r] + k0 + kk + 256 * (SK_PREFETCH + 1));
      }
#ifdef SK_NO_MATH  // diagnostic build: the weight stream alone (loads kept alive by an integer fold), no products
#pragma unroll
      for (int r = 0; r < SK_R; ++r) acc[0][r] ^= (uint64_t)(cur[r].x ^ cur[r].y ^ cur[r].z ^ cur[r].w);
      if (false) {
#else
      {
#endif
      uint64_t p[SK_R][4];
#pragma unroll
      for (int r = 0; r < SK_R; ++r) sk_unpack8(cur[r], p[r]);
      const float* sa = sA + (kk - lane * 8) + lane * 4;
#pragma unroll
      for (int m = 0; m < M; ++m) {
        const float4 a = *reinterpret_cast<const float4*>(sa + m * ksm);
        const float4 b = *reinterpret_cast<const float4*>(sa + m * ksm + 128);
        const uint64_t pa[4] = {pack_f32x2(a.x, a.y), pack_f32x2(a.z, a.w), pack_f32x2(b.x, b.y), pack_f32x2(b.z, b.w)};
#pragma unroll
        for (int r = 0; r < SK_R; ++r)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[m][r] = ffma2(p[r][j], pa[j], acc[m][r]);
      }
      }
#pragma unroll
      for (int r = 0; r < SK_R; ++r) cur[r] = nxt[r];
    }
  }
  // warp totals -> red[rank][warp][m * SK_R + r] of the cluster's first CTA (lane m * SK_R + r stores its own entry)
  const uint32_t red_dst = splits > 1 ? mapa_smem(&red[rank][warp][0], 0) : smem_u32(&red[0][warp][0]);
#pragma unroll
  for (int m = 0; m < M; ++m)
#pragma unroll
    for (int r = 0; r < SK_R; ++r) {
      float v, t;
      unpack_f32x2(acc[m][r], v, t), v += t;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == m * SK_R + r) {
        if (splits > 1) st_shared_cluster_f32(red_dst + 4u * (m * SK_R + r), v);
        else red[0][warp][m * SK_R + r] = v;
      }
    }
  if (splits > 1) cluster_sync_all();  // every thread of every CTA of the cluster gets here (no early exits above)
  else __syncwarp();
  if (rank != 0) return;
  const int m = lane / (SK_R / 2), n = n0 + 2 * (lane % (SK_R / 2));
  if (lane >= M * (SK_R / 2) || m >= rows || n >= N) return;
  const bool have1 = n + 1 < N;
  float v0 = 0.0f, v1 = 0.0f;
  for (int s = 0; s < splits; ++s) {  // fixed order: bit-reproducible
    v0 += red[s][warp][m * SK_R + (n - n0)];
    v1 += red[s][warp][m * SK_R + (n - n0) + 1];
  }
  const ActCoef ac = act_coef(act, glu);
  if (bias) v0 += bias[n], v1 += have1 ? bias[n + 1] : 0.0f;
  if (glu) {  // interleaved rows: 2j = value, 2j + 1 = gate
    const float o = v0 * act_eval(v1, ac);
    if (out_fp32) reinterpret_cast<float*>(C)[m * ldc + (n >> 1)] = o;
    else reinterpret_cast<__nv_bfloat16*>(C)[m * ldc + (n >> 1)] = __float2bfloat16(o);
    return;
  }
  if (act != B200MIX_ACT_NONE) v0 = act_eval(v0, ac), v1 = act_eval(v1, ac);
  if (residual) {
    v0 += __bfloat162float(residual[m * ldr + n]);
    if (have1) v1 += __bfloat162float(residual[m * ldr + n + 1]);
  }
  if (out_fp32) {
    float* c = reinterpret_cast<float*>(C) + m * ldc + n;
    c[0] = v0;
    if (have1) c[1] = v1;
  } else {
    __nv_bfloat16* c = reinterpret_cast<__nv_bfloat16*>(C) + m * ldc + n;
    c[0] = __float2bfloat16(v0);
    if (have1) c[1] = __float2bfloat16(v1);
  }
}

static int g_skinny = 1;  // test hook: 0 = M <= 8 problems go through the tensor-core kernel again
static int g_skinny_splits = 0;  // test hook: force the K split (0 = automatic)

template <int M>
static int launch_skinny(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int rows, int N,
                         int K, const b200mix_epilogue* e, cudaStream_t stream) {
  constexpr int kcap = SK_SMEM_FLOATS / M / 256 * 256;  // K elements one CTA can stage
  const int ctas_n = (N + SK_ROWS_PER_CTA - 1) / SK_ROWS_PER_CTA;
  // K ranges (= cluster size): every candidate that lets a CTA stage its range in one pass is costed as
  // rounds-over-the-machine x (K elements per CTA + a fixed per-CTA cost in the same unit); ranges are at least 512 long.
  const int slots = (M <= 4 ? 2 : 1) * num_sms();
  const int s_min = std::min(SK_MAX_SPLITS, (K + kcap - 1) / kcap);
  int splits = s_min, kpart = 0;
  long long best = -1;
  for (int s = s_min; s <= SK_MAX_SPLITS && (s == s_min || K / s >= 512); ++s) {
    const int kp = ((K + s - 1) / s + 255) / 256 * 256;
    const int parts = (K + kp - 1) / kp;  // empty ranges dropped
    const long long rounds = ((long long)ctas_n * parts + slots - 1) / slots;
    const long long cost = rounds * (std::min(kp, K) + 768ll);
    if (best < 0 || cost < best) best = cost, splits = parts, kpart = kp;
  }
  if (g_skinny_splits > 0) {
    splits = std::min(g_skinny_splits, SK_MAX_SPLITS);
    kpart = ((K + splits - 1) / splits + 255) / 256 * 256;
    splits = (K + kpart - 1) / kpart;
  }
  const int ksm = std::min(kpart, kcap);
  const size_t smem = (size_t)M * ksm * sizeof(float);
  static bool configured = false;
  if (!configured) {
    B200_CUDA(cudaFuncSetAttribute(skinny_linear_kernel<M>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)(SK_SMEM_FLOATS * sizeof(float))));
    configured = true;
  }
  B200_CUDA(launch_pdl(skinny_linear_kernel<M>, dim3((unsigned)(ctas_n * splits)), dim3(256), smem, stream, splits,
                       reinterpret_cast<const __nv_bfloat16*>(A), lda, reinterpret_cast<const __nv_bfloat16*>(W), ldw, C, ldc, N,
                       K, e ? e->bias : nullptr, e ? reinterpret_cast<const __nv_bfloat16*>(e->residual) : nullptr,
                       e ? (long long)e->ldr : 0ll, e ? e->act : 0, e ? e->glu : 0, e ? e->out_fp32 : 0, rows, splits, kpart,
                       ksm));
  return 0;
}

static int g_max_clusters = 0;  // measurement hook: cap the persistent grid (0 = all SMs)
#ifndef GEMM_STREAMK_DEFAULT
#define GEMM_STREAMK_DEFAULT 1
#endif
// test / measurement hook: 0 = plain round-robin tile schedule (b200mix_debug_streamk, or B200MIX_STREAMK=0 in the environment)
static int g_streamk = [] {
  const char* e = getenv("B200MIX_STREAMK");
  return e ? atoi(e) : GEMM_STREAMK_DEFAULT;
}();
// A split tile sends its 256 KB of fp32 partials through L2 twice; a tile's own operand traffic is 32 KB per k-block, so
// only deep reductions (>= 64 k-blocks: the 3x3 convs and FF2 of the SDXL step) are split.
constexpr int SK_MIN_KBLOCKS = 64;
constexpr int SK_MAX_CLUSTERS = 74;
static int sk_min_kblocks() { return g_streamk >= 2 ? 8 : SK_MIN_KBLOCKS; }  // 2 = tests: split shallow reductions too

// Stream-K workspaces: SK_POOL slots per device (19 MB of partial accumulators + 148 flags each, sized for up to 74 clusters of 2 CTAs), allocated together on
// the first eager GEMM call (never inside a stream capture). A slot belongs to ONE stream: launches on a stream are
// ordered (a kernel's first global access follows griddepcontrol.wait = completion of its predecessor), so they can
// share it; kernels captured into a CUDA graph keep the slot of their capture stream. Streams beyond the pool, and
// launches that arrive before the pool exists, keep the round-robin schedule (same results up to fp32 summation order).
// Not covered: two graphs captured on the same stream and replayed concurrently on different streams.
constexpr int SK_POOL = 4;
struct SkPool {
  float4* ws[SK_POOL] = {};
  unsigned int* flags[SK_POOL] = {};
  cudaStream_t owner[SK_POOL] = {};
  int assigned = 0;
  bool ready = false, failed = false;
};
static SkPool g_sk[16];
static std::mutex g_sk_mutex;

static bool sk_workspace(cudaStream_t stream, float4** ws, unsigned int** flags) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 16) return false;
  std::lock_guard<std::mutex> lock(g_sk_mutex);
  SkPool& w = g_sk[dev];
  if (w.failed) return false;
  if (!w.ready) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(stream, &cs) != cudaSuccess || cs != cudaStreamCaptureStatusNone) {
      cudaGetLastError();
      return false;
    }
    const size_t bytes = (size_t)SK_MAX_CLUSTERS * 2 * SK_WS_FLOAT4_PER_CTA * sizeof(float4);
    const size_t fbytes = SK_MAX_CLUSTERS * 2 * sizeof(unsigned int);
    for (int i = 0; i < SK_POOL; ++i) {
      void *a = nullptr, *f = nullptr;
      if (cudaMalloc(&a, bytes) != cudaSuccess || cudaMalloc(&f, fbytes) != cudaSuccess ||
          cudaMemset(f, 0, fbytes) != cudaSuccess) {
        cudaGetLastError();
        w.failed = true;
        return false;
      }
      w.ws[i] = reinterpret_cast<float4*>(a), w.flags[i] = reinterpret_cast<unsigned int*>(f);
    }
    if (cudaDeviceSynchronize() != cudaSuccess) {
      cudaGetLastError();
      w.failed = true;
      return false;
    }
    w.ready = true;
  }
  int slot = -1;
  for (int i = 0; i < w.assigned; ++i)
    if (w.owner[i] == stream) slot = i;
  if (slot < 0) {
    if (w.assigned == SK_POOL) return false;
    slot = w.assigned++;
    w.owner[slot] = stream;
  }
  *ws = w.ws[slot], *flags = w.flags[slot];
  return true;
}

template <int BN, int STAGES, bool MCAST, int LNM>
static int launch_igemm_mode(const CUtensorMap& tmA, const CUtensorMap& tmB, IGemmParams p, cudaStream_t stream) {
  using Cfg = IGemmCfg<BN>;
  constexpr int smem_bytes = STAGES * Cfg::STAGE_BYTES + Cfg::EXTRA_BYTES;
  static_assert(smem_bytes <= 227 * 1024, "stage count does not fit shared memory");
  static bool configured = false;
  if (!configured) {
    B200_CUDA(cudaFuncSetAttribute(igemm_kernel<BN, STAGES, MCAST, LNM>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   smem_bytes));
    configured = true;
  }
  const int tiles_m = p.up ? 4 * p.par_tiles : p.tiles_x * p.tiles_y * p.tiles_b;
  const int total_super = ((tiles_m + 1) / 2) * p.tiles_n;
  int clusters = num_sms() / 2;
  if (g_max_clusters > 0 && clusters > g_max_clusters) clusters = g_max_clusters;
  if (clusters > total_super) clusters = total_super;
  // stream-K head over the partial round + one full round (see SegIter): needs more than one round of tiles
  p.sk_tiles = 0;
  const int rem = total_super % clusters;
  if (g_streamk && rem != 0 && total_super > clusters && clusters <= SK_MAX_CLUSTERS &&
      p.ntaps * p.kchunks >= sk_min_kblocks() && sk_workspace(stream, &p.sk_ws, &p.sk_flags))
    p.sk_tiles = clusters + rem;
  B200_CUDA(launch_pdl(igemm_kernel<BN, STAGES, MCAST, LNM>, dim3(2 * clusters), dim3(IG_THREADS), smem_bytes, stream,
                       MCAST ? 2 : 1, tmA, tmB, p));
  return 0;
}

template <int BN, int STAGES, bool MCAST>
static int launch_igemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const IGemmParams& p, cudaStream_t stream) {
  if (p.ln_stats && p.stats_out) {
    set_error("one GEMM cannot both consume and produce row statistics");
    return B200MIX_ERR_INVALID;
  }
  if (p.ln_stats || p.stats_out) {
    if constexpr (MCAST) {
      return p.ln_stats ? launch_igemm_mode<BN, STAGES, true, LNM_CONSUMER>(tmA, tmB, p, stream)
                        : launch_igemm_mode<BN, STAGES, true, LNM_PRODUCER>(tmA, tmB, p, stream);
    } else {
      set_error("the folded-LayerNorm epilogues are built for the multicast kernel only");
      return B200MIX_ERR_INVALID;
    }
  }
  return launch_igemm_mode<BN, STAGES, MCAST, LNM_NONE>(tmA, tmB, p, stream);
}

// Test / measurement hook (see b200mix_debug_gemm_pair): 1 = CTA pairs sharing the B tile through TMA multicast
// (default), 0 = independent CTAs, each loading its own B tile.
static int g_gemm_pair = 1;

static int pick_bn(long long tiles_m, long long N, int kblocks) {
  // cost = waves x time per tile; time per tile ~ BN / rate(BN). The relative rates follow the operand traffic of a
  // 128 x BN tile (A tile + half a B tile per k-block and CTA, shared through multicast): per MAC it is proportional to
  // (128 + BN/2) / (128 BN), so narrower tiles are only chosen when they avoid wave / N-padding waste. A model, not a
  // measurement: eff = (128 BN / (128 + BN/2)) normalised to BN = 256.
  const int cands[7] = {256, 224, 192, 160, 128, 64, 32};
  double eff[7];
  for (int i = 0; i < 7; ++i) eff[i] = (128.0 * cands[i] / (128.0 + cands[i] / 2.0)) / (128.0 * 256 / (128.0 + 128.0));
  double best = 1e30;
  int best_bn = 256;
  const int clusters = num_sms() / 2;
  for (int i = 0; i < 7; ++i) {
    const int bn = cands[i];
    const long long tn = (N + bn - 1) / bn;
    const long long tiles = ((tiles_m + 1) / 2) * tn;
    double waves = double((tiles + clusters - 1) / clusters);
    // stream-K head (launch_igemm): a ragged last round costs its fraction plus about a fifth of a tile for the split
    if (g_streamk && kblocks >= sk_min_kblocks() && tiles > clusters && tiles % clusters != 0)
      waves = double(tiles) / clusters + 0.2;
    const double cost = waves * (bn / eff[i]);
    if (cost < best * 0.999) best = cost, best_bn = bn;
  }
  return best_bn;
}

static int dispatch_igemm(const CUtensorMap& tmA, const void* W, long long ldw, long long Ktot, IGemmParams& p,
                          cudaStream_t stream, int force_bn) {
  const long long tiles_m = p.up ? 4ll * p.par_tiles : (long long)p.tiles_x * p.tiles_y * p.tiles_b;
  const int bn = force_bn > 0 ? force_bn : pick_bn(tiles_m, p.N, p.ntaps * p.kchunks);
  p.tiles_n = (p.N + bn - 1) / bn;
  CUtensorMap tmB;
  {
    uint64_t dims[2] = {(uint64_t)Ktot, (uint64_t)p.N};
    uint64_t strides[1] = {(uint64_t)ldw * 2};
    uint32_t box[2] = {64, (uint32_t)(bn / 2)};  // the B tile is loaded in two halves (one per CTA of a cluster)
    int rc = encode_tmap_bf16_sw128(&tmB, W, 2, dims, strides, box);
    if (rc) return rc;
  }
  // stage counts: as many as fit next to the epilogue buffers (IGemmCfg::EXTRA_BYTES) in 227 KB
  if (g_gemm_pair) {
    switch (bn) {
      case 256: return launch_igemm<256, 3, true>(tmA, tmB, p, stream);
      case 224: return launch_igemm<224, 3, true>(tmA, tmB, p, stream);
      case 192: return launch_igemm<192, 4, true>(tmA, tmB, p, stream);
      case 160: return launch_igemm<160, 4, true>(tmA, tmB, p, stream);
      case 128: return launch_igemm<128, 5, true>(tmA, tmB, p, stream);
      case 64: return launch_igemm<64, 6, true>(tmA, tmB, p, stream);
      case 32: return launch_igemm<32, 8, true>(tmA, tmB, p, stream);
      default: set_error("unsupported BN %d", bn); return B200MIX_ERR_INVALID;
    }
  }
  switch (bn) {
    case 256: return launch_igemm<256, 3, false>(tmA, tmB, p, stream);
    case 224: return launch_igemm<224, 3, false>(tmA, tmB, p, stream);
    case 192: return launch_igemm<192, 4, false>(tmA, tmB, p, stream);
    case 160: return launch_igemm<160, 4, false>(tmA, tmB, p, stream);
    case 128: return launch_igemm<128, 5, false>(tmA, tmB, p, stream);
    case 64: return launch_igemm<64, 6, false>(tmA, tmB, p, stream);
    case 32: return launch_igemm<32, 8, false>(tmA, tmB, p, stream);
    default: set_error("unsupported BN %d", bn); return B200MIX_ERR_INVALID;
  }
}

static int fill_epilogue(IGemmParams& p, const b200mix_epilogue* e, void* C, long long ldc, long long rows_default) {
  static const b200mix_epilogue kNone = {nullptr, nullptr, nullptr, 0, 0, nullptr, 0, 0, 0, 0, 1.0f, 0, nullptr, nullptr, nullptr, 0, 0.0f};
  if (!e) e = &kNone;
  p.bias = e->bias;
  p.row_add = e->row_add;
  p.row_gate = e->row_gate;
  p.ld_row = e->ld_row;
  p.rows_per_group = (int)(e->rows_per_group > 0 ? e->rows_per_group : rows_default);
  p.residual = reinterpret_cast<const __nv_bfloat16*>(e->residual);
  p.ldr = e->ldr;
  p.res_row_mod = e->residual_row_mod;
  p.C = C;
  p.ldc = ldc;
  p.act = e->act;
  p.glu = e->glu;
  p.out_fp32 = e->out_fp32;
  p.out_scale = e->out_scale == 0.0f ? 1.0f : e->out_scale;
  p.stats_out = reinterpret_cast<long long*>(e->stats_out);
  p.ln_stats = reinterpret_cast<const long long*>(e->ln_stats);
  p.ln_colsum = e->ln_colsum;
  p.ln_rms = e->ln_rms, p.ln_eps = e->ln_eps;
  p.ln_inv_k = static_cast<float>(1.0 / 16777216.0 / static_cast<double>(p.Kc));
  B200_CHECK_ARG(!(p.ln_stats || p.stats_out) || p.ntaps == 1, "row statistics (folded LayerNorm) are a Linear feature");
  B200_CHECK_ARG(!p.ln_stats || p.ln_colsum, "ln_stats needs ln_colsum");
  B200_CHECK_ARG(!p.ln_stats || reinterpret_cast<uintptr_t>(p.ln_stats) % 16 == 0, "ln_stats must be 16-byte aligned");
  B200_CHECK_ARG(!p.stats_out || reinterpret_cast<uintptr_t>(p.stats_out) % 16 == 0, "stats_out must be 16-byte aligned");
  B200_CHECK_ARG(!(p.glu && (p.N & 1)), "GLU epilogue needs an even N (got %d)", p.N);
  B200_CHECK_ARG(!(p.glu && (p.row_gate || p.residual || p.act)),
                 "GLU epilogue cannot be combined with gate / residual / activation");
  const int out_elem = p.out_fp32 ? 4 : 2;
  bool vec = (reinterpret_cast<uintptr_t>(C) % 16 == 0) && ((ldc * out_elem) % 16 == 0);
  if (p.residual) vec = vec && (reinterpret_cast<uintptr_t>(p.residual) % 16 == 0) && ((p.ldr * 2) % 16 == 0);
  if (p.bias) vec = vec && (reinterpret_cast<uintptr_t>(p.bias) % 16 == 0);
  // the coalesced epilogue reads the per-group vectors as float4 at (group * ld_row + 32-column chunk)
  if (p.row_add) vec = vec && (reinterpret_cast<uintptr_t>(p.row_add) % 16 == 0) && (p.ld_row % 4 == 0);
  if (p.row_gate) vec = vec && (reinterpret_cast<uintptr_t>(p.row_gate) % 16 == 0) && (p.ld_row % 4 == 0);
  p.vec_ok = vec ? 1 : 0;
  // the statistics are taken in the coalesced bf16 epilogue: whole 32-column chunks, 16-byte aligned rows
  B200_CHECK_ARG(!p.stats_out || (vec && !p.glu && !p.out_fp32 && p.N % 32 == 0),
                 "stats_out needs a bf16 output with N %% 32 == 0 and 16-byte aligned rows, no GLU");
  return 0;
}

}  // namespace b200

using namespace b200;

// Test hook: force a tile width (0 = heuristic). Not part of the public header.
static int g_force_bn = 0;
extern "C" void b200mix_debug_force_bn(int bn) { g_force_bn = bn; }
extern "C" void b200mix_debug_gemm_pair(int on) { b200::g_gemm_pair = on; }
extern "C" void b200mix_debug_max_clusters(int n) { b200::g_max_clusters = n; }
extern "C" void b200mix_debug_skinny(int on) { b200::g_skinny = on; }
extern "C" void b200mix_debug_streamk(int on) { b200::g_streamk = on; }
extern "C" void b200mix_debug_skinny_splits(int splits) { b200::g_skinny_splits = splits; }

extern "C" int b200mix_linear(const void* A, int64_t lda, const void* W, int64_t ldw, void* C, int64_t ldc, int64_t M,
                              int64_t N, int64_t K, const b200mix_epilogue* epi, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(A && W && C, "linear: null pointer");
  B200_CHECK_ARG(M > 0 && N > 0 && K > 0, "linear: bad shape M=%lld N=%lld K=%lld", (long long)M, (long long)N,
                 (long long)K);
  B200_CHECK_ARG(lda % 8 == 0 && ldw % 8 == 0, "linear: lda/ldw must be multiples of 8 elements (16 B TMA strides)");
  B200_CHECK_ARG(lda >= K && ldw >= K, "linear: leading dimensions smaller than K");
  B200_CHECK_ARG(M < (1ll << 31) && N < (1ll << 31), "linear: M/N too large");

  // M <= 8: weight-streaming kernel (decode steps, embedding MLPs) unless the epilogue needs per-group vectors
  if (g_skinny && M <= 8 && K % 8 == 0 && K < (1ll << 31) &&
      (!epi || (!epi->row_add && !epi->row_gate && epi->residual_row_mod == 0 && !epi->stats_out && !epi->ln_stats &&
                (epi->out_scale == 0.0f || epi->out_scale == 1.0f) && !(epi->glu && (N & 1)) &&
                !(epi->glu && (epi->residual || epi->act))))) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    switch ((int)M) {
      case 1: return launch_skinny<1>(A, lda, W, ldw, C, ldc, 1, (int)N, (int)K, epi, st);
      case 2: return launch_skinny<2>(A, lda, W, ldw, C, ldc, 2, (int)N, (int)K, epi, st);
      case 3: case 4: return launch_skinny<4>(A, lda, W, ldw, C, ldc, (int)M, (int)N, (int)K, epi, st);
      default: return launch_skinny<8>(A, lda, W, ldw, C, ldc, (int)M, (int)N, (int)K, epi, st);
    }
  }

  IGemmParams p = {};
  p.N = (int)N;
  p.Kc = (int)K;
  p.ntaps = 1;
  p.kchunks = (int)((K + 63) / 64);
  p.TW = 128, p.TH = 1, p.TB = 1;
  p.Wo = (int)M, p.Ho = 1, p.Bn = 1;
  p.tiles_x = (int)((M + 127) / 128), p.tiles_y = 1, p.tiles_b = 1;
  if (int rc = fill_epilogue(p, epi, C, ldc, M)) return rc;

  CUtensorMap tmA;
  {
    uint64_t dims[5] = {(uint64_t)K, (uint64_t)M, 1, 1, 1};
    uint64_t rowb = (uint64_t)lda * 2;
    uint64_t strides[4] = {rowb, rowb * (uint64_t)M, rowb * (uint64_t)M, rowb * (uint64_t)M};
    uint32_t box[5] = {64, 128, 1, 1, 1};
    if (int rc = encode_tmap_bf16_sw128(&tmA, A, 5, dims, strides, box)) return rc;
  }
  return dispatch_igemm(tmA, W, ldw, K, p, reinterpret_cast<cudaStream_t>(stream), g_force_bn);
}

// tile box of a conv: TW x TH x TB = 128 pixels of the [B, Ho, Wo] grid the m-tiles walk over
static int conv_tile_box(IGemmParams& p, int64_t B, int64_t Ho, int64_t Wo) {
  int TW = 1;
  while (TW * 2 <= Wo && TW < 128 && Wo % (TW * 2) == 0) TW *= 2;
  int TH = 1;
  while (TW * TH * 2 <= 128 && TH * 2 <= Ho && Ho % (TH * 2) == 0) TH *= 2;
  int TB = 128 / (TW * TH);
  B200_CHECK_ARG(TW * TH * TB == 128, "conv3x3: cannot tile %lldx%lld output into 128-pixel boxes", (long long)Ho,
                 (long long)Wo);
  p.TW = TW, p.TH = TH, p.TB = TB;
  p.Wo = (int)Wo, p.Ho = (int)Ho, p.Bn = (int)B;
  p.tiles_x = (int)((Wo + TW - 1) / TW);
  p.tiles_y = (int)((Ho + TH - 1) / TH);
  p.tiles_b = (int)((B + TB - 1) / TB);
  return 0;
}

extern "C" int b200mix_conv3x3(const void* x, const void* w, void* y, int64_t B, int64_t H, int64_t W, int64_t Cin,
                               int64_t Cout, int32_t stride, const b200mix_epilogue* epi, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(x && w && y, "conv3x3: null pointer");
  B200_CHECK_ARG(stride == 1 || stride == 2, "conv3x3: stride must be 1 or 2");
  B200_CHECK_ARG(Cin % 64 == 0, "conv3x3: Cin=%lld must be a multiple of 64 (use conv3x3_small_cin)", (long long)Cin);
  B200_CHECK_ARG(B > 0 && H > 0 && W > 0 && Cout > 0, "conv3x3: bad shape");
  B200_CHECK_ARG(stride == 1 || (H % 2 == 0 && W % 2 == 0), "conv3x3: stride 2 needs even H, W");
  const int64_t Ho = H / stride, Wo = W / stride;

  IGemmParams p = {};
  p.N = (int)Cout;
  p.Kc = (int)Cin;
  p.ntaps = 9;
  p.kchunks = (int)(Cin / 64);
  if (int rc = conv_tile_box(p, B, Ho, Wo)) return rc;
  for (int kh = 0; kh < 3; ++kh) {
    for (int kw = 0; kw < 3; ++kw) {
      const int t = kh * 3 + kw;
      if (stride == 1) {
        p.tap_dc[t] = 0, p.tap_dx[t] = kw - 1, p.tap_p[t] = 0, p.tap_dy[t] = kh - 1;
      } else {
        // input (h, w) = (2*oh + kh - 1, 2*ow + kw - 1) on the parity view [B, H/2, 2, W/2, 2*C]
        const int wp = (kw == 1) ? 0 : 1, dx = (kw == 0) ? -1 : 0;
        const int hp = (kh == 1) ? 0 : 1, dy = (kh == 0) ? -1 : 0;
        p.tap_dc[t] = wp * (int)Cin, p.tap_dx[t] = dx, p.tap_p[t] = hp, p.tap_dy[t] = dy;
      }
    }
  }
  if (int rc = fill_epilogue(p, epi, y, Cout, Ho * Wo)) return rc;
  if (p.glu) {
    set_error("conv3x3: GLU epilogue not supported");
    return B200MIX_ERR_INVALID;
  }

  CUtensorMap tmA;
  {
    uint64_t dims[5], strides[4];
    if (stride == 1) {
      dims[0] = Cin, dims[1] = W, dims[2] = 1, dims[3] = H, dims[4] = B;
      strides[0] = Cin * 2, strides[1] = W * Cin * 2, strides[2] = W * Cin * 2, strides[3] = H * W * Cin * 2;
    } else {
      dims[0] = 2 * Cin, dims[1] = W / 2, dims[2] = 2, dims[3] = H / 2, dims[4] = B;
      strides[0] = 2 * Cin * 2, strides[1] = W * Cin * 2, strides[2] = 2 * W * Cin * 2, strides[3] = H * W * Cin * 2;
    }
    uint32_t box[5] = {64, (uint32_t)p.TW, 1, (uint32_t)p.TH, (uint32_t)p.TB};
    if (int rc = encode_tmap_bf16_sw128(&tmA, x, 5, dims, strides, box)) return rc;
  }
  return dispatch_igemm(tmA, w, 9 * Cin, 9 * Cin, p, reinterpret_cast<cudaStream_t>(stream), g_force_bn);
}


// nearest-2x upsample + conv3x3 in one pass over the LOW-resolution input (Upsample2D, resnet.py:137-216: F.interpolate
// (scale 2, nearest) followed by the 3x3 conv). Output pixel (2i + py, 2j + px) only sees the 2 x 2 input neighbourhood
// (i - 1 + py .. i + py, j - 1 + px .. j + px): taps of the 3x3 filter that hit the same input pixel are pre-summed per
// output parity, so the conv is 4 taps instead of 9 (4/9 of the FLOPs), the 4x larger upsampled tensor is never written
// or read, and the halo is TMA zero fill exactly as for the plain conv (U[-1] = 0 <-> X[-1], U[2H] = 0 <-> X[H]).
// w4: bf16 [Cout, 4 parities (py, px), 4 taps (a, b), Cin] with tap (a, b) of parity (py, px) = sum of w[ky][kx] over
// ky in {0 | 1,2} (py = 0: a = 0 | 1) resp. {0,1 | 2} (py = 1), same for kx (ops.fold_upsample_conv_weight).
extern "C" int b200mix_conv3x3_up2x(const void* x, const void* w4, void* y, int64_t B, int64_t H, int64_t W, int64_t Cin,
                                    int64_t Cout, const b200mix_epilogue* epi, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(x && w4 && y, "conv3x3_up2x: null pointer");
  B200_CHECK_ARG(Cin % 64 == 0, "conv3x3_up2x: Cin=%lld must be a multiple of 64", (long long)Cin);
  B200_CHECK_ARG(B > 0 && H > 0 && W > 0 && Cout > 0, "conv3x3_up2x: bad shape");
  IGemmParams p = {};
  p.N = (int)Cout;
  p.Kc = (int)Cin;
  p.ntaps = 4;
  p.kchunks = (int)(Cin / 64);
  if (int rc = conv_tile_box(p, B, H, W)) return rc;
  p.up = 1;
  p.par_tiles = (p.tiles_x * p.tiles_y * p.tiles_b + 1) / 2 * 2;
  for (int par = 0; par < 4; ++par)
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b) {
        const int t = par * 4 + a * 2 + b;
        p.tap_dc[t] = 0, p.tap_p[t] = 0, p.tap_dy[t] = a - 1 + (par >> 1), p.tap_dx[t] = b - 1 + (par & 1);
      }
  if (int rc = fill_epilogue(p, epi, y, Cout, 4 * H * W)) return rc;
  if (p.glu) {
    set_error("conv3x3_up2x: GLU epilogue not supported");
    return B200MIX_ERR_INVALID;
  }
  CUtensorMap tmA;
  {
    uint64_t dims[5] = {(uint64_t)Cin, (uint64_t)W, 1, (uint64_t)H, (uint64_t)B};
    uint64_t strides[4] = {(uint64_t)Cin * 2, (uint64_t)(W * Cin * 2), (uint64_t)(W * Cin * 2), (uint64_t)(H * W * Cin * 2)};
    uint32_t box[5] = {64, (uint32_t)p.TW, 1, (uint32_t)p.TH, (uint32_t)p.TB};
    if (int rc = encode_tmap_bf16_sw128(&tmA, x, 5, dims, strides, box)) return rc;
  }
  return dispatch_igemm(tmA, w4, 16 * Cin, 16 * Cin, p, reinterpret_cast<cudaStream_t>(stream), g_force_bn);
}


// Batched-strided Linear: for b in [0, nbatch): C_b[rows, N] = epilogue(A_b[rows, K] @ W[N, K]^T) with
// A_b = A + b*a_bstride, C_b = C + b*c_bstride, residual_b = residual + b*r_bstride (strides in elements). The
// epilogue's per-group vectors (row_add / row_gate) are indexed by b. Used to read / write the image and text token
// ranges of SD3's joint [B, n_img + n_txt, *] buffers in place (attention_processor.py:934-975 concatenates and
// splits them; here the concat is never materialised).
extern "C" int b200mix_linear_batched(const void* A, int64_t lda, int64_t a_bstride, const void* W, int64_t ldw, void* C,
                                      int64_t ldc, int64_t c_bstride, int64_t rows, int64_t nbatch, int64_t N, int64_t K,
                                      const b200mix_epilogue* epi, int64_t r_bstride, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(A && W && C, "linear_batched: null pointer");
  B200_CHECK_ARG(rows > 0 && nbatch > 0 && N > 0 && K > 0, "linear_batched: bad shape");
  B200_CHECK_ARG(lda % 8 == 0 && ldw % 8 == 0 && a_bstride % 8 == 0 && c_bstride > 0,
                 "linear_batched: strides must be multiples of 8 elements and c_bstride > 0");
  IGemmParams p = {};
  p.N = (int)N;
  p.Kc = (int)K;
  p.ntaps = 1;
  p.kchunks = (int)((K + 63) / 64);
  p.TW = 128, p.TH = 1, p.TB = 1;
  p.Wo = (int)rows, p.Ho = 1, p.Bn = (int)nbatch;
  p.tiles_x = (int)((rows + 127) / 128), p.tiles_y = 1, p.tiles_b = (int)nbatch;
  if (int rc = fill_epilogue(p, epi, C, ldc, rows)) return rc;
  p.c_bstride = c_bstride;
  p.r_bstride = r_bstride;
  const int out_elem = p.out_fp32 ? 4 : 2;
  if ((c_bstride * out_elem) % 16 != 0 || (p.residual && (r_bstride * 2) % 16 != 0)) p.vec_ok = 0;
  CUtensorMap tmA;
  {
    uint64_t dims[5] = {(uint64_t)K, (uint64_t)rows, 1, 1, (uint64_t)nbatch};
    uint64_t rowb = (uint64_t)lda * 2;
    uint64_t bb = (uint64_t)(nbatch > 1 ? a_bstride : (int64_t)(lda * rows)) * 2;
    uint64_t strides[4] = {rowb, bb, bb, bb};
    uint32_t box[5] = {64, 128, 1, 1, 1};
    if (int rc = encode_tmap_bf16_sw128(&tmA, A, 5, dims, strides, box)) return rc;
  }
  return dispatch_igemm(tmA, W, ldw, K, p, reinterpret_cast<cudaStream_t>(stream), g_force_bn);
}
