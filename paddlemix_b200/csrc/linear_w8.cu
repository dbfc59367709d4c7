// Weight-only int8 Linear: out[m, n] = epilogue(scale[n] * sum_k A[m, k] * q[n, k]), A bf16, q int8 with one fp32
// scale per output row. The weight-only int8 mode of PaddleNLP's inference models (qwen/modeling.py:194-235,
// llama/modeling.py:523-578: paddle.nn.quant.weight_quantize + weight_only_linear; PaddleMIX's
// triton_ops.py:363-563 weight_only_int8 spells out the rule, :481,505-508,545-546).
//
// Device layout of q (written by b200mix_quantize_w8 only, read by both paths below): [N / 16][K / 32][32 lanes][16 B].
// One 512-byte piece = a 16-row x 32-k block in the order of the A operand of two mma.m16n8k16 (k16 steps s = 0, 1):
// lane l = 4 g + t holds, in byte s * 8 + 2 r + e, element (row g + 8 (r & 1), k 16 s + 2 t + 8 (r >> 1) + e).
// A warp's 16-byte-per-lane load of one piece is one coalesced 512-byte read and is already its A fragments.
//
// Small M (decode, batched decode): w8_linear_kernel streams q once from HBM through mma.sync (bf16 x bf16 -> fp32).
//   * one warp = one 16-row tile, 8 warps per CTA; the CTA's activation rows (token blocks of 8, zero padded) are staged
//     in shared memory as bf16 and read as B fragments with ldmatrix.x4 (rows padded by 16 B: conflict-free);
//   * weights -> bf16 in registers: exact, |q| <= 127 needs 8 significant bits and bf16 has 8;
//   * K runs in chunks of 256: each chunk is an mma chain from zero (fp32) and is added to an fp64 accumulator. Chunk
//     boundaries do not depend on how K is split, and an fp64 sum of fp32 partials is exact unless they span more
//     than ~2^22, so the result is the same for every split (short of an fp64 rounding landing on an fp32 tie);
//   * K is split over a thread-block cluster with the cost model of the bf16 skinny kernel (skinny_split); rank 0
//     adds the other ranks' fp64 accumulators in rank order through distributed shared memory (no workspace, no atomics).
// Large M (prefill): bf16(q * scale) is expanded into the caller's workspace as a row-major [N, K] bf16 weight and
// b200mix_linear (the wgmma implicit GEMM) runs on it; there the problem is compute-bound and the expansion costs
// 3 bytes per weight once per call.
#include <cuda_bf16.h>

#include <algorithm>

#include "act.cuh"
#include "common.cuh"
#include "ptx.cuh"

namespace b200 {
namespace {

constexpr int W8_WARPS = 8;
constexpr int W8_CHUNK = 256;                 // K elements per fp32 partial
constexpr int W8_SMEM_BYTES = 96 * 1024;      // staged activations per CTA
constexpr int W8_PAD = 8;                     // bf16 elements of padding per staged row
constexpr int W8_MAX_TOKENS = 64;             // rows per launch of the small-M kernel (8 token blocks)
constexpr int W8_PREFETCH = 16;               // 512-byte pieces the L2 prefetch runs ahead of the register ring
// The largest M that takes the small-M kernel; above it the weight is expanded and the wgmma GEMM runs
// (tools/bench_w8.py times both paths at M = 1 .. 64 on the Qwen2-VL-7B projections: the small-M kernel is the faster
// one at every such M, and 64 is the most rows one launch of it takes).
constexpr int W8_SMALL_MAX = 64;
static int g_small_max = W8_SMALL_MAX;  // test hook: b200mix_debug_w8_small_max

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}

__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                               uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
               "{%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint4 ldg_stream16(const uint8_t* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}

__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

__device__ __forceinline__ double ld_shared_cluster_f64(uint32_t addr) {
  double v;
  asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(addr) : "memory");
  return v;
}

// four int8 (bytes 0..3 of w) -> two bf16x2 (bytes 0, 1 -> lo; 2, 3 -> hi). Byte b + 128 is placed in the mantissa of
// 2^23 and 2^23 + 128 subtracted: exact integers, and exact again in bf16.
__device__ __forceinline__ void i8x4_to_bf16(uint32_t w, uint32_t& lo, uint32_t& hi) {
  const uint32_t u = w ^ 0x80808080u;
  const float f0 = __int_as_float(__byte_perm(u, 0x4B000000u, 0x7650)) - 8388736.0f;
  const float f1 = __int_as_float(__byte_perm(u, 0x4B000000u, 0x7651)) - 8388736.0f;
  const float f2 = __int_as_float(__byte_perm(u, 0x4B000000u, 0x7652)) - 8388736.0f;
  const float f3 = __int_as_float(__byte_perm(u, 0x4B000000u, 0x7653)) - 8388736.0f;
  lo = pack_bf16x2(f0, f1), hi = pack_bf16x2(f2, f3);
}

// byte offset of block (tile, blk) of lane `lane` in the device layout
__device__ __forceinline__ long long w8_offset(int tile, int blk, int kblocks, int lane) {
  return ((static_cast<long long>(tile) * kblocks + blk) * 32 + lane) * 16;
}

// grid: CTA = (16-row tiles [8 c, 8 c + 8)) x cluster rank (K range). MB = token blocks of 8.
template <int MB>
__global__ void __launch_bounds__(W8_WARPS * 32, MB <= 4 ? 2 : 1)
    w8_linear_kernel(const __nv_bfloat16* __restrict__ A, long long lda, const uint8_t* __restrict__ q,
                     const float* __restrict__ scale, void* __restrict__ C, long long ldc, int N, int K,
                     const float* __restrict__ bias, const __nv_bfloat16* __restrict__ residual, long long ldr, int act,
                     int glu, int out_fp32, int rows, int splits, int kpart, int ksm) {
  constexpr int T = 8 * MB;  // staged token rows
  extern __shared__ __align__(16) uint8_t w8_smem[];
  __nv_bfloat16* sA = reinterpret_cast<__nv_bfloat16*>(w8_smem);  // [T][ksm + W8_PAD]
  const int sstride = ksm + W8_PAD;
  pdl_wait();
  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rank = splits > 1 ? (int)cluster_ctarank() : 0;
  const int tile = (int)(blockIdx.x / splits) * W8_WARPS + warp;
  const bool tile_ok = tile < N / 16;
  const int kblocks = K / 32;
  const uint8_t* qt = q + w8_offset(tile_ok ? tile : 0, 0, kblocks, lane);
  // ldmatrix.x4 source of this lane: token row (lane & 7) of a token block, k offset 8 (lane >> 3) of a 32-k block
  const uint32_t b_base = smem_u32(sA) + 2u * ((lane & 7) * sstride + (lane >> 3) * 8);

  double acc[MB][4];
#pragma unroll
  for (int j = 0; j < MB; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[j][e] = 0.0;

  const int kend = min(K, (rank + 1) * kpart);
  for (int k0 = rank * kpart; k0 < kend; k0 += ksm) {
    const int kc = min(ksm, kend - k0);
    const int nblk = kc / 32, blk0 = k0 / 32;
    // the weight stream does not depend on the staged activations: its first 8 pieces go out first
    uint4 wq[8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if (tile_ok && i < nblk) wq[i] = ldg_stream16(qt + (long long)(blk0 + i) * 512);
    for (int i = 8; i < 8 + W8_PREFETCH; ++i)
      if (tile_ok && i < nblk) prefetch_l2(qt + (long long)(blk0 + i) * 512);
    __syncthreads();  // the previous pass's reads of sA are done
    for (int i = threadIdx.x; i < T * (kc / 8); i += W8_WARPS * 32) {
      const int m = i / (kc / 8), k = (i - m * (kc / 8)) * 8;
      const uint4 v = m < rows ? __ldg(reinterpret_cast<const uint4*>(A + m * lda + k0 + k)) : make_uint4(0u, 0u, 0u, 0u);
      *reinterpret_cast<uint4*>(sA + m * sstride + k) = v;
    }
    __syncthreads();
    if (tile_ok) {
      for (int c0 = 0; c0 < nblk; c0 += W8_CHUNK / 32) {
        float part[MB][4];
#pragma unroll
        for (int j = 0; j < MB; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) part[j][e] = 0.0f;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int b = c0 + i;
          if (b < nblk) {
            uint32_t a[8];
            i8x4_to_bf16(wq[i].x, a[0], a[1]);
            i8x4_to_bf16(wq[i].y, a[2], a[3]);
            i8x4_to_bf16(wq[i].z, a[4], a[5]);
            i8x4_to_bf16(wq[i].w, a[6], a[7]);
            if (b + 8 < nblk) wq[i] = ldg_stream16(qt + (long long)(blk0 + b + 8) * 512);
            if (b + 8 + W8_PREFETCH < nblk) prefetch_l2(qt + (long long)(blk0 + b + 8 + W8_PREFETCH) * 512);
#pragma unroll
            for (int j = 0; j < MB; ++j) {
              uint32_t bf[4];
              ldmatrix_x4(bf, b_base + 2u * (j * 8 * sstride + b * 32));
              mma_bf16_16816(part[j], a[0], a[1], a[2], a[3], bf[0], bf[1]);
              mma_bf16_16816(part[j], a[4], a[5], a[6], a[7], bf[2], bf[3]);
            }
          }
        }
#pragma unroll
        for (int j = 0; j < MB; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[j][e] += (double)part[j][e];
      }
    }
  }

  // K ranks: every rank parks its accumulators in its own shared memory; rank 0 adds them in rank order
  if (splits > 1) {
    double* red = reinterpret_cast<double*>(w8_smem) + warp * (MB * 4 * 32) + lane;  // [warp][j * 4 + e][lane]
    __syncthreads();  // every warp is done with sA
    if (rank != 0) {
#pragma unroll
      for (int j = 0; j < MB; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) red[(j * 4 + e) * 32] = acc[j][e];
    }
    cluster_sync_all();
    if (rank == 0) {
      for (int s = 1; s < splits; ++s) {
        const uint32_t peer = mapa_smem(red, (uint32_t)s);
#pragma unroll
        for (int j = 0; j < MB; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[j][e] += ld_shared_cluster_f64(peer + 8u * 32u * (j * 4 + e));
      }
    }
    cluster_sync_all();  // the peers' shared memory stays alive until rank 0 has read it
    if (rank != 0) return;
  }
  if (!tile_ok) return;

  // epilogue: acc[j][e] is (row g + 8 (e >> 1), token 8 j + 2 t + (e & 1)) with g = lane / 4, t = lane % 4
  const int g = lane >> 2, t = lane & 3;
  const ActCoef ac = act_coef(act, glu);
  float sc[2], bi[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int n = tile * 16 + g + 8 * h;
    sc[h] = scale[n];
    bi[h] = bias ? bias[n] : 0.0f;
  }
#pragma unroll
  for (int j = 0; j < MB; ++j) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int h = e >> 1, m = 8 * j + 2 * t + (e & 1);
      const int n = tile * 16 + g + 8 * h;
      float v = __fmaf_rn((float)acc[j][e], sc[h], bi[h]);
      if (glu) {
        // interleaved rows: value row n (g even) and gate row n + 1 sit in lanes l and l + 4
        const float gate = __shfl_down_sync(0xffffffffu, v, 4);
        if ((g & 1) || m >= rows) continue;
        const float o = v * act_eval(gate, ac);
        if (out_fp32) reinterpret_cast<float*>(C)[m * ldc + (n >> 1)] = o;
        else reinterpret_cast<__nv_bfloat16*>(C)[m * ldc + (n >> 1)] = __float2bfloat16(o);
        continue;
      }
      if (m >= rows) continue;
      if (act != B200MIX_ACT_NONE) v = act_eval(v, ac);
      if (residual) v += __bfloat162float(residual[m * ldr + n]);
      if (out_fp32) reinterpret_cast<float*>(C)[m * ldc + n] = v;
      else reinterpret_cast<__nv_bfloat16*>(C)[m * ldc + n] = __float2bfloat16(v);
    }
  }
}

// One CTA per 16-row tile: the 16 row scales, then every (k block, lane) piece of the device layout.
template <typename Tin>
__global__ void __launch_bounds__(256) w8_quantize_kernel(const Tin* __restrict__ W, uint8_t* __restrict__ q,
                                                          float* __restrict__ scale, int K) {
  __shared__ float s_scale[16];
  pdl_wait();
  pdl_launch_dependents();
  const int tile = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const Tin* Wt = W + static_cast<long long>(tile) * 16 * K;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = 2 * warp + h;
    float m = 0.0f;
    for (int k = lane; k < K; k += 32) m = fmaxf(m, fabsf(static_cast<float>(Wt[static_cast<long long>(r) * K + k])));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) {
      const float s = __fdiv_rn(m, 127.0f);
      s_scale[r] = s;
      scale[tile * 16 + r] = s;
    }
  }
  __syncthreads();
  const int kblocks = K / 32;
  for (int i = threadIdx.x; i < kblocks * 32; i += 256) {
    const int blk = i >> 5, l = i & 31, g = l >> 2, t = l & 3;
    uint32_t word[4];
#pragma unroll
    for (int wi = 0; wi < 4; ++wi) {  // word wi = step s = wi / 2, registers r = 2 (wi % 2) and 2 (wi % 2) + 1
      uint32_t bytes = 0;
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const int s = wi >> 1, r = 2 * (wi & 1) + (b >> 1), e = b & 1;
        const int row = g + 8 * (r & 1), k = blk * 32 + 16 * s + 2 * t + 8 * (r >> 1) + e;
        const float x = static_cast<float>(Wt[static_cast<long long>(row) * K + k]);
        const float sc = s_scale[row];
        // q = clip(round(w / scale), -127, 127): IEEE division, rounding half away from zero (roundf, paddle.round);
        // an all-zero row has scale 0 and q 0 (not 0 / 0)
        const float v = sc == 0.0f ? 0.0f : fminf(fmaxf(roundf(__fdiv_rn(x, sc)), -127.0f), 127.0f);
        bytes |= (static_cast<uint32_t>(static_cast<int>(v)) & 0xFFu) << (8 * b);
      }
      word[wi] = bytes;
    }
    *reinterpret_cast<uint4*>(q + w8_offset(tile, blk, kblocks, l)) = make_uint4(word[0], word[1], word[2], word[3]);
  }
}

// device layout -> row-major bf16(q * scale) [N, K]; one thread per 16-byte piece
__global__ void __launch_bounds__(256) w8_expand_kernel(const uint8_t* __restrict__ q, const float* __restrict__ scale,
                                                        __nv_bfloat16* __restrict__ out, int N, int K) {
  pdl_wait();
  pdl_launch_dependents();
  const int kblocks = K / 32;
  const long long pieces = static_cast<long long>(N / 16) * kblocks * 32;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < pieces; i += static_cast<long long>(gridDim.x) * 256) {
    const int l = (int)(i & 31), g = l >> 2, t = l & 3;
    const long long tb = i >> 5;
    const int blk = (int)(tb % kblocks), tile = (int)(tb / kblocks);
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(q) + i);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    const float sc[2] = {scale[tile * 16 + g], scale[tile * 16 + g + 8]};
#pragma unroll
    for (int wi = 0; wi < 4; ++wi) {
#pragma unroll
      for (int p = 0; p < 2; ++p) {  // register r = 2 (wi % 2) + p: bytes 2 p, 2 p + 1 of the word
        const int s = wi >> 1, r = 2 * (wi & 1) + p;
        const int row = tile * 16 + g + 8 * (r & 1), k = blk * 32 + 16 * s + 2 * t + 8 * (r >> 1);
        const float x0 = (float)(int8_t)(w[wi] >> (16 * p)), x1 = (float)(int8_t)(w[wi] >> (16 * p + 8));
        *reinterpret_cast<uint32_t*>(out + static_cast<long long>(row) * K + k) = pack_bf16x2(x0 * sc[r & 1], x1 * sc[r & 1]);
      }
    }
  }
}

template <int MB>
int launch_w8_small(const __nv_bfloat16* A, long long lda, const uint8_t* q, const float* scale, void* C, long long ldc,
                    int rows, int N, int K, const b200mix_epilogue* e, cudaStream_t stream) {
  constexpr int T = 8 * MB;
  // K elements one CTA stages in a pass (multiple of 256), leaving room for the fp64 reduction buffer
  constexpr int kcap = (W8_SMEM_BYTES / (2 * T) - W8_PAD) / 256 * 256;
  const int ctas_n = (N / 16 + W8_WARPS - 1) / W8_WARPS;
  int splits, kpart;
  skinny_split(ctas_n, K, kcap, (MB <= 4 ? 2 : 1) * num_sms(), &splits, &kpart);
  const int ksm = std::min(kpart, kcap);
  const size_t smem = std::max<size_t>((size_t)T * (ksm + W8_PAD) * 2, splits > 1 ? (size_t)W8_WARPS * MB * 4 * 32 * 8 : 0);
  static bool configured = false;
  if (!configured) {
    B200_CUDA(cudaFuncSetAttribute(w8_linear_kernel<MB>, cudaFuncAttributeMaxDynamicSharedMemorySize, W8_SMEM_BYTES));
    configured = true;
  }
  B200_CUDA(launch_pdl(w8_linear_kernel<MB>, dim3((unsigned)(ctas_n * splits)), dim3(W8_WARPS * 32), smem, stream, splits,
                       A, lda, q, scale, C, ldc, N, K, e ? e->bias : nullptr,
                       e ? reinterpret_cast<const __nv_bfloat16*>(e->residual) : nullptr, e ? (long long)e->ldr : 0ll,
                       e ? e->act : 0, e ? e->glu : 0, e ? e->out_fp32 : 0, rows, splits, kpart, ksm));
  return 0;
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" void b200mix_debug_w8_small_max(int m) { g_small_max = m < 0 ? W8_SMALL_MAX : m; }

extern "C" int b200mix_quantize_w8(const void* W, int32_t w_is_fp32, void* q, float* scale, int64_t N, int64_t K,
                                   void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(W && q && scale, "quantize_w8: null pointer");
  B200_CHECK_ARG(N > 0 && K > 0 && N % 16 == 0 && K % 64 == 0,
                 "quantize_w8: N=%lld must be a multiple of 16 and K=%lld a multiple of 64", (long long)N, (long long)K);
  B200_CHECK_ARG(N * K < (1ll << 40) && K < (1ll << 31), "quantize_w8: weight too large");
  B200_CHECK_ARG(reinterpret_cast<uintptr_t>(q) % 16 == 0, "quantize_w8: q must be 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (w_is_fp32)
    B200_CUDA(launch_pdl(w8_quantize_kernel<float>, dim3((unsigned)(N / 16)), dim3(256), 0, st, 1,
                         reinterpret_cast<const float*>(W), reinterpret_cast<uint8_t*>(q), scale, (int)K));
  else
    B200_CUDA(launch_pdl(w8_quantize_kernel<__nv_bfloat16>, dim3((unsigned)(N / 16)), dim3(256), 0, st, 1,
                         reinterpret_cast<const __nv_bfloat16*>(W), reinterpret_cast<uint8_t*>(q), scale, (int)K));
  return 0;
}

extern "C" int b200mix_linear_w8_workspace_size(int64_t M, int64_t N, int64_t K, int64_t* bytes) {
  B200_CHECK_ARG(bytes, "linear_w8_workspace_size: null pointer");
  B200_CHECK_ARG(M > 0 && N > 0 && K > 0, "linear_w8_workspace_size: bad shape");
  *bytes = M > g_small_max ? N * K * 2 : 0;
  return 0;
}

extern "C" int b200mix_linear_w8(const void* A, int64_t lda, const void* q, const float* scale, void* C, int64_t ldc,
                                 int64_t M, int64_t N, int64_t K, const b200mix_epilogue* epi, void* workspace,
                                 int64_t workspace_bytes, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(A && q && scale && C, "linear_w8: null pointer");
  B200_CHECK_ARG(M > 0 && N > 0 && K > 0, "linear_w8: bad shape M=%lld N=%lld K=%lld", (long long)M, (long long)N,
                 (long long)K);
  B200_CHECK_ARG(N % 16 == 0 && K % 64 == 0, "linear_w8: N=%lld must be a multiple of 16 and K=%lld a multiple of 64",
                 (long long)N, (long long)K);
  B200_CHECK_ARG(M < (1ll << 31) && N < (1ll << 31) && K < (1ll << 31), "linear_w8: M/N/K too large");
  B200_CHECK_ARG(lda % 8 == 0 && lda >= K && reinterpret_cast<uintptr_t>(A) % 16 == 0,
                 "linear_w8: A must be 16-byte aligned with lda a multiple of 8 and >= K");
  B200_CHECK_ARG(reinterpret_cast<uintptr_t>(q) % 16 == 0, "linear_w8: q must be 16-byte aligned");
  if (epi && (epi->row_add || epi->row_gate || epi->residual_row_mod || epi->stats_out || epi->ln_stats ||
              epi->ln_colsum || epi->ln_rms || (epi->out_scale != 0.0f && epi->out_scale != 1.0f))) {
    set_error("linear_w8: only bias / act / glu / residual / out_fp32 epilogues are supported");
    return B200MIX_ERR_UNSUPPORTED;
  }
  B200_CHECK_ARG(!epi || (epi->act >= B200MIX_ACT_NONE && epi->act <= B200MIX_ACT_QUICK_GELU &&
                          epi->glu >= B200MIX_GLU_NONE && epi->glu <= B200MIX_GLU_SWIGLU),
                 "linear_w8: unknown act / glu");
  B200_CHECK_ARG(!(epi && epi->glu && (epi->residual || epi->act)),
                 "linear_w8: GLU epilogue cannot be combined with residual / activation");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (M > g_small_max) {
    const int64_t need = N * K * 2;
    B200_CHECK_ARG(workspace && workspace_bytes >= need && reinterpret_cast<uintptr_t>(workspace) % 16 == 0,
                   "linear_w8: M=%lld needs a 16-byte aligned workspace of %lld bytes (got %lld)", (long long)M,
                   (long long)need, (long long)workspace_bytes);
    const long long pieces = N / 16 * (K / 32) * 32;
    const unsigned blocks = (unsigned)std::min<long long>((pieces + 255) / 256, 16ll * num_sms());
    B200_CUDA(launch_pdl(w8_expand_kernel, dim3(blocks), dim3(256), 0, st, 1, reinterpret_cast<const uint8_t*>(q), scale,
                         reinterpret_cast<__nv_bfloat16*>(workspace), (int)N, (int)K));
    return b200mix_linear(A, lda, workspace, K, C, ldc, M, N, K, epi, stream);
  }
  const __nv_bfloat16* a = reinterpret_cast<const __nv_bfloat16*>(A);
  const uint8_t* qq = reinterpret_cast<const uint8_t*>(q);
  const int out_elem = epi && epi->out_fp32 ? 4 : 2;
  for (int64_t m0 = 0; m0 < M; m0 += W8_MAX_TOKENS) {  // the small path takes any M (tests force it past the crossover)
    const int rows = (int)std::min<int64_t>(W8_MAX_TOKENS, M - m0);
    b200mix_epilogue e = {};
    if (epi) {
      e = *epi;
      if (e.residual) e.residual = reinterpret_cast<const __nv_bfloat16*>(e.residual) + m0 * e.ldr;
    }
    void* c = reinterpret_cast<uint8_t*>(C) + m0 * ldc * out_elem;
    const __nv_bfloat16* am = a + m0 * lda;
    int rc;
    if (rows <= 8) rc = launch_w8_small<1>(am, lda, qq, scale, c, ldc, rows, (int)N, (int)K, &e, st);
    else if (rows <= 16) rc = launch_w8_small<2>(am, lda, qq, scale, c, ldc, rows, (int)N, (int)K, &e, st);
    else if (rows <= 32) rc = launch_w8_small<4>(am, lda, qq, scale, c, ldc, rows, (int)N, (int)K, &e, st);
    else rc = launch_w8_small<8>(am, lda, qq, scale, c, ldc, rows, (int)N, (int)K, &e, st);
    if (rc) return rc;
  }
  return 0;
}
