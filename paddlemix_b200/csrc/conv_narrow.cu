// conv3x3 (padding 1, stride 1 | 2) for narrow channel counts: the ControlNet conditioning embedding
// (ControlNetConditioningEmbedding, controlnet.py:71-113: 3 -> 16 -> 16 -> 32 -> 32 -> 96 -> 96 -> 256 at image
// resolution). The wgmma implicit GEMM needs Cin % 64 == 0 (one k-chunk = one 128-byte swizzled TMA row), so these
// layers get their own tensor-core implicit GEMM on mma.sync.m16n8k16 (bf16 in, fp32 accumulate):
//   K = 9 taps x Cp, Cp = Cin rounded up to 16 (the padded channels are zero in both operands);
//   one CTA = 8 warps = an 8 x 16 output-pixel tile (one output row of 16 pixels per warp, i.e. one m16 tile) times
//   CN_BN = 32 output channels (4 n8 tiles), so a CTA holds only a 32-wide slice of the filter bank in shared memory
//   (96 -> 256 is 442 KB of bf16 weights, which no single CTA can hold);
//   the input halo tile ((8-1)*s+3) x ((16-1)*s+3) x Cp is staged once in shared memory with cp.async 16-byte copies
//   when Cin % 8 == 0 and scalar loads otherwise (the Cin = 3 first layer);
//   the Cout slices of one pixel tile are adjacent in the launch order, so the halo re-reads hit L2.
// Epilogue: + bias, optional SiLU, bf16 NHWC store.
#include <cuda_bf16.h>

#include "common.cuh"
#include "ptx.cuh"

namespace b200 {
namespace {

constexpr int CN_WARPS = 8;      // output rows per CTA
constexpr int CN_TW = 16;        // output columns per CTA (= the m16 tile of a warp)
constexpr int CN_BN = 32;        // output channels per CTA
constexpr int CN_PAD = 8;        // bf16 elements of padding per smem row (16 B): spreads ldmatrix rows over banks

struct NarrowGeom {
  int Cp;      // Cin rounded up to 16
  int HR, HC;  // halo rows / columns
  int xs;      // smem elements per halo pixel (Cp + CN_PAD)
  int ws;      // smem elements per weight row (9*Cp + CN_PAD)
};

__host__ __device__ inline NarrowGeom narrow_geom(int Cin, int stride) {
  NarrowGeom g;
  g.Cp = (Cin + 15) & ~15;
  g.HR = (CN_WARPS - 1) * stride + 3;
  g.HC = (CN_TW - 1) * stride + 3;
  g.xs = g.Cp + CN_PAD;
  g.ws = 9 * g.Cp + CN_PAD;
  return g;
}

inline size_t narrow_smem_bytes(const NarrowGeom& g) {
  return ((size_t)g.HR * g.HC * g.xs + (size_t)CN_BN * g.ws) * sizeof(__nv_bfloat16);
}

__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p)));
}

__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
               "{%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// grid: one CTA per (b, tile row, tile column, Cout slice), Cout slice fastest
__global__ void __launch_bounds__(CN_WARPS * 32) conv3x3_narrow_kernel(
    const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w, const float* __restrict__ bias,
    __nv_bfloat16* __restrict__ y, int H, int W, int Cin, int Cout, int stride, int act, int tiles_x, int tiles_y,
    int n_slices, int vec) {
  extern __shared__ __align__(16) unsigned char cn_smem[];
  const NarrowGeom g = narrow_geom(Cin, stride);
  __nv_bfloat16* sx = reinterpret_cast<__nv_bfloat16*>(cn_smem);  // [HR][HC][xs]
  __nv_bfloat16* sw = sx + (size_t)g.HR * g.HC * g.xs;             // [CN_BN][ws], k = tap * Cp + c

  long long bid = blockIdx.x;
  const int ns = (int)(bid % n_slices);
  bid /= n_slices;
  const int tx = (int)(bid % tiles_x);
  bid /= tiles_x;
  const int ty = (int)(bid % tiles_y);
  const long long b = bid / tiles_y;
  const int Ho = H / stride, Wo = W / stride;
  const int oy0 = ty * CN_WARPS, ox0 = tx * CN_TW, n0 = ns * CN_BN;
  const int iy0 = oy0 * stride - 1, ix0 = ox0 * stride - 1;
  const __nv_bfloat16 zero = __float2bfloat16(0.0f);

  pdl_wait();
  pdl_launch_dependents();

  // ---- stage the input halo and the weight slice (zero fill: borders, padded channels, channels >= Cout) -------
  const __nv_bfloat16* xb = x + b * H * W * Cin;
  if (vec) {  // Cin % 8 == 0, 16-byte aligned rows: 8-channel chunks
    const int cv = g.Cp / 8, cin_v = Cin / 8;
    const int nx = g.HR * g.HC * cv;
    for (int i = threadIdx.x; i < nx; i += blockDim.x) {
      const int c8 = i % cv, pix = i / cv;
      const int hy = pix / g.HC, hx = pix % g.HC;
      const int iy = iy0 + hy, ix = ix0 + hx;
      __nv_bfloat16* dst = sx + (size_t)pix * g.xs + c8 * 8;
      if (c8 < cin_v && iy >= 0 && iy < H && ix >= 0 && ix < W)
        cp_async16(dst, xb + ((long long)iy * W + ix) * Cin + c8 * 8);
      else
        *reinterpret_cast<uint4*>(dst) = make_uint4(0, 0, 0, 0);
    }
    const int nw = CN_BN * 9 * cv;
    for (int i = threadIdx.x; i < nw; i += blockDim.x) {
      const int c8 = i % cv, r = i / cv;
      const int tap = r % 9, n = r / 9;
      __nv_bfloat16* dst = sw + (size_t)n * g.ws + tap * g.Cp + c8 * 8;
      if (c8 < cin_v && n0 + n < Cout)
        cp_async16(dst, w + ((long long)(n0 + n) * 9 + tap) * Cin + c8 * 8);
      else
        *reinterpret_cast<uint4*>(dst) = make_uint4(0, 0, 0, 0);
    }
    cp_async_wait_all();
  } else {
    const int nx = g.HR * g.HC * g.Cp;
    for (int i = threadIdx.x; i < nx; i += blockDim.x) {
      const int c = i % g.Cp, pix = i / g.Cp;
      const int hy = pix / g.HC, hx = pix % g.HC;
      const int iy = iy0 + hy, ix = ix0 + hx;
      sx[(size_t)pix * g.xs + c] =
          (c < Cin && iy >= 0 && iy < H && ix >= 0 && ix < W) ? xb[((long long)iy * W + ix) * Cin + c] : zero;
    }
    const int nw = CN_BN * 9 * g.Cp;
    for (int i = threadIdx.x; i < nw; i += blockDim.x) {
      const int c = i % g.Cp, r = i / g.Cp;
      const int tap = r % 9, n = r / 9;
      sw[(size_t)n * g.ws + tap * g.Cp + c] =
          (c < Cin && n0 + n < Cout) ? w[((long long)(n0 + n) * 9 + tap) * Cin + c] : zero;
    }
  }
  __syncthreads();

  // ---- 9 taps x Cp/16 k-steps of mma.m16n8k16 per warp ---------------------------------------------------------
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q = lane >> 3, r8 = lane & 7;
  // A (ldmatrix.x4): lane supplies row (r8 + (q&1)*8) = output pixel ox0 + that, k offset (q>>1)*8
  const int a_px = r8 + (q & 1) * 8, a_k = (q >> 1) * 8;
  // B (ldmatrix.x4 over two n8 tiles): lane supplies n = r8 + (q>>1)*8, k offset (q&1)*8
  const int b_n = r8 + (q >> 1) * 8, b_k = (q & 1) * 8;
  float acc[4][4];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[j][e] = 0.0f;

  for (int tap = 0; tap < 9; ++tap) {
    const int ky = tap / 3, kx = tap % 3;
    const __nv_bfloat16* arow = sx + ((size_t)(warp * stride + ky) * g.HC + a_px * stride + kx) * g.xs + a_k;
    const __nv_bfloat16* brow = sw + (size_t)b_n * g.ws + tap * g.Cp + b_k;
    for (int c0 = 0; c0 < g.Cp; c0 += 16) {
      uint32_t a[4], b01[4], b23[4];
      ldmatrix_x4(a, arow + c0);
      ldmatrix_x4(b01, brow + c0);
      ldmatrix_x4(b23, brow + (size_t)16 * g.ws + c0);
      mma_bf16_16816(acc[0], a, b01[0], b01[1]);
      mma_bf16_16816(acc[1], a, b01[2], b01[3]);
      mma_bf16_16816(acc[2], a, b23[0], b23[1]);
      mma_bf16_16816(acc[3], a, b23[2], b23[3]);
    }
  }

  // ---- epilogue: accumulator (row lane/4 [+8], cols 2*(lane%4) + {0,1}) -> bias, SiLU, bf16 -------------------
  const int oy = oy0 + warp;
  if (oy >= Ho) return;
  __nv_bfloat16* yrow = y + (b * Ho + oy) * (long long)Wo * Cout;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int n = n0 + j * 8 + 2 * (lane & 3);
    if (n >= Cout) continue;  // Cout % 8 == 0: both columns of the pair are valid or neither
    const float b0 = bias ? bias[n] : 0.0f, b1 = bias ? bias[n + 1] : 0.0f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int ox = ox0 + (lane >> 2) + h * 8;
      if (ox >= Wo) continue;
      float v0 = acc[j][2 * h] + b0, v1 = acc[j][2 * h + 1] + b1;
      if (act == B200MIX_ACT_SILU) {
        v0 = v0 / (1.0f + __expf(-v0));
        v1 = v1 / (1.0f + __expf(-v1));
      }
      *reinterpret_cast<uint32_t*>(yrow + (long long)ox * Cout + n) = pack_bf16x2(v0, v1);
    }
  }
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int b200mix_conv3x3_narrow(const void* x, const void* w, const float* bias, void* y, int64_t B, int64_t H,
                                      int64_t W, int64_t Cin, int64_t Cout, int32_t stride, int32_t act,
                                      void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(x && w && y, "conv3x3_narrow: null pointer");
  B200_CHECK_ARG(Cin >= 1 && Cin <= 128, "conv3x3_narrow: Cin=%lld must be in [1, 128]", (long long)Cin);
  B200_CHECK_ARG(Cout >= 8 && Cout <= 256 && Cout % 8 == 0, "conv3x3_narrow: Cout=%lld must be a multiple of 8 in [8, 256]",
                 (long long)Cout);
  B200_CHECK_ARG(stride == 1 || stride == 2, "conv3x3_narrow: stride must be 1 or 2");
  B200_CHECK_ARG(act == B200MIX_ACT_NONE || act == B200MIX_ACT_SILU, "conv3x3_narrow: act must be NONE or SILU");
  B200_CHECK_ARG(B > 0 && H > 0 && W > 0, "conv3x3_narrow: bad shape");
  B200_CHECK_ARG(stride == 1 || (H % 2 == 0 && W % 2 == 0), "conv3x3_narrow: stride 2 needs even H, W (got %lldx%lld)",
                 (long long)H, (long long)W);
  B200_CHECK_ARG(H * W * Cin < (1ll << 31) && H * W * Cout < (1ll << 31), "conv3x3_narrow: image too large");
  const NarrowGeom g = narrow_geom((int)Cin, stride);
  const size_t smem = narrow_smem_bytes(g);
  static bool configured = false;
  if (!configured) {
    B200_CUDA(cudaFuncSetAttribute(conv3x3_narrow_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   narrow_smem_bytes(narrow_geom(128, 2))));
    configured = true;
  }
  const int Ho = (int)(H / stride), Wo = (int)(W / stride);
  const int tiles_x = (Wo + CN_TW - 1) / CN_TW, tiles_y = (Ho + CN_WARPS - 1) / CN_WARPS;
  const int n_slices = (int)((Cout + CN_BN - 1) / CN_BN);
  const long long blocks = B * tiles_x * tiles_y * n_slices;
  B200_CHECK_ARG(blocks < (1ll << 31), "conv3x3_narrow: grid too large");
  const int vec = (Cin % 8 == 0 && reinterpret_cast<uintptr_t>(x) % 16 == 0 && reinterpret_cast<uintptr_t>(w) % 16 == 0);
  B200_CUDA(launch_pdl(conv3x3_narrow_kernel, dim3((unsigned)blocks), dim3(CN_WARPS * 32), smem,
                       reinterpret_cast<cudaStream_t>(stream), 1, reinterpret_cast<const __nv_bfloat16*>(x),
                       reinterpret_cast<const __nv_bfloat16*>(w), bias, reinterpret_cast<__nv_bfloat16*>(y), (int)H,
                       (int)W, (int)Cin, (int)Cout, stride, act, tiles_x, tiles_y, n_slices, vec));
  return 0;
}
