// LoRA weight update: b200mix_lora_apply rebuilds every device-layout weight a set of LoRAs touches in one launch.
// Replaces LoRACompatibleLinear._fuse_lora / _unfuse_lora (ppdiffusers/models/lora.py:117-165) and
// LoRACompatibleConv._fuse_lora / _unfuse_lora (:312-362), which merge W + scale * (down @ up) layer by layer in fp32.
//
// Work: a flat list of (item, 64-row tile) units, one item per target (a weight or a row slice of a batched weight).
// A CTA of 4 warps takes one unit at a time (persistent grid): it stages the tile's 64 rows of U in shared memory,
// rounded to tf32, then each warp owns 16 rows and sweeps K in 64-column chunks, computing U @ D with
// mma.sync.m16n8k8 tf32 (fp32 accumulate, j in order) and writing out = bf16(base + col_scale * acc) in the register
// epilogue. The colsum difference of a row is summed by the 4 lanes that own it, each over its own columns in order,
// then combined by a fixed butterfly, so every output is deterministic.
#include "common.cuh"
#include "ptx.cuh"

#include <cuda_bf16.h>

#include <vector>

namespace b200 {

struct LoraWork {
  b200mix_lora_item it;
  long long tile0;  // first global tile index of this item
};

constexpr int kLoraRows = 64;     // rows per work unit (4 warps x 16)
constexpr int kLoraCols = 64;     // columns per warp step (8 n-tiles of 8)
constexpr int kLoraThreads = 128;

__device__ __forceinline__ uint32_t to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
               "{%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(kLoraThreads) lora_apply_kernel(const LoraWork* __restrict__ work, int n_items,
                                                                  long long total_tiles) {
  extern __shared__ uint32_t u_s[];  // [kLoraRows][R + 4] tf32 bits (the +4 makes the A-fragment reads conflict-free)
  pdl_wait();
  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    int lo = 0, hi = n_items - 1;  // last item with tile0 <= tile
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (work[mid].tile0 <= tile) lo = mid; else hi = mid - 1;
    }
    const b200mix_lora_item it = work[lo].it;
    const long long row0 = (tile - work[lo].tile0) * kLoraRows;
    const int R = (int)it.R, ldu = R + 4;
    const long long K = it.K;
    __syncthreads();  // the previous unit's readers of u_s are done
    for (int i = threadIdx.x; i < kLoraRows * (R / 4); i += kLoraThreads) {
      const int r = i / (R / 4), c = (i - r * (R / 4)) * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (row0 + r < it.N) v = __ldg(reinterpret_cast<const float4*>(it.U + (row0 + r) * R + c));
      uint32_t* dst = u_s + r * ldu + c;
      dst[0] = to_tf32(v.x), dst[1] = to_tf32(v.y), dst[2] = to_tf32(v.z), dst[3] = to_tf32(v.w);
    }
    __syncthreads();
    const long long rw = row0 + warp * 16;  // this warp's first row
    if (rw >= it.N) continue;
    const uint32_t* ua = u_s + (warp * 16 + g) * ldu + t;
    const long long ra = rw + g, rb = ra + 8;
    const bool va = ra < it.N, vb = rb < it.N;
    const __nv_bfloat16* base = static_cast<const __nv_bfloat16*>(it.base);
    __nv_bfloat16* out = static_cast<__nv_bfloat16*>(it.out);
    float dsum_a = 0.f, dsum_b = 0.f;
    for (long long c0 = 0; c0 < K; c0 += kLoraCols) {
      float acc[8][4];
#pragma unroll
      for (int n = 0; n < 8; ++n) acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f;
      const float* dcol = it.D + c0 + g;
      for (int j = 0; j < R; j += 8) {
        const uint32_t a[4] = {ua[j], ua[8 * ldu + j], ua[j + 4], ua[8 * ldu + j + 4]};
        const float* d0 = dcol + (long long)(j + t) * K;
        const float* d1 = d0 + 4 * K;
#pragma unroll
        for (int n = 0; n < 8; ++n) {
          if (c0 + n * 8 < K) mma_tf32(acc[n], a, to_tf32(__ldg(d0 + n * 8)), to_tf32(__ldg(d1 + n * 8)));
        }
      }
#pragma unroll
      for (int n = 0; n < 8; ++n) {
        const long long col = c0 + n * 8 + 2 * t;
        if (col >= K) continue;
        float s0 = 1.f, s1 = 1.f;
        if (it.col_scale) s0 = __ldg(it.col_scale + col), s1 = __ldg(it.col_scale + col + 1);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!(h ? vb : va)) continue;
          const long long r = h ? rb : ra;
          const __nv_bfloat162 b2 = *reinterpret_cast<const __nv_bfloat162*>(base + r * it.ld_base + col);
          const float b0 = __bfloat162float(b2.x), b1 = __bfloat162float(b2.y);
          const float e0 = __fmul_rn(s0, acc[n][2 * h]), e1 = __fmul_rn(s1, acc[n][2 * h + 1]);
          const __nv_bfloat16 o0 = e0 == 0.f ? b2.x : __float2bfloat16_rn(__fadd_rn(b0, e0));
          const __nv_bfloat16 o1 = e1 == 0.f ? b2.y : __float2bfloat16_rn(__fadd_rn(b1, e1));
          *reinterpret_cast<__nv_bfloat162*>(out + r * it.ld_out + col) = __halves2bfloat162(o0, o1);
          const float dd = __fadd_rn(__fsub_rn(__bfloat162float(o0), b0), __fsub_rn(__bfloat162float(o1), b1));
          if (h) dsum_b = __fadd_rn(dsum_b, dd); else dsum_a = __fadd_rn(dsum_a, dd);
        }
      }
    }
    if (it.colsum) {
      dsum_a = __fadd_rn(dsum_a, __shfl_xor_sync(0xffffffffu, dsum_a, 1));
      dsum_a = __fadd_rn(dsum_a, __shfl_xor_sync(0xffffffffu, dsum_a, 2));
      dsum_b = __fadd_rn(dsum_b, __shfl_xor_sync(0xffffffffu, dsum_b, 1));
      dsum_b = __fadd_rn(dsum_b, __shfl_xor_sync(0xffffffffu, dsum_b, 2));
      if (t == 0) {
        if (va) it.colsum[ra] = dsum_a == 0.f ? it.colsum_base[ra] : __fadd_rn(it.colsum_base[ra], dsum_a);
        if (vb) it.colsum[rb] = dsum_b == 0.f ? it.colsum_base[rb] : __fadd_rn(it.colsum_base[rb], dsum_b);
      }
    }
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200mix_lora_workspace_size(int32_t n_items, int64_t* bytes) {
  B200_CHECK_ARG(bytes && n_items >= 1, "lora_workspace_size: need at least one item");
  *bytes = (int64_t)n_items * (int64_t)sizeof(LoraWork);
  return 0;
}

extern "C" int b200mix_lora_apply(const b200mix_lora_item* items, int32_t n_items, void* workspace,
                                  int64_t workspace_bytes, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(items && n_items >= 1 && workspace, "lora_apply: need at least one item and a workspace");
  int64_t need = 0;
  b200mix_lora_workspace_size(n_items, &need);
  auto al16 = [](const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 == 0; };
  B200_CHECK_ARG(workspace_bytes >= need && al16(workspace), "lora_apply: workspace of %lld bytes < %lld or unaligned",
                 (long long)workspace_bytes, (long long)need);
  std::vector<LoraWork> w(n_items);
  long long tiles = 0;
  int max_r = 8;
  for (int i = 0; i < n_items; ++i) {
    const b200mix_lora_item& it = items[i];
    B200_CHECK_ARG(it.out && it.base && it.U && it.D && al16(it.out) && al16(it.base) && al16(it.U) && al16(it.D),
                   "lora_apply: item %d: out, base, U and D must be 16-byte aligned device pointers", i);
    B200_CHECK_ARG(it.N > 0 && it.K > 0 && it.K % 8 == 0 && it.R > 0 && it.R % 8 == 0 &&
                       it.R <= B200MIX_LORA_MAX_RANK && it.ld_out >= it.K && it.ld_base >= it.K &&
                       it.ld_out % 8 == 0 && it.ld_base % 8 == 0,
                   "lora_apply: item %d: bad shape N=%lld K=%lld R=%lld ld_out=%lld ld_base=%lld", i, (long long)it.N,
                   (long long)it.K, (long long)it.R, (long long)it.ld_out, (long long)it.ld_base);
    B200_CHECK_ARG(!it.colsum == !it.colsum_base, "lora_apply: item %d: colsum and colsum_base go together", i);
    w[i].it = it;
    w[i].tile0 = tiles;
    tiles += (it.N + kLoraRows - 1) / kLoraRows;
    if (it.R > max_r) max_r = (int)it.R;
  }
  const size_t smem = (size_t)kLoraRows * (max_r + 4) * sizeof(uint32_t);
  B200_CUDA(cudaFuncSetAttribute(lora_apply_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  // pageable source: the call returns once the table is staged, so `w` may go out of scope
  B200_CUDA(cudaMemcpyAsync(workspace, w.data(), need, cudaMemcpyHostToDevice, s));
  int per_sm = 0;
  B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lora_apply_kernel, kLoraThreads, smem));
  const long long cap = (long long)num_sms() * (per_sm > 0 ? per_sm : 1);
  const unsigned grid = (unsigned)(tiles < cap ? tiles : cap);
  B200_CUDA(launch_pdl(lora_apply_kernel, dim3(grid), dim3(kLoraThreads), smem, s, 1,
                       static_cast<const LoraWork*>(workspace), (int)n_items, tiles));
  return 0;
}
