// Flash-style scaled-dot-product attention on Hopper tensor cores (wgmma).
//
// One CTA = one 128-row query tile of one (batch, head). 288 threads:
//   warp 8     TMA producer: Q once, then K/V tiles through a shared-memory ring (128B swizzle)
//   warps 0-7  two consumer warpgroups; warpgroup g owns query rows [64 g, 64 g + 64): S = Q K_j^T (wgmma, both operands
//              K-major in shared memory, fp32 accumulators in registers), online softmax in fp32 with exp2 and a lazy
//              rescale of the register-resident O (only when the running max grows by more than 2^8), then
//              O += P_j V_j with P taken straight from registers as the bf16 A operand and V consumed in its natural
//              [kv, d] layout as an MN-major B operand. The two warpgroups interleave: while one exponentiates, the
//              other's MMAs use the tensor cores.
//
// Semantics follow the reference's `math` SDPA (ppdiffusers/patches/paddle_patch.py:445-461): softmax(q k^T * scale
// [+ causal]) v, [B,S,H,D] in / out; GQA per modeling_qwen2_vl.py:497-506; varlen block-diagonal per :354-381.
#include <algorithm>

#include "common.cuh"
#include "ptx.cuh"

namespace b200 {

struct AttnParams {
  int Hq, Hkv, Sq, Sk;
  float scale_log2;
  int causal;
  const int* cu;
  int nseq;
  const int* kv_lens;  // optional per-batch number of valid keys (<= Sk)
  int q_pos[3], k_pos[3], v_pos[3];  // tensor-map coordinate slot (1..3) of (seq, head, batch)
  __nv_bfloat16* o;
  long long o_sb, o_ss, o_sh;
  // optional additive mask / bias on the scaled scores (attn_mask of scaled_dot_product_attention_,
  // paddle_patch.py:418,454-455): element (b, h, q, k) at mask + b*m_sb + h*m_sh + q*m_sq + k; a stride of 0 broadcasts
  const void* mask;
  int mask_fp32;
  long long m_sb, m_sh, m_sq;
  float inv_scale;  // 1 / scale: the bias is folded into the raw score as s + mask * inv_scale
};

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ void tma_load_rows(void* dst, const CUtensorMap* m, uint64_t* bar, const int (&pos)[3], int d0,
                                              int s0, int h, int b) {
  int c[4];
  c[0] = d0;
  c[pos[0]] = s0;
  c[pos[1]] = h;
  c[pos[2]] = b;
  tma_load_4d(dst, m, bar, c[0], c[1], c[2], c[3]);
}

__device__ __forceinline__ float mask_value(const AttnParams& p, long long row_off, int k) {
  return p.mask_fp32 ? __ldg(reinterpret_cast<const float*>(p.mask) + row_off + k)
                     : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p.mask)[row_off + k]);
}

// BN = keys per K/V block; KS = K/V ring depth. The register budget of a consumer thread (S: BN / 2, O: D / 2, P: BN / 4
// fp32 / bf16x2 registers) sets BN: 128 keys for D = 64, 64 keys for D = 128 and 192.
template <int D, int BN>
struct AttnCfg {
  static constexpr int KS = 2;
  // dynamic smem is declared __align__(1024) (128B-swizzle atoms), so no alignment slack
  static constexpr int SMEM = 128 * D * 2 + 2 * KS * BN * D * 2 + 256;
};
constexpr int ATTN_THREADS = 288;

template <int D, int BN>
__global__ void __launch_bounds__(ATTN_THREADS, 1)
    attn_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const __grid_constant__ AttnParams p) {
  constexpr int DC = D / 64;               // 64-wide head-dim chunks (one 128B swizzle atom each)
  constexpr int TILE_BYTES = 128 * D * 2;  // the 128-row Q tile
  constexpr int KV_BYTES = BN * D * 2;     // one BN-row tile of K / V
  constexpr int KV_PANEL = BN * 128;       // one 64-wide head-dim panel of it
  constexpr int KS = AttnCfg<D, BN>::KS;

  // cu_seqlens / kv_lens are read right away: if they are given, wait for the previous kernel first
  if (p.cu || p.kv_lens) pdl_wait();
  // ---- which tile am I? (uniform across the CTA) ----
  int qt = blockIdx.x;
  const int h = blockIdx.y, b = blockIdx.z;
  int q_begin, q_end, kv_begin, kv_end, q_rel0, causal_off;
  if (p.cu) {
    int i = 0;
    bool found = false;
    for (; i < p.nseq; ++i) {
      const int len = p.cu[i + 1] - p.cu[i];
      const int nt = (len + 127) >> 7;
      if (qt < nt) {
        found = true;
        break;
      }
      qt -= nt;
    }
    if (!found) return;
    q_begin = p.cu[i] + qt * 128;
    q_end = p.cu[i + 1];
    kv_begin = p.cu[i];
    kv_end = p.cu[i + 1];
    q_rel0 = qt * 128;
    causal_off = 0;
  } else {
    q_begin = qt * 128;
    q_end = p.Sq;
    kv_begin = 0;
    kv_end = p.kv_lens ? min(p.Sk, p.kv_lens[b]) : p.Sk;
    q_rel0 = q_begin;
    causal_off = p.Sk - p.Sq;
  }
  const int kv_len = kv_end - kv_begin;
  int n_kv = kv_len;
  if (p.causal) n_kv = min(kv_len, q_rel0 + 128 + causal_off);
  const int n_tiles = (n_kv + BN - 1) / BN;
  const int hk = h / (p.Hq / p.Hkv);

  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + TILE_BYTES;
  uint8_t* sV = sK + KS * KV_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + KS * KV_BYTES);
  uint64_t* q_full = bars;            // 1
  uint64_t* k_full = bars + 1;        // KS
  uint64_t* k_empty = k_full + KS;    // KS
  uint64_t* v_full = k_empty + KS;    // KS
  uint64_t* v_empty = v_full + KS;    // KS

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < KS; ++s) {
      mbar_init(&k_full[s], 1);
      mbar_init(&k_empty[s], 8);  // every consumer warp
      mbar_init(&v_full[s], 1);
      mbar_init(&v_empty[s], 8);
    }
    fence_barrier_init();
    prefetch_tmap(&tmQ);
    prefetch_tmap(&tmK);
    prefetch_tmap(&tmV);
  }
  __syncthreads();
  pdl_wait();
  pdl_launch_dependents();

  if (warp == 8) {
    // ===== TMA producer (converged warp, one elected lane issues: see ptx.cuh) =====
    if (elect_one_sync()) {
      mbar_expect_tx(q_full, TILE_BYTES);
#pragma unroll
      for (int dc = 0; dc < DC; ++dc) tma_load_rows(sQ + dc * 16384, &tmQ, q_full, p.q_pos, dc * 64, q_begin, h, b);
    }
    __syncwarp();
    int st = 0;
    uint32_t ph = 0;
    for (int j = 0; j < n_tiles; ++j) {
      const int row0 = kv_begin + j * BN;
      mbar_wait(&k_empty[st], ph ^ 1);
      if (elect_one_sync()) {
        mbar_expect_tx(&k_full[st], KV_BYTES);
#pragma unroll
        for (int dc = 0; dc < DC; ++dc)
          tma_load_rows(sK + st * KV_BYTES + dc * KV_PANEL, &tmK, &k_full[st], p.k_pos, dc * 64, row0, hk, b);
      }
      __syncwarp();
      mbar_wait(&v_empty[st], ph ^ 1);
      if (elect_one_sync()) {
        mbar_expect_tx(&v_full[st], KV_BYTES);
#pragma unroll
        for (int dc = 0; dc < DC; ++dc)
          tma_load_rows(sV + st * KV_BYTES + dc * KV_PANEL, &tmV, &v_full[st], p.v_pos, dc * 64, row0, hk, b);
      }
      __syncwarp();
      if (++st == KS) st = 0, ph ^= 1;
    }
    return;
  }

  // ===== consumers: accumulator fragment rows r0 = 16 w + lane / 4 and r0 + 8 of the warpgroup's 64 rows, columns
  // 8 n + 2 (lane % 4) + {0, 1} of every 8-column block n =====
  const int grp = warp >> 2, w = warp & 3;
  const int lm = lane & 3;
  const int rloc = 64 * grp + 16 * w + (lane >> 2);  // query row (in the tile) of fragment elements 0, 1; +8 for 2, 3
  int row_limit[2];
  long long mask_row[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int row = rloc + 8 * e;
    row_limit[e] = p.causal ? min(kv_len, q_rel0 + row + causal_off + 1) : kv_len;
    // additive mask row of this query (rows past the end of the sequence read row Sq - 1: in bounds, never stored)
    mask_row[e] = static_cast<long long>(b) * p.m_sb + static_cast<long long>(h) * p.m_sh +
                  static_cast<long long>(min(q_begin + row, p.Sq - 1)) * p.m_sq;
  }
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.0f, 0.0f};
  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.0f;
  const uint32_t q_addr = smem_u32(sQ) + grp * 64 * 128;
  mbar_wait(q_full, 0);
  int st = 0;
  uint32_t ph = 0;
  for (int j = 0; j < n_tiles; ++j) {
    float s[BN / 2];
    mbar_wait(&k_full[st], ph);
    const uint32_t k_addr = smem_u32(sK + st * KV_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < D / 16; ++k)
      wgmma_ss(s, make_wgmma_desc_sw128(q_addr + (k >> 2) * 16384 + (k & 3) * 32, 16, 1024),
               make_wgmma_desc_sw128(k_addr + (k >> 2) * KV_PANEL + (k & 3) * 32, 16, 1024), k != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(s);
    if (lane == 0) mbar_arrive(&k_empty[st]);

    const int k0 = j * BN;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int n = 0; n < BN / 8; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int col = 8 * n + 2 * lm + (e & 1);
        float v = s[4 * n + e];
        if (p.mask && k0 + col < kv_len) v = fmaf(mask_value(p, mask_row[e >> 1], kv_begin + k0 + col), p.inv_scale, v);
        v = (k0 + col < row_limit[e >> 1]) ? v : -INFINITY;  // columns [0, limit) of this tile are visible
        s[4 * n + e] = v;
        mx[e >> 1] = fmaxf(mx[e >> 1], v);
      }
    float alpha[2], m_scaled[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 1));
      mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 2));
      const float m_cand = fmaxf(m_run[e], mx[e]);
      const bool grow = (m_cand - m_run[e]) * p.scale_log2 > 8.0f;  // also true for the first finite tile (m = -inf)
      alpha[e] = 1.0f;
      if (grow) {
        alpha[e] = fast_exp2((m_run[e] - m_cand) * p.scale_log2);
        m_run[e] = m_cand;
        l_run[e] *= alpha[e];
      }
      m_scaled[e] = (m_run[e] == -INFINITY) ? 0.0f : m_run[e] * p.scale_log2;
    }
#pragma unroll
    for (int n = 0; n < D / 8; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e) o[4 * n + e] *= alpha[e >> 1];
    // P = exp2(s * scale_log2 - m) as bf16 A fragments of the PV MMA: 16-key slice kk is n8 blocks 2 kk and 2 kk + 1
    uint32_t pa[BN / 16][4];
#pragma unroll
    for (int kk = 0; kk < BN / 16; ++kk)
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int n = 2 * kk + half;
        const float e0 = fast_exp2(fmaf(s[4 * n + 0], p.scale_log2, -m_scaled[0]));
        const float e1 = fast_exp2(fmaf(s[4 * n + 1], p.scale_log2, -m_scaled[0]));
        const float e2 = fast_exp2(fmaf(s[4 * n + 2], p.scale_log2, -m_scaled[1]));
        const float e3 = fast_exp2(fmaf(s[4 * n + 3], p.scale_log2, -m_scaled[1]));
        l_run[0] += e0 + e1;
        l_run[1] += e2 + e3;
        pa[kk][2 * half + 0] = pack_bf16x2(e0, e1);
        pa[kk][2 * half + 1] = pack_bf16x2(e2, e3);
      }
    mbar_wait(&v_full[st], ph);
    const uint32_t v_addr = smem_u32(sV + st * KV_BYTES);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BN / 16; ++kk)
      wgmma_rs_mn(o, pa[kk], make_wgmma_desc_sw128(v_addr + kk * 2048, KV_PANEL, 1024), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(o);
    if (lane == 0) mbar_arrive(&v_empty[st]);
    if (++st == KS) st = 0, ph ^= 1;
  }

  // ---- epilogue: O / l -> global (a row without any visible key gets zeros: O was never written) ----
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    l_run[e] += __shfl_xor_sync(0xffffffffu, l_run[e], 1);
    l_run[e] += __shfl_xor_sync(0xffffffffu, l_run[e], 2);
  }
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const float inv_l = (l_run[e] > 0.0f) ? 1.0f / l_run[e] : 0.0f;
    const int q_abs = q_begin + rloc + 8 * e;
    if (q_abs >= q_end) continue;
    __nv_bfloat16* dst = p.o + static_cast<long long>(b) * p.o_sb + static_cast<long long>(q_abs) * p.o_ss +
                         static_cast<long long>(h) * p.o_sh + 2 * lm;
#pragma unroll
    for (int n = 0; n < D / 8; ++n)
      *reinterpret_cast<uint32_t*>(dst + 8 * n) = pack_bf16x2(o[4 * n + 2 * e] * inv_l, o[4 * n + 2 * e + 1] * inv_l);
  }
}

// Build a 4-D tensor map over (d, seq, head, batch) for a [.., D]-contiguous bf16 tensor with arbitrary (16-byte
// aligned) strides; outer dims are ordered by increasing stride. pos[] returns the coordinate slot of (seq, head, batch).
static int make_attn_tmap(CUtensorMap* tm, const void* ptr, int64_t D, int64_t S, int64_t H, int64_t B, int64_t ss,
                          int64_t sh, int64_t sb, int pos[3], uint32_t box_rows = 128) {
  struct Dim {
    int64_t size, stride;
    int which;
  };
  Dim d[3] = {{S, ss, 0}, {H, sh, 1}, {B, sb, 2}};
  int64_t span = D;
  for (int i = 0; i < 3; ++i)
    if (d[i].size > 1) span = std::max(span, d[i].size * d[i].stride);
  for (int i = 0; i < 3; ++i)
    if (d[i].size <= 1) d[i].stride = (span + 7) / 8 * 8 + 8 * (i + 1);  // size-1 dims: any valid stride, sorted last
  std::sort(d, d + 3, [](const Dim& a, const Dim& b2) { return a.stride < b2.stride; });
  uint64_t dims[4] = {(uint64_t)D, 0, 0, 0};
  uint64_t strides[3];
  uint32_t box[4] = {64, 1, 1, 1};
  for (int i = 0; i < 3; ++i) {
    dims[i + 1] = (uint64_t)d[i].size;
    strides[i] = (uint64_t)d[i].stride * 2;
    pos[d[i].which] = i + 1;
    if (d[i].which == 0) box[i + 1] = box_rows;
  }
  return encode_tmap_bf16_sw128(tm, ptr, 4, dims, strides, box);
}

template <int D, int BN>
static int launch_attn(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const AttnParams& p,
                       dim3 grid, cudaStream_t stream) {
  constexpr int smem_bytes = AttnCfg<D, BN>::SMEM;
  static_assert(smem_bytes <= 227 * 1024, "K/V ring does not fit shared memory");
  static bool configured = false;
  if (!configured) {
    B200_CUDA(cudaFuncSetAttribute(attn_kernel<D, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    configured = true;
  }
  B200_CUDA(launch_pdl(attn_kernel<D, BN>, grid, dim3(ATTN_THREADS), smem_bytes, stream, 1, tq, tk, tv, p));
  return 0;
}

// D = 64: 1 = 64-key blocks, 0 (default) = 128-key blocks. Kept selectable for A/B runs and tested.
static int g_attn_bn64 = 0;

}  // namespace b200

using namespace b200;

extern "C" void b200mix_debug_attn_bn64(int on) { b200::g_attn_bn64 = on; }

extern "C" int b200mix_sdpa(const void* q, const void* k, const void* v, void* o, int64_t B, int64_t Hq, int64_t Hkv,
                            int64_t Sq, int64_t Sk, int64_t D, int64_t q_sb, int64_t q_ss, int64_t q_sh, int64_t k_sb,
                            int64_t k_ss, int64_t k_sh, int64_t v_sb, int64_t v_ss, int64_t v_sh, int64_t o_sb,
                            int64_t o_ss, int64_t o_sh, float scale, int32_t causal, const int32_t* cu_seqlens,
                            int32_t nseq, const int32_t* kv_lens, const void* attn_mask, int32_t mask_fp32,
                            int64_t m_sb, int64_t m_sh, int64_t m_sq, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(q && k && v && o, "sdpa: null pointer");
  B200_CHECK_ARG(D == 64 || D == 128 || D == 192,
                 "sdpa: head_dim %lld unsupported (64, 128 or 192; pad at weight-load time)",
                 (long long)D);
  B200_CHECK_ARG(B > 0 && Hq > 0 && Hkv > 0 && Sq > 0 && Sk > 0, "sdpa: bad shape");
  B200_CHECK_ARG(Hq % Hkv == 0, "sdpa: Hq %% Hkv != 0");
  B200_CHECK_ARG(!cu_seqlens || (B == 1 && nseq > 0 && Sq == Sk), "sdpa: varlen mode needs B == 1, Sq == Sk");
  // bottom-right aligned causal mask (query i sees keys <= i + Sk - Sq): with Sq > Sk the first rows see nothing
  B200_CHECK_ARG(!(causal && Sq > Sk), "sdpa: causal attention needs Sq <= Sk (got Sq=%lld, Sk=%lld)", (long long)Sq,
                 (long long)Sk);
  // the reference drops attn_mask when is_causal is set (paddle_patch.py:451-455,502,513); refuse the combination
  B200_CHECK_ARG(!(attn_mask && (causal || cu_seqlens)), "sdpa: attn_mask cannot be combined with causal / varlen");
  B200_CHECK_ARG(!attn_mask || scale != 0.0f, "sdpa: attn_mask needs a non-zero scale");
  const int64_t all_strides[12] = {q_sb, q_ss, q_sh, k_sb, k_ss, k_sh, v_sb, v_ss, v_sh, o_sb, o_ss, o_sh};
  for (int i = 0; i < 12; ++i)
    B200_CHECK_ARG(all_strides[i] % 8 == 0, "sdpa: stride %d (= %lld) must be a multiple of 8 elements", i,
                   (long long)all_strides[i]);
  B200_CHECK_ARG(reinterpret_cast<uintptr_t>(o) % 16 == 0, "sdpa: output must be 16-byte aligned");

  AttnParams p = {};
  p.Hq = (int)Hq, p.Hkv = (int)Hkv, p.Sq = (int)Sq, p.Sk = (int)Sk;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.causal = causal;
  p.cu = cu_seqlens;
  p.nseq = nseq;
  p.kv_lens = kv_lens;
  p.o = reinterpret_cast<__nv_bfloat16*>(o);
  p.o_sb = o_sb, p.o_ss = o_ss, p.o_sh = o_sh;
  p.mask = attn_mask;
  p.mask_fp32 = mask_fp32;
  p.m_sb = m_sb, p.m_sh = m_sh, p.m_sq = m_sq;
  p.inv_scale = attn_mask ? 1.0f / scale : 0.0f;
  CUtensorMap tq, tk, tv;
  if (int rc = make_attn_tmap(&tq, q, D, Sq, Hq, B, q_ss, q_sh, q_sb, p.q_pos)) return rc;
  const uint32_t kv_box = (D == 64 && !g_attn_bn64) ? 128u : 64u;
  if (int rc = make_attn_tmap(&tk, k, D, Sk, Hkv, B, k_ss, k_sh, k_sb, p.k_pos, kv_box)) return rc;
  if (int rc = make_attn_tmap(&tv, v, D, Sk, Hkv, B, v_ss, v_sh, v_sb, p.v_pos, kv_box)) return rc;
  int64_t q_tiles = (Sq + 127) / 128 + (cu_seqlens ? nseq : 0);
  dim3 grid((unsigned)q_tiles, (unsigned)Hq, (unsigned)B);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (D == 64) return kv_box == 64 ? launch_attn<64, 64>(tq, tk, tv, p, grid, st) : launch_attn<64, 128>(tq, tk, tv, p, grid, st);
  if (D == 128) return launch_attn<128, 64>(tq, tk, tv, p, grid, st);
  return launch_attn<192, 64>(tq, tk, tv, p, grid, st);
}
