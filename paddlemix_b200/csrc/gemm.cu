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
#include "act.cuh"

#include <algorithm>
#include <cstdlib>
#include <mutex>
#include <type_traits>

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
  double ln_inv_k;            // 2^-24 / K
  // stream-K head (see SegIter): the first sk_tiles super-tiles are cut into equal k-block ranges, one per cluster
  int sk_tiles;
  float4* sk_ws;          // [cluster][cta rank][n8 block][consumer thread] fp32 partial accumulators (fragment layout)
  unsigned int* sk_flags; // [cluster][cta rank]: 1 = the partial of that CTA's tail piece is in sk_ws
};

// ---- work schedule -------------------------------------------------------------------------------------------------
// A problem of T super-tiles (256 x BN) on C clusters needs ceil(T / C) rounds; SDXL's 8192 x 1280 projections have
// T = 160 on the C = 66 clusters of 132 SMs: 2.42 rounds of work in 3 rounds of time. The schedule therefore starts with a STREAM-K head: the
// first sk_tiles = C + (T mod C) tiles are laid end to end in units of one 64-deep k-block and cluster c takes the
// contiguous unit range [c, c+1) * units / C (>= one whole tile, so a tile is shared by at most two clusters: its k
// range splits into a HEAD piece = the last piece of cluster c and a TAIL piece = the first piece of cluster c + 1).
// The tail piece's fp32 accumulators go to a per-cluster workspace slot right after that cluster's first few k-blocks;
// the head piece's epilogue - which runs (1 + T mod C / C) tiles later - adds them to its own accumulators and finishes
// the tile (fixed split and fixed order: results are reproducible run to run). The remaining T - sk_tiles tiles (a
// multiple of C) follow round-robin as before. Every cluster thus gets T / C tiles' worth of k-blocks.
constexpr int SK_WS_FLOAT4_PER_CTA = 32 * 256;  // <= 32 n8 blocks x 256 consumer threads x float4 = 128 KB
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

// ---- epilogue staging buffer ------------------------------------------------------------------------------------------
// The epilogue works on the wgmma accumulator fragments where they are: per n8 block a thread owns columns
// (2 (lane % 4), + 1) of rows (lane / 4) and (lane / 4 + 8) of its warp's 16 rows. Global memory wants whole rows, so
// the bf16 results (and, the other way, the residual) of 64 columns cross a 2 KB per-warp buffer: 16 rows x 8 pieces
// of 16 bytes, XOR-swizzled so that the 4-byte fragment accesses and the 16-byte row accesses (8 lanes = one row's
// 128 contiguous bytes) are both conflict-free.
__device__ __forceinline__ uint32_t stage_addr(int row, int piece) {
  return static_cast<uint32_t>(row * 128 + ((piece ^ (row & 7)) << 4));
}
constexpr uint32_t ROW_ABSENT = 0xFFFFFFFFu;  // row table entry of a row outside the problem

// two adjacent values of a per-group / per-row fp32 vector; the scalar form serves unaligned tables and the ragged
// last columns (in0 / in1: the column exists)
__device__ __forceinline__ float2 load_pair(const float* ptr, bool vec, bool in0, bool in1) {
  if (vec) return in0 ? __ldg(reinterpret_cast<const float2*>(ptr)) : make_float2(0.0f, 0.0f);
  return make_float2(in0 ? __ldg(ptr) : 0.0f, in1 ? __ldg(ptr + 1) : 0.0f);
}

// MCAST = the two CTAs of a cluster work on the same n-tile and each loads one half of the B tile with TMA multicast into
// both CTAs' shared memory, so the L2 -> SM traffic per MAC drops from (128+BN)/(128*BN) to (128+BN/2)/(128*BN).
// !MCAST = every CTA loads its whole B tile itself (no cluster); the tile schedule is the same.
template <int BN>
struct IGemmCfg {
  static constexpr int A_BYTES = 128 * 128;  // 128 rows x 64 bf16 (128 B per row, SW128)
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  // alignment slack | barriers | 8 epilogue warps x 2 KB staging | per consumer warpgroup 256 bias + 256 column sums |
  // 8 epilogue warps x 16-row offset tables
  static constexpr int EXTRA_BYTES = 1024 + 256 + 8 * 2048 + 2 * 2 * 1024 + 8 * 128;
};

// Roles (384 threads = three warpgroups): warpgroup 0 = producer (warp 0 issues the TMA loads from one elected lane,
// warps 1-3 idle), warpgroups 1-2 = consumers. The producer warpgroup gives its registers back (setmaxnreg 40) and each
// consumer warpgroup takes 232: 128 fp32 accumulators at BN = 256 plus the epilogue's operands fit without spilling.
// Consumer warpgroup g multiplies rows [64 g, 64 g + 64) of the 128-row tile (wgmma m64 x BN x k16, accumulators in
// registers) and then runs the epilogue of those rows on the fragments in place (see stage_addr).
constexpr int IG_THREADS = 384;
constexpr int IG_PRODUCER_REGS = 40, IG_CONSUMER_REGS = 232;

// Cycle-accounting build (compiled with -DIGEMM_CYCLES, off in the shipped library; tools/igemm_cycles.py builds and
// reads it): per CTA and consumer warpgroup, clock64() totals of the wait on full_bar, the k-loop (those waits included)
// and the epilogue (the stream-K exchange included), plus the pieces and k-blocks run, summed over launches until read
// with b200mix_debug_igemm_cycles.
#ifdef IGEMM_CYCLES
#define IG_CYC(...) __VA_ARGS__
enum { CYC_WAIT = 0, CYC_KLOOP = 1, CYC_EPI = 2, CYC_PIECES = 3, CYC_KBLOCKS = 4, CYC_FIELDS = 5 };
constexpr int CYC_SLOTS = 1024;  // CTA * 2 + consumer warpgroup
__device__ unsigned long long g_igemm_cycles[CYC_SLOTS][CYC_FIELDS];
#else
#define IG_CYC(...)
#endif

// Epilogue families (see the dispatch in the kernel): bias / residual / statistics only, GLU, everything else on the
// row-wise path, and the element-wise path (fp32 output, rows that are not whole 16-byte pieces).
enum { EPI_PLAIN = 0, EPI_GLU = 1, EPI_GENERAL = 2, EPI_DIRECT = 3 };
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
  uint8_t* stage_all = smem + STAGES * Cfg::STAGE_BYTES + 256;
  float* bias_all = reinterpret_cast<float*>(stage_all + 8 * 2048);  // per consumer warpgroup: the tile's BN bias values
  float* colsum_all = bias_all + 2 * 256;                            // same layout: folded-LayerNorm column sums
  uint2* rows_all = reinterpret_cast<uint2*>(colsum_all + 2 * 256);  // per epilogue warp: 16 x (C offset, residual offset)

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

  if (warp < 4) {
    setmaxnreg_dec<IG_PRODUCER_REGS>();
    if (warp == 0) {
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
          // MCAST: the peer CTA's consumers release this stage too (remote arrivals). A plain wait: the TMA writes that
          // follow need no acquire (see mbar_arrive_remote_stage)
          mbar_wait(&empty_bar[stage], phase ^ 1);
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
    }
  } else {
    setmaxnreg_inc<IG_CONSUMER_REGS>();
    // ===== consumers: MMA of 64 rows, then their epilogue =====
    const int cwarp = warp - 4;             // consumer warp 0-7
    const int grp = cwarp >> 2, w = cwarp & 3;
    const int l4 = lane >> 2, lm = lane & 3;
    const int ctid = threadIdx.x - 128;     // consumer thread 0-255
    uint8_t* stage = stage_all + cwarp * 2048;
    float* bias_s = bias_all + grp * 256;
    float* colsum_s = colsum_all + grp * 256;
    uint2* rows_s = rows_all + cwarp * 16;
    const ActCoef ac = act_coef(p.act, p.glu);
    const bool staged_ok = p.vec_ok && !p.out_fp32 && ((p.c_bstride | p.r_bstride) & 7) == 0;
    // this thread's two rows of the tile: position inside the tile box
    int tw[2], th[2], tbb[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = grp * 64 + w * 16 + l4 + 8 * h;
      tw[h] = row % p.TW, th[h] = (row / p.TW) % p.TH, tbb[h] = row / (p.TW * p.TH);
    }
    const uint32_t peer_empty = MCAST ? mapa_smem(&empty_bar[0], cta_rank ^ 1u) : 0u;
    int kstage = 0;
    uint32_t kphase = 0;
    auto release = [&](int s) {  // this warp's wgmma reads of stage s are complete
      if (lane == 0) {
        mbar_arrive(&empty_bar[s]);
        if (MCAST) mbar_arrive_remote_stage(peer_empty + 8u * s);
      }
    };
    IG_CYC(unsigned long long cyc[CYC_FIELDS] = {}; long long cyc_epi0 = -1;)
    for (SegIter seg(p.sk_tiles, total_super, kblocks, cluster_id, num_clusters); seg.next();) {
      // the previous piece's epilogue ends where this piece's k-loop starts (the stream-K tail piece skips the epilogue)
      IG_CYC(const long long cyc_k0 = clock64(); if (cyc_epi0 >= 0) cyc[CYC_EPI] += cyc_k0 - cyc_epi0;
             cyc[CYC_PIECES] += 1, cyc[CYC_KBLOCKS] += seg.kb1 - seg.kb0;)
      float acc[BN / 2];
      {
        int prev = -1;
        for (int kb = seg.kb0; kb < seg.kb1; ++kb) {
          IG_CYC(const long long cyc_w0 = clock64();)
          mbar_wait(&full_bar[kstage], kphase);
          IG_CYC(cyc[CYC_WAIT] += clock64() - cyc_w0;)
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
      IG_CYC(cyc_epi0 = clock64(); cyc[CYC_KLOOP] += cyc_epi0 - cyc_k0;)

      const int st = seg.st;
      const int seg_mode = seg.mode();
      // stream-K pieces: the tail piece (my first) goes to MY workspace slot; the head piece (my last) is completed with
      // the tail piece of the same tile, which the NEXT cluster produced at its very start. A partial travels in the
      // fragment layout (n8 block j of consumer thread t at [j][t]: 512 contiguous bytes per warp and access).
      const int sk_slot = (seg_mode == SEG_TAIL ? cluster_id : cluster_id + 1) * 2 + (int)cta_rank;
      float4* sk_ws = p.sk_ws + static_cast<size_t>(sk_slot) * SK_WS_FLOAT4_PER_CTA + ctid;
      if (seg_mode == SEG_TAIL) {
#pragma unroll
        for (int j = 0; j < BN / 8; ++j)
          __stcg(sk_ws + j * 256, make_float4(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]));
        // all 256 consumer threads' partials are visible device-wide before the flag goes up
        __threadfence();
        named_bar_sync(1, 256);
        if (ctid == 0) st_release_gpu(p.sk_flags + sk_slot, 1u);
        continue;
      }
      if (seg_mode == SEG_HEAD) {
        // the partner's partial was published ~a tile ago; a bounded spin (2^35 cycles, ~18 s: far beyond any time slice
        // the context can lose) turns a scheduling accident (the partner cluster never resident) into an error instead
        // of a hang
        const unsigned int* flag = p.sk_flags + sk_slot;
        const long long t_start = clock64();
        while (ld_acquire_gpu(flag) == 0u) {
          if (clock64() - t_start > (1ll << 35)) __trap();
        }
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const float4 part = __ldcg(sk_ws + j * 256);
          acc[4 * j] += part.x, acc[4 * j + 1] += part.y, acc[4 * j + 2] += part.z, acc[4 * j + 3] += part.w;
        }
        // everybody has read the partial before the flag is lowered for the next launch
        named_bar_sync(1, 256);
        if (ctid == 0) p.sk_flags[sk_slot] = 0u;
      }

      const int mp = st / p.tiles_n, nt = st - mp * p.tiles_n;
      int mt = mp * 2 + (int)cta_rank;
      const bool in_range = mt < tiles_m;
      int par = 0;
      if (p.up) par = mt / p.par_tiles, mt -= par * p.par_tiles;
      const int tx = mt % p.tiles_x;
      const int ty = (mt / p.tiles_x) % p.tiles_y;
      const int tb = mt / (p.tiles_x * p.tiles_y);
      const int n0 = nt * BN;
      // my two rows: rows outside the problem (phantom m-tile of an odd pair, rows past M) still run the warp-collective
      // epilogue; they get group 0 so their row_add / row_gate reads stay inside the [groups, N] tables (nothing is stored)
      bool valid[2];
      long long gm[2], g[2], c_off[2], r_off[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int x = tx * p.TW + tw[h], y = ty * p.TH + th[h], b = tb * p.TB + tbb[h];
        valid[h] = in_range && (x < p.Wo) && (y < p.Ho) && (b < p.Bn);
        gm[h] = p.up ? (static_cast<long long>(b) * (2 * p.Ho) + (2 * y + (par >> 1))) * (2 * p.Wo) + (2 * x + (par & 1))
                     : (static_cast<long long>(b) * p.Ho + y) * p.Wo + x;
        if (p.c_bstride) {  // batched-strided: group == batch
          g[h] = b;
          c_off[h] = static_cast<long long>(b) * p.c_bstride + static_cast<long long>(x) * p.ldc;
          r_off[h] = static_cast<long long>(b) * p.r_bstride + static_cast<long long>(x) * p.ldr;
        } else {
          g[h] = gm[h] / p.rows_per_group;
          c_off[h] = gm[h] * p.ldc;
          r_off[h] = (p.res_row_mod > 0 ? gm[h] % p.res_row_mod : gm[h]) * p.ldr;
        }
        if (!valid[h]) g[h] = 0, gm[h] = 0;
        // offsets in 16-byte units for the row-wise accesses (multiples of 8 elements whenever staged_ok)
        if (lm == 0)
          rows_s[l4 + 8 * h] = make_uint2(valid[h] ? static_cast<uint32_t>(c_off[h] >> 3) : ROW_ABSENT,
                                          static_cast<uint32_t>(r_off[h] >> 3));
      }
      // The tile's bias values go to shared memory once per warpgroup. Folded LayerNorm (consumer side):
      // y = rstd * (acc - mean * colsum[n]) + bias'[n] needs the column sums the same way plus my rows' fixed-point
      // totals. ALL of these loads are issued before any of them is consumed: one L2 round trip per tile, not three.
      constexpr int NI = (BN + 127) / 128;
      const int gt = ctid & 127;
      float bias_r[NI], cs_r[NI];
      longlong2 t_stats[2] = {make_longlong2(0ll, 0ll), make_longlong2(0ll, 0ll)};
#pragma unroll
      for (int i = 0; i < NI; ++i) {
        const int col = n0 + i * 128 + gt;
        bias_r[i] = (p.bias && col < p.N) ? __ldg(p.bias + col) : 0.0f;
        if (LNM == LNM_CONSUMER) cs_r[i] = col < p.N ? __ldg(p.ln_colsum + col) : 0.0f;
      }
      if (LNM == LNM_CONSUMER) {
#pragma unroll
        for (int h = 0; h < 2; ++h) t_stats[h] = __ldg(reinterpret_cast<const longlong2*>(p.ln_stats) + gm[h]);
      }
      named_bar_sync(2 + grp, 128);  // every warp of the group has finished reading the previous tile's values
#pragma unroll
      for (int i = 0; i < NI; ++i) {
        if (i * 128 + gt < BN) {
          bias_s[i * 128 + gt] = bias_r[i];
          if (LNM == LNM_CONSUMER) colsum_s[i * 128 + gt] = cs_r[i];
        }
      }
      named_bar_sync(2 + grp, 128);
      float ln_rstd[2] = {1.0f, 1.0f}, ln_shift[2] = {0.0f, 0.0f};
      if (LNM == LNM_CONSUMER) {  // mean / rstd of my rows from the totals the producing GEMM's epilogues accumulated
        // in fp64: E[x^2] - mean^2 cancels mean^2 / var, so fp32 loses ~2^-24 * mean^2 / var of the variance (2^-8 at
        // |mean| / std = 2^8). A handful of fp64 operations per row and tile, off the MMA critical path.
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const double mean = p.ln_rms ? 0.0 : __ll2double_rn(t_stats[h].x) * p.ln_inv_k;
          const double var = fmax(fma(-mean, mean, __ll2double_rn(t_stats[h].y) * p.ln_inv_k), 0.0);
          ln_rstd[h] = rsqrtf(static_cast<float>(var) + p.ln_eps);
          ln_shift[h] = static_cast<float>(-static_cast<double>(ln_rstd[h]) * mean);
        }
      }
      float st_sum[2] = {0.0f, 0.0f}, st_sq[2] = {0.0f, 0.0f};  // producer side: my rows' sum / sum of squares over my columns
      const int n_end = p.glu ? p.N >> 1 : p.N;  // output columns
      const int srow = lane >> 3, spiece = lane & 7;  // row-wise pattern: row 4 s + srow, 16-byte piece spiece
      // residual pieces of one 64-column group, row-wise (coalesced); fetched one group ahead of their use
      uint4 resv[4];
      auto residual_fetch = [&](int n_abs, int nb) {
#pragma unroll
        for (int s = 0; s < 4; ++s) {
          const uint2 ro = rows_s[4 * s + srow];
          const bool ok = ro.x != ROW_ABSENT && spiece < nb && n_abs + 8 * spiece < p.N;
          resv[s] = ok ? __ldg(reinterpret_cast<const uint4*>(p.residual + n_abs) + ro.y + spiece) : make_uint4(0u, 0u, 0u, 0u);
        }
      };
      __syncwarp();  // rows_s
      constexpr int NG = (BN + 63) / 64;
      // The tile takes the row-wise path when every output row splits into whole 16-byte pieces. The loop over the
      // fragment is fully unrolled, so it is instantiated per epilogue family with the other families' code left out:
      // what a tile executes stays a few thousand instructions, inside the instruction cache.
      const bool tile_staged = staged_ok && p.N % (p.glu ? 16 : 8) == 0;
      auto epilogue = [&](auto mode_c) {
        constexpr int MODE = decltype(mode_c)::value;
        constexpr bool staged = MODE != EPI_DIRECT;
        constexpr bool general = MODE == EPI_GENERAL || MODE == EPI_DIRECT;
        const bool glu_on = MODE == EPI_GLU || (MODE == EPI_DIRECT && p.glu);
        const bool radd_on = MODE != EPI_PLAIN && p.row_add;
        const bool act_on = general && p.act != B200MIX_ACT_NONE;
        const bool gate_on = general && p.row_gate;
        const bool scale_on = general && p.out_scale != 1.0f;
        const bool res_on = MODE != EPI_GLU && p.residual;
        const bool fp32_on = MODE == EPI_DIRECT && p.out_fp32;
        if (staged && res_on) residual_fetch(n0, BN / 8 < 8 ? BN / 8 : 8);
  #pragma unroll
        for (int i = 0; i < NG; ++i) {
          // columns [64 i, 64 i + 64) of the tile: nb n8 blocks of the fragment
          const int nb = BN / 8 - 8 * i < 8 ? BN / 8 - 8 * i : 8;
          const int n_abs = n0 + 64 * i;
          if (n_abs >= p.N) break;
          if (staged && res_on) {
  #pragma unroll
            for (int s = 0; s < 4; ++s) *reinterpret_cast<uint4*>(stage + stage_addr(4 * s + srow, spiece)) = resv[s];
            __syncwarp();
            if (i + 1 < NG) {
              const int nb1 = BN / 8 - 8 * (i + 1) < 8 ? BN / 8 - 8 * (i + 1) : 8;
              if (n_abs + 64 < p.N) residual_fetch(n_abs + 64, nb1);
            }
          }
  #pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            if (jj >= nb) continue;
            const int j = 8 * i + jj;              // n8 block of the accumulator fragment
            const int cl = 64 * i + 8 * jj + 2 * lm;  // my column pair inside the tile
            const int col = n0 + cl;
            const bool in0 = col < p.N, in1 = col + 1 < p.N;
            const float2 bias2 = *reinterpret_cast<const float2*>(bias_s + cl);
            float2 cs2 = make_float2(0.0f, 0.0f);
            if (LNM == LNM_CONSUMER) cs2 = *reinterpret_cast<const float2*>(colsum_s + cl);
            float glu_out[2];
  #pragma unroll
            for (int h = 0; h < 2; ++h) {
              float x = acc[4 * j + 2 * h], y = acc[4 * j + 2 * h + 1];
              if (LNM == LNM_CONSUMER) {
                x = __fmaf_rn(x, ln_rstd[h], __fmul_rn(ln_shift[h], cs2.x));
                y = __fmaf_rn(y, ln_rstd[h], __fmul_rn(ln_shift[h], cs2.y));
              }
              if (p.bias) x += bias2.x, y += bias2.y;
              if (radd_on) {
                const float2 a = load_pair(p.row_add + g[h] * p.ld_row + col, staged, in0, in1);
                x += a.x, y += a.y;
              }
              if (glu_on) {  // value / gate are adjacent columns
                glu_out[h] = x * act_eval(y, ac);
                if (!staged && valid[h] && in1) {
                  if (fp32_on) reinterpret_cast<float*>(p.C)[c_off[h] + (col >> 1)] = glu_out[h];
                  else reinterpret_cast<__nv_bfloat16*>(p.C)[c_off[h] + (col >> 1)] = __float2bfloat16(glu_out[h]);
                }
                continue;
              }
              if (act_on) x = act_eval(x, ac), y = act_eval(y, ac);
              if (gate_on) {
                const float2 a = load_pair(p.row_gate + g[h] * p.ld_row + col, staged, in0, in1);
                x *= a.x, y *= a.y;
              }
              uint32_t* word = reinterpret_cast<uint32_t*>(stage + stage_addr(l4 + 8 * h, jj) + 4 * lm);
              if (res_on) {
                if (staged) {
                  const uint32_t r2 = *word;
                  x += bf16_lo(r2), y += bf16_hi(r2);
                } else if (valid[h]) {
                  const __nv_bfloat16* rs = p.residual + r_off[h] + col;
                  if (in0) x += __bfloat162float(rs[0]);
                  if (in1) y += __bfloat162float(rs[1]);
                }
              }
              if (scale_on) x *= p.out_scale, y *= p.out_scale;
              if (staged) {
                const uint32_t o2 = pack_bf16x2(x, y);
                *word = o2;  // the word this thread read its residual from
                if (LNM == LNM_PRODUCER && in0) {  // row statistics of the ROUNDED values (what the consumer of this tensor reads)
                  const float rx = bf16_lo(o2), ry = bf16_hi(o2);
                  st_sum[h] += rx + ry;
                  st_sq[h] = fmaf(ry, ry, fmaf(rx, rx, st_sq[h]));
                }
              } else if (valid[h]) {
                if (fp32_on) {
                  float* dst = reinterpret_cast<float*>(p.C) + c_off[h] + col;
                  if (in0) dst[0] = x;
                  if (in1) dst[1] = y;
                } else {
                  __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(p.C) + c_off[h] + col;
                  if (in0) dst[0] = __float2bfloat16(x);
                  if (in1) dst[1] = __float2bfloat16(y);
                }
              }
            }
            if (glu_on && staged) {
              // the output column of this pair is cl / 2: lanes lm and lm ^ 1 hold adjacent output columns of both rows.
              // Even lanes collect row l4, odd lanes row l4 + 8, so every lane stores one bf16 pair.
              const float got = __shfl_xor_sync(0xffffffffu, (lm & 1) ? glu_out[0] : glu_out[1], 1);
              const uint32_t o2 = (lm & 1) ? pack_bf16x2(got, glu_out[1]) : pack_bf16x2(glu_out[0], got);
              *reinterpret_cast<uint32_t*>(stage + stage_addr(l4 + 8 * (lm & 1), jj >> 1) + (jj & 1) * 8 + (lm >> 1) * 4) = o2;
            }
          }
          if (staged) {
            // staging buffer -> global memory, a row's contiguous bytes by adjacent lanes
            __syncwarp();
            const int npieces = glu_on ? nb >> 1 : nb;
            const int col_out = glu_on ? n_abs >> 1 : n_abs;
            uint4* cbase = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.C) + col_out) + spiece;
  #pragma unroll
            for (int s = 0; s < 4; ++s) {
              const uint32_t c16 = rows_s[4 * s + srow].x;
              const uint4 o4 = *reinterpret_cast<const uint4*>(stage + stage_addr(4 * s + srow, spiece));
              if (c16 != ROW_ABSENT && spiece < npieces && col_out + 8 * spiece < n_end) cbase[c16] = o4;
            }
            __syncwarp();
          }
        }
      };
      if (!tile_staged) epilogue(std::integral_constant<int, EPI_DIRECT>{});
      else if (p.glu) epilogue(std::integral_constant<int, EPI_GLU>{});
      else if (p.act != B200MIX_ACT_NONE || p.row_add || p.row_gate || p.out_scale != 1.0f)
        epilogue(std::integral_constant<int, EPI_GENERAL>{});
      else epilogue(std::integral_constant<int, EPI_PLAIN>{});
      if (LNM == LNM_PRODUCER) {
        // quad reduction in a fixed order, then 2^24 fixed point: integer adds commute, so the row totals are the same
        // bits whatever order the tiles finish in
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float s = st_sum[h], q = st_sq[h];
          s += __shfl_xor_sync(0xffffffffu, s, 1), q += __shfl_xor_sync(0xffffffffu, q, 1);
          s += __shfl_xor_sync(0xffffffffu, s, 2), q += __shfl_xor_sync(0xffffffffu, q, 2);
          if (lm == 0 && valid[h]) {
            unsigned long long* dst = reinterpret_cast<unsigned long long*>(p.stats_out + 2 * gm[h]);
            atomicAdd(dst, static_cast<unsigned long long>(__float2ll_rn(s * 16777216.0f)));
            atomicAdd(dst + 1, static_cast<unsigned long long>(__float2ll_rn(q * 16777216.0f)));
          }
        }
      }
    }
    IG_CYC(if (cyc_epi0 >= 0) cyc[CYC_EPI] += clock64() - cyc_epi0;
           if ((ctid & 127) == 0 && blockIdx.x * 2 + grp < CYC_SLOTS) {
             for (int f = 0; f < CYC_FIELDS; ++f) atomicAdd(&g_igemm_cycles[blockIdx.x * 2 + grp][f], cyc[f]);
           })
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

void skinny_split(int ctas_n, int K, int kcap, int slots, int* splits_out, int* kpart_out) {
  // K ranges (= cluster size): every candidate that lets a CTA stage its range in one pass is costed as
  // rounds-over-the-machine x (K elements per CTA + a fixed per-CTA cost in the same unit); ranges are at least 512 long.
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
  *splits_out = splits, *kpart_out = kpart;
}

template <int M>
static int launch_skinny(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int rows, int N,
                         int K, const b200mix_epilogue* e, cudaStream_t stream) {
  constexpr int kcap = SK_SMEM_FLOATS / M / 256 * 256;  // K elements one CTA can stage
  const int ctas_n = (N + SK_ROWS_PER_CTA - 1) / SK_ROWS_PER_CTA;
  int splits, kpart;
  skinny_split(ctas_n, K, kcap, (M <= 4 ? 2 : 1) * num_sms(), &splits, &kpart);
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
constexpr int SK_MAX_CLUSTERS = 66;  // 132 SMs
static int sk_min_kblocks() { return g_streamk >= 2 ? 8 : SK_MIN_KBLOCKS; }  // 2 = tests: split shallow reductions too

// Stream-K workspaces: SK_POOL slots per device (17 MB of partial accumulators + 132 flags each: 66 clusters of 2 CTAs), allocated together on
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
  // stage counts: as many (up to 8) as fit next to the epilogue buffers (IGemmCfg::EXTRA_BYTES) in 227 KB
  if (g_gemm_pair) {
    switch (bn) {
      case 256: return launch_igemm<256, 4, true>(tmA, tmB, p, stream);
      case 224: return launch_igemm<224, 4, true>(tmA, tmB, p, stream);
      case 192: return launch_igemm<192, 5, true>(tmA, tmB, p, stream);
      case 160: return launch_igemm<160, 5, true>(tmA, tmB, p, stream);
      case 128: return launch_igemm<128, 6, true>(tmA, tmB, p, stream);
      case 64: return launch_igemm<64, 8, true>(tmA, tmB, p, stream);
      case 32: return launch_igemm<32, 8, true>(tmA, tmB, p, stream);
      default: set_error("unsupported BN %d", bn); return B200MIX_ERR_INVALID;
    }
  }
  switch (bn) {
    case 256: return launch_igemm<256, 4, false>(tmA, tmB, p, stream);
    case 224: return launch_igemm<224, 4, false>(tmA, tmB, p, stream);
    case 192: return launch_igemm<192, 5, false>(tmA, tmB, p, stream);
    case 160: return launch_igemm<160, 5, false>(tmA, tmB, p, stream);
    case 128: return launch_igemm<128, 6, false>(tmA, tmB, p, stream);
    case 64: return launch_igemm<64, 8, false>(tmA, tmB, p, stream);
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
  p.ln_inv_k = 1.0 / 16777216.0 / static_cast<double>(p.Kc);
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
  // the row-wise epilogue reads the per-group vectors as float2 at (group * ld_row + even column)
  if (p.row_add) vec = vec && (reinterpret_cast<uintptr_t>(p.row_add) % 16 == 0) && (p.ld_row % 4 == 0);
  if (p.row_gate) vec = vec && (reinterpret_cast<uintptr_t>(p.row_gate) % 16 == 0) && (p.ld_row % 4 == 0);
  p.vec_ok = vec ? 1 : 0;
  // the statistics are taken in the row-wise bf16 epilogue: whole 16-byte pieces, 16-byte aligned rows
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
#ifdef IGEMM_CYCLES
// Cycle-accounting build only: copies the [1024][5] counters (see g_igemm_cycles) to `out`, then zeroes them if `reset`.
extern "C" int b200mix_debug_igemm_cycles(unsigned long long* out, int reset) {
  if (int rc = ensure_device()) return rc;
  B200_CUDA(cudaDeviceSynchronize());
  if (out) B200_CUDA(cudaMemcpyFromSymbol(out, b200::g_igemm_cycles, sizeof(b200::g_igemm_cycles)));
  if (reset) {
    static const unsigned long long zeros[b200::CYC_SLOTS][b200::CYC_FIELDS] = {};
    B200_CUDA(cudaMemcpyToSymbol(b200::g_igemm_cycles, zeros, sizeof(zeros)));
  }
  return 0;
}
#endif

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
