// Next-token selection for autoregressive generation (PaddleNLP GenerationMixin: greedy_search / sample,
// generation/utils.py:1028-1271, with RepetitionPenaltyLogitsProcessor, TopKProcess and TopPProcess from
// generation/logits_process.py:89-110,293-341). One CTA of 512 threads per row; the row (up to 2^20 fp32 logits) is
// read from global memory once per pass and stays in L2 between passes:
//   greedy:   1 pass   argmax of the penalised logits (lowest id on ties);
//   sampling: 1 pass   max of x = penalised / T;   1 pass   s = sum exp(x - max);   p = exp(x - max) / s
//             3 passes top-k: radix select (11 + 11 + 10 bits) of the k-th largest p on its fp32 bit pattern
//                      (positive floats order like uint32), counts per bucket;
//             3 passes top-p: radix select of the boundary probability v*, histograms of probability MASS per bucket;
//                      (top_p == 1: 1 pass for the kept mass instead)
//             <= 1 pass inverse CDF: block scan of the kept mass in ascending id order, stops at the chosen id.
// Probability masses are summed as 2^-48 fixed-point integers, floor(p * 2^48), which is exact for p >= 2^-25: the
// kept set and the drawn token do not depend on the order of the (atomic) additions.
// Top-p order: descending probability, lower token id first among equal probabilities. A token is dropped when the
// mass ranked above it exceeds top_p, so the first token is always kept.
// Draw: Philox4x32-10 (Salmon et al., SC'11), key = seed, counter = (step, row, 0, 0); u = (x0 >> 8) * 2^-24, the token
// is the first kept id whose inclusive prefix mass exceeds u * kept mass.
// Bookkeeping (generation/utils.py:1239-1259): a finished row emits pad_id; finished |= token in eos_ids; the token
// goes to out[b, step] and next_ids[b], and its bit is set in the row's presence bitmap. The last CTA to arrive sets
// the all-finished flag (and the step at which it happened) and advances the step, so a CUDA-graph replay draws new
// numbers.
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include <float.h>

#include "common.cuh"
#include "philox.cuh"
#include "ptx.cuh"

namespace b200 {
namespace {

constexpr int SP_THREADS = 512;
constexpr int SP_BUCKETS = 2048;  // radix digit of 11 bits
constexpr int SP_BPT = SP_BUCKETS / SP_THREADS;  // buckets per thread in the bucket scans
constexpr int SP_ITEMS = 8;       // ids per thread per inverse-CDF chunk
constexpr float SP_FX = 281474976710656.0f;  // 2^48

struct SampleArgs {
  const float* logits;
  long long ld;
  int V, words;
  uint32_t* presence;
  int32_t* finished;
  unsigned long long* state;  // [0] step, [1] arrivals, [2] all finished, [3] step at which the last row finished
  long long* out;
  long long ld_out, max_new;
  long long* next_ids;
  const long long* eos;
  int n_eos;
  long long pad;
  int do_sample, top_k;
  float temperature, top_p, penalty;
  unsigned long long seed;
};

struct Row {
  const float* x;
  const uint32_t* bits;
  float penalty, temperature, max, sum;
  uint32_t topk_bits;

  // RepetitionPenaltyLogitsProcessor: l < 0 ? l * p : l / p on every id present so far
  __device__ __forceinline__ float logit(int i) const {
    float l = x[i];
    if (penalty != 1.0f && ((bits[i >> 5] >> (i & 31)) & 1u)) l = l < 0.0f ? l * penalty : l / penalty;
    return l;
  }
  __device__ __forceinline__ float scaled(int i) const { return logit(i) / temperature; }
  __device__ __forceinline__ float prob(int i) const { return expf(scaled(i) - max) / sum; }
  // probability after top-k (0 below the k-th largest), as its bit pattern
  __device__ __forceinline__ uint32_t q(int i) const {
    const uint32_t b = __float_as_uint(prob(i));
    return b >= topk_bits ? b : 0u;
  }
};

__device__ __forceinline__ unsigned long long fx(uint32_t pbits) {
  return __float2ull_rz(__uint_as_float(pbits) * SP_FX);
}

using BlockScanU64 = cub::BlockScan<unsigned long long, SP_THREADS>;
using BlockRedF = cub::BlockReduce<float, SP_THREADS>;
using BlockRedU64 = cub::BlockReduce<unsigned long long, SP_THREADS>;

struct Smem {
  uint32_t cnt[SP_BUCKETS];
  unsigned long long mass[SP_BUCKETS];
  union {
    typename BlockScanU64::TempStorage scan;
    typename BlockRedF::TempStorage redf;
    typename BlockRedU64::TempStorage redu;
  } tmp;
  float f;
  int sel;
  int found;
  unsigned long long u64a, u64b;
  int last;
};

__device__ __forceinline__ int digit_shift(int level) { return level == 0 ? 21 : (level == 1 ? 10 : 0); }
__device__ __forceinline__ int digit_buckets(int level) { return level == 2 ? 1024 : 2048; }

// Bit pattern of the k-th largest probability (1 <= k < V).
__device__ uint32_t select_kth(const Row& row, int V, int k, Smem& sm) {
  uint32_t prefix = 0, mask = 0;
  int kr = k;
  for (int level = 0; level < 3; ++level) {
    const int shift = digit_shift(level), nb = digit_buckets(level);
    for (int j = threadIdx.x; j < SP_BUCKETS; j += SP_THREADS) sm.cnt[j] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < V; i += SP_THREADS) {
      const uint32_t v = __float_as_uint(row.prob(i));
      const bool in = (v & mask) == prefix;
      const uint32_t d = in ? (v >> shift) & (nb - 1) : 0xFFFFFFFFu;
      // most ids share a handful of top-level buckets: one atomic per bucket per warp
      const unsigned peers = __match_any_sync(__activemask(), d);
      if (in && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&sm.cnt[d], (uint32_t)__popc(peers));
    }
    __syncthreads();
    // thread t owns buckets nb-1-SP_BPT*t down to nb-SP_BPT*(t+1) (descending order)
    const int dtop = nb - 1 - SP_BPT * (int)threadIdx.x;
    unsigned long long tot = 0;
#pragma unroll
    for (int j = 0; j < SP_BPT; ++j) tot += dtop - j >= 0 ? sm.cnt[dtop - j] : 0u;
    unsigned long long above;
    BlockScanU64(sm.tmp.scan).ExclusiveSum(tot, above);
#pragma unroll
    for (int j = 0; j < SP_BPT; ++j) {
      const unsigned long long c = dtop - j >= 0 ? sm.cnt[dtop - j] : 0u;
      if (above < (unsigned long long)kr && above + c >= (unsigned long long)kr) {
        sm.sel = dtop - j;
        sm.u64a = above;
      }
      above += c;
    }
    __syncthreads();
    prefix |= (uint32_t)sm.sel << shift;
    mask |= (uint32_t)(nb - 1) << shift;
    kr -= (int)sm.u64a;
    __syncthreads();
  }
  return prefix;
}

// Top-p boundary: the smallest present value v* whose mass above, M(> v*), is <= tp (fixed point). Returns v* and
// sets *m_above = M(> v*), *n_eq = number of ids with q == v*.
__device__ uint32_t select_top_p(const Row& row, int V, unsigned long long tp, Smem& sm, unsigned long long* m_above,
                                 unsigned long long* n_eq) {
  uint32_t prefix = 0, mask = 0;
  unsigned long long M = 0, neq = 0;
  for (int level = 0; level < 3; ++level) {
    const int shift = digit_shift(level), nb = digit_buckets(level);
    for (int j = threadIdx.x; j < SP_BUCKETS; j += SP_THREADS) {
      sm.cnt[j] = 0;
      sm.mass[j] = 0;
    }
    if (threadIdx.x == 0) sm.sel = -1;
    __syncthreads();
    for (int i = threadIdx.x; i < V; i += SP_THREADS) {
      const uint32_t v = row.q(i);
      // ids removed by top-k (q = 0) carry no mass; leaving them out only moves v* from 0 to the smallest kept value
      if (v != 0u && (v & mask) == prefix) {
        const int d = (v >> shift) & (nb - 1);
        atomicAdd(&sm.cnt[d], 1u);
        atomicAdd(&sm.mass[d], fx(v));
      }
    }
    __syncthreads();
    const int dtop = nb - 1 - SP_BPT * (int)threadIdx.x;
    unsigned long long tot = 0;
#pragma unroll
    for (int j = 0; j < SP_BPT; ++j) tot += dtop - j >= 0 ? sm.mass[dtop - j] : 0ull;
    unsigned long long above;
    BlockScanU64(sm.tmp.scan).ExclusiveSum(tot, above);
    // the condition M + mass(> d) <= tp holds for every bucket above some point: take the lowest non-empty one
    int cand = -1;
    unsigned long long cand_above = 0;
#pragma unroll
    for (int j = 0; j < SP_BPT; ++j) {
      const int d = dtop - j;
      if (d >= 0 && sm.cnt[d] && M + above <= tp) {
        cand = d;
        cand_above = above;
      }
      if (d >= 0) above += sm.mass[d];
    }
    if (cand >= 0) atomicMin(reinterpret_cast<unsigned int*>(&sm.sel), (unsigned int)cand);
    __syncthreads();
    if (cand >= 0 && cand == sm.sel) {
      sm.u64a = cand_above;
      sm.u64b = sm.cnt[cand];
    }
    __syncthreads();
    prefix |= (uint32_t)sm.sel << shift;
    mask |= (uint32_t)(nb - 1) << shift;
    M += sm.u64a;
    neq = sm.u64b;
    __syncthreads();
  }
  *m_above = M;
  *n_eq = neq;
  return prefix;
}

__global__ void __launch_bounds__(SP_THREADS, 1) sample_tokens_kernel(SampleArgs a) {
  __shared__ Smem sm;
  const int b = blockIdx.x, tid = threadIdx.x;
  pdl_wait();
  pdl_launch_dependents();
  const unsigned long long step = a.state[0];
  const bool was_finished = a.finished[b] != 0;
  Row row;
  row.x = a.logits + (long long)b * a.ld;
  row.bits = a.presence + (long long)b * a.words;
  row.penalty = a.penalty;
  row.temperature = a.temperature;
  row.topk_bits = 0;
  int token = 0;

  if (was_finished) {
    // the row emits pad_id whatever its logits are
  } else if (!a.do_sample) {
    float best = -INFINITY;
    int arg = INT_MAX;
    for (int i = tid; i < a.V; i += SP_THREADS) {
      const float l = row.logit(i);
      if (l > best || (l == best && i < arg)) best = l, arg = i;
    }
    const float m = BlockRedF(sm.tmp.redf).Reduce(best, cub::Max());
    if (tid == 0) {
      sm.f = m;
      sm.found = INT_MAX;
    }
    __syncthreads();
    if (best == sm.f) atomicMin(&sm.found, arg);
    __syncthreads();
    token = sm.found == INT_MAX ? 0 : sm.found;  // all-NaN row: id 0
  } else {
    // ---- softmax(x / T) ------------------------------------------------------------------------------------------
    float m = -INFINITY;
    for (int i = tid; i < a.V; i += SP_THREADS) m = fmaxf(m, row.scaled(i));
    m = BlockRedF(sm.tmp.redf).Reduce(m, cub::Max());
    if (tid == 0) sm.f = m;
    __syncthreads();
    row.max = sm.f;
    __syncthreads();
    float s = 0.0f;
    for (int i = tid; i < a.V; i += SP_THREADS) s += expf(row.scaled(i) - row.max);
    s = BlockRedF(sm.tmp.redf).Sum(s);
    if (tid == 0) sm.f = s;
    __syncthreads();
    row.sum = sm.f;
    __syncthreads();
    // ---- TopKProcess: keep p >= k-th largest p (ties at the k-th value kept) ---------------------------------------
    if (a.top_k > 0 && a.top_k < a.V) row.topk_bits = select_kth(row, a.V, a.top_k, sm);
    // ---- TopPProcess on the top-k output (not renormalised) -------------------------------------------------------
    uint32_t vstar = 0;
    unsigned long long kept, keep_eq = ~0ull, n_eq = 0;
    if (a.top_p < 1.0f) {
      const unsigned long long tp = __float2ull_rz(a.top_p * SP_FX);
      unsigned long long m_above;
      vstar = select_top_p(row, a.V, tp, sm, &m_above, &n_eq);
      const unsigned long long fv = fx(vstar);
      keep_eq = fv == 0 ? n_eq : min(n_eq, (tp - m_above) / fv + 1);
      kept = m_above + keep_eq * fv;
    } else {
      unsigned long long k = 0;
      for (int i = tid; i < a.V; i += SP_THREADS) k += fx(row.q(i));
      k = BlockRedU64(sm.tmp.redu).Sum(k);
      if (tid == 0) sm.u64a = k;
      __syncthreads();
      kept = sm.u64a;
      __syncthreads();
    }
    const bool rank_ties = keep_eq < n_eq;  // some ids of value v* are dropped: their order by id matters
    // ---- multinomial: inverse CDF over the kept, unnormalised mass in ascending id order --------------------------
    const uint4 r = philox4x32_10(make_uint4((uint32_t)step, (uint32_t)b, 0u, 0u),
                                  make_uint2((uint32_t)a.seed, (uint32_t)(a.seed >> 32)));
    const double target = (double)(r.x >> 8) * (1.0 / 16777216.0) * (double)kept;
    unsigned long long carry = 0, eq_carry = 0;
    if (tid == 0) sm.found = INT_MAX;
    __syncthreads();
    for (int base = 0; base < a.V; base += SP_THREADS * SP_ITEMS) {
      const int i0 = base + tid * SP_ITEMS;
      uint32_t v[SP_ITEMS];
#pragma unroll
      for (int j = 0; j < SP_ITEMS; ++j) v[j] = i0 + j < a.V ? row.q(i0 + j) : 0u;
      unsigned long long eq_before = 0;
      if (rank_ties) {
        unsigned long long e = 0, agg;
#pragma unroll
        for (int j = 0; j < SP_ITEMS; ++j) e += v[j] == vstar;
        BlockScanU64(sm.tmp.scan).ExclusiveSum(e, eq_before, agg);
        eq_before += eq_carry;
        eq_carry += agg;
        __syncthreads();
      }
      unsigned long long tot = 0;
#pragma unroll
      for (int j = 0; j < SP_ITEMS; ++j) {
        bool keep = v[j] > vstar;
        if (v[j] == vstar) keep = eq_before++ < keep_eq;
        if (!keep) v[j] = 0u;
        tot += fx(v[j]);
      }
      unsigned long long before, agg;
      BlockScanU64(sm.tmp.scan).ExclusiveSum(tot, before, agg);
      if ((double)(carry + agg) > target) {
        unsigned long long run = carry + before;
#pragma unroll
        for (int j = 0; j < SP_ITEMS; ++j) {
          run += fx(v[j]);
          if ((double)run > target) {
            atomicMin(&sm.found, i0 + j);
            break;
          }
        }
        __syncthreads();
        break;
      }
      carry += agg;
      __syncthreads();
    }
    __syncthreads();
    token = sm.found == INT_MAX ? 0 : sm.found;
  }

  // ---- bookkeeping ---------------------------------------------------------------------------------------------
  if (tid == 0) {
    const long long tok = was_finished ? a.pad : (long long)token;
    if ((long long)step < a.max_new) a.out[(long long)b * a.ld_out + (long long)step] = tok;
    a.next_ids[b] = tok;
    a.presence[(long long)b * a.words + (tok >> 5)] |= 1u << (tok & 31);
    if (!was_finished) {
      bool eos = false;
      for (int e = 0; e < a.n_eos; ++e) eos |= a.eos[e] == tok;
      if (eos) a.finished[b] = 1;
    }
    __threadfence();
    sm.last = atomicAdd(&a.state[1], 1ull) == (unsigned long long)gridDim.x - 1;
  }
  __syncthreads();
  if (!sm.last) return;
  // last CTA: every other CTA has read `step` and published its row
  __threadfence();
  int all = a.n_eos > 0;
  for (int r = tid; r < (int)gridDim.x; r += SP_THREADS)
    if (!*reinterpret_cast<volatile int32_t*>(&a.finished[r])) all = 0;
  all = __syncthreads_and(all);
  if (tid == 0) {
    if (all && a.state[2] == 0) {
      a.state[2] = 1;
      a.state[3] = step;
    }
    a.state[1] = 0;
    a.state[0] = step + 1;
  }
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int b200mix_sample_tokens(const float* logits, int64_t ld, int64_t B, int64_t V, uint32_t* presence,
                                     int32_t* finished, uint64_t* state, int64_t* out, int64_t ld_out, int64_t max_new,
                                     int64_t* next_ids, const int64_t* eos_ids, int32_t n_eos, int64_t pad_id,
                                     int32_t do_sample, float temperature, int32_t top_k, float top_p, float penalty,
                                     uint64_t seed, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(logits && presence && finished && state && out && next_ids, "sample_tokens: null pointer");
  B200_CHECK_ARG(B >= 1 && B < (1ll << 31), "sample_tokens: B=%lld out of range", (long long)B);
  B200_CHECK_ARG(V >= 1 && V <= (1ll << 20), "sample_tokens: V=%lld must be in [1, 2^20]", (long long)V);
  B200_CHECK_ARG(ld >= V, "sample_tokens: row stride %lld < V=%lld", (long long)ld, (long long)V);
  B200_CHECK_ARG(max_new >= 1 && ld_out >= max_new, "sample_tokens: bad output shape (max_new=%lld, ld_out=%lld)",
                 (long long)max_new, (long long)ld_out);
  B200_CHECK_ARG(reinterpret_cast<uintptr_t>(logits) % 4 == 0 && reinterpret_cast<uintptr_t>(presence) % 4 == 0 &&
                     reinterpret_cast<uintptr_t>(finished) % 4 == 0 && reinterpret_cast<uintptr_t>(state) % 8 == 0 &&
                     reinterpret_cast<uintptr_t>(out) % 8 == 0 && reinterpret_cast<uintptr_t>(next_ids) % 8 == 0 &&
                     reinterpret_cast<uintptr_t>(eos_ids) % 8 == 0,
                 "sample_tokens: misaligned buffer");
  B200_CHECK_ARG(n_eos >= 0 && n_eos <= 1024 && (n_eos == 0 || eos_ids), "sample_tokens: bad eos list (n_eos=%d)",
                 (int)n_eos);
  B200_CHECK_ARG(n_eos == 0 || (pad_id >= 0 && pad_id < V), "sample_tokens: pad_id=%lld must be in [0, V)",
                 (long long)pad_id);
  B200_CHECK_ARG(temperature > 0.0f && temperature <= FLT_MAX, "sample_tokens: temperature must be > 0 (got %g)",
                 (double)temperature);
  B200_CHECK_ARG(top_p > 0.0f && top_p <= 1.0f, "sample_tokens: top_p must be in (0, 1] (got %g)", (double)top_p);
  B200_CHECK_ARG(top_k >= 0, "sample_tokens: top_k must be >= 0 (got %d)", (int)top_k);
  B200_CHECK_ARG(penalty > 0.0f && penalty <= FLT_MAX, "sample_tokens: repetition penalty must be > 0 (got %g)",
                 (double)penalty);
  SampleArgs a;
  a.logits = logits;
  a.ld = ld;
  a.V = (int)V;
  a.words = (int)((V + 31) / 32);
  a.presence = presence;
  a.finished = finished;
  a.state = reinterpret_cast<unsigned long long*>(state);
  a.out = reinterpret_cast<long long*>(out);
  a.ld_out = ld_out;
  a.max_new = max_new;
  a.next_ids = reinterpret_cast<long long*>(next_ids);
  a.eos = reinterpret_cast<const long long*>(eos_ids);
  a.n_eos = n_eos;
  a.pad = pad_id;
  a.do_sample = do_sample != 0;
  a.top_k = top_k;
  a.temperature = temperature;
  a.top_p = top_p;
  a.penalty = penalty;
  a.seed = seed;
  B200_CUDA(launch_pdl(sample_tokens_kernel, dim3((unsigned)B), dim3(SP_THREADS), 0,
                       reinterpret_cast<cudaStream_t>(stream), 1, a));
  return 0;
}
