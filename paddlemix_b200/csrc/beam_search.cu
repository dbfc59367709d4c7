// Beam search for autoregressive generation (PaddleNLP GenerationMixin.beam_search, generation/utils.py:1484-1649, with
// BeamHypotheses / BeamSearchScorer :98-316 and reorder_cache :1480-1482), entirely on the device so that a decode loop
// can run as CUDA-graph replays.
//
// b200mix_beam_search_step: three launches chained with PDL, over B items of nb beams (rows b*nb .. b*nb + nb - 1):
//   stats:  one CTA per 4096-logit chunk of each row: chunk max m_c and sum_c exp(x - m_c);
//   topk:   one CTA per chunk again (the row now comes from L2): the row's max M = max m_c and sum = sum_c s_c *
//           exp(m_c - M), merged by every CTA in chunk order (so every CTA of a row holds the same two numbers), the
//           exact fp32 step scores log(exp(x - M) / sum) -> repetition penalty (score < 0 ? score * p : score / p on the
//           ids present in the row) -> + running beam score, and the chunk's top 2*nb by (score desc, flat id asc),
//           flat id = beam * V + token;
//   merge:  one CTA per item: the item's top 2*nb candidates (diversity_rate > 0: each row's top 2*nb, minus
//           rank * diversity_rate, top 2*nb of those in (beam, rank) row-major order), then BeamSearchScorer.process
//           sequentially in fp64 and the bookkeeping; the last CTA to arrive sets the all-done flag and advances the step.
// Selection keeps one sorted top-32 list per warp in registers (one entry per lane): a batch of 32 candidates is skipped
// unless one of them beats the current 2*nb-th entry, otherwise bitonic-sorted by shuffles and merged in.
// Candidates are 64-bit keys (order-preserving score bits << 32 | ~flat id), so "larger key" is "higher score, then
// lower id": ties go to the lower flat index.
//
// b200mix_kv_reorder: the cache rows of the generated region [S, S + t) move from parent beam to child, every layer in
// one launch. A CTA owns (position block, item, layer); it stages the nb rows of each position in shared memory and
// writes back the rows whose parent is not themselves, so duplicated and dropped parents need no scratch cache.
#include <cub/block/block_reduce.cuh>
#include <float.h>

#include "common.cuh"
#include "ptx.cuh"

namespace b200 {
namespace {

constexpr int BS_THREADS = 256;
constexpr int BS_WARPS = BS_THREADS / 32;
constexpr int BS_ITEMS = 16;
constexpr int BS_CHUNK = BS_THREADS * BS_ITEMS;
constexpr int BS_MAX_BEAMS = 16;
constexpr int RO_THREADS = 256;
constexpr int RO_SMEM = 32 * 1024;  // staged rows per reorder CTA: positions_per_cta * nb * row bytes

struct StepArgs {
  const float* logits;
  long long ld;
  int B, nb, V, words, n_chunks;
  b200mix_beam_state st;
  unsigned long long* keys;  // [B*nb, n_chunks, 2*nb]
  float2* stats;             // [B*nb, n_chunks]
  long long max_new, eos, pad;
  float penalty, diversity;
  double length_penalty;
  int early_stopping;
};

__device__ __forceinline__ unsigned long long make_key(float s, uint32_t idx) {
  const uint32_t u = __float_as_uint(s);
  uint32_t o = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  if (s != s) o = 0;  // NaN ranks below every number
  return ((unsigned long long)o << 32) | (uint32_t)~idx;
}
__device__ __forceinline__ float key_score(unsigned long long k) {
  const uint32_t o = (uint32_t)(k >> 32);
  return __uint_as_float((o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o);
}
__device__ __forceinline__ uint32_t key_index(unsigned long long k) { return ~(uint32_t)k; }

__device__ __forceinline__ bool step_active(const StepArgs& a, unsigned long long* step) {
  *step = a.st.state[0];
  return *step < (unsigned long long)a.max_new && a.st.state[2] == 0;
}

// `best` holds a descending list across the warp's lanes; merges the descending list `v` into it (top 32 kept).
__device__ __forceinline__ unsigned long long warp_merge(unsigned long long best, unsigned long long v) {
  const int lane = threadIdx.x & 31;
  unsigned long long c = max(best, __shfl_sync(0xFFFFFFFFu, v, 31 - lane));  // bitonic: top 32 of the union
#pragma unroll
  for (int stride = 16; stride > 0; stride >>= 1) {
    const unsigned long long o = __shfl_xor_sync(0xFFFFFFFFu, c, stride);
    c = (lane & stride) == 0 ? max(c, o) : min(c, o);
  }
  return c;
}

__device__ __forceinline__ unsigned long long warp_sort_desc(unsigned long long v) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int size = 2; size <= 32; size <<= 1) {
#pragma unroll
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      const unsigned long long o = __shfl_xor_sync(0xFFFFFFFFu, v, stride);
      const bool desc = (lane & size) == 0, lower = (lane & stride) == 0;
      v = (lower == desc) ? max(v, o) : min(v, o);
    }
  }
  return v;
}

// Top K (<= 32) keys of key_of(0 .. n-1) over the whole CTA, written descending to out[0 .. K); missing entries are 0.
template <class F>
__device__ void block_topk(F key_of, int n, int K, unsigned long long (*lists)[32], unsigned long long* out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long best = 0;
  for (int base = warp * 32; base < n; base += BS_THREADS) {
    const unsigned long long k = base + lane < n ? key_of(base + lane) : 0ull;
    const unsigned long long kth = __shfl_sync(0xFFFFFFFFu, best, K - 1);
    if (!__any_sync(0xFFFFFFFFu, k > kth)) continue;
    best = warp_merge(best, warp_sort_desc(k));
  }
  lists[warp][lane] = best;
  __syncthreads();
  if (warp == 0) {
    for (int w = 1; w < BS_WARPS; ++w) best = warp_merge(best, lists[w][lane]);
    out[lane] = best;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(BS_THREADS) beam_stats_kernel(StepArgs a) {
  using Red = cub::BlockReduce<float, BS_THREADS>;
  __shared__ typename Red::TempStorage red;
  __shared__ float m_sh;
  pdl_wait();
  pdl_launch_dependents();
  unsigned long long step;
  if (!step_active(a, &step)) return;
  const int row = blockIdx.y, c = blockIdx.x, tid = threadIdx.x;
  const float* x = a.logits + (long long)row * a.ld + (long long)c * BS_CHUNK;
  const int n = min(BS_CHUNK, a.V - c * BS_CHUNK);
  float v[BS_ITEMS];
  float m = -INFINITY;
#pragma unroll
  for (int j = 0; j < BS_ITEMS; ++j) {
    const int i = j * BS_THREADS + tid;
    v[j] = i < n ? x[i] : -INFINITY;
    m = fmaxf(m, v[j]);
  }
  m = Red(red).Reduce(m, cub::Max());
  if (tid == 0) m_sh = m;
  __syncthreads();
  m = m_sh;
  float s = 0.0f;
  if (m != -INFINITY) {
#pragma unroll
    for (int j = 0; j < BS_ITEMS; ++j) s += expf(v[j] - m);
  }
  __syncthreads();
  s = Red(red).Sum(s);
  if (tid == 0) a.stats[(long long)row * a.n_chunks + c] = make_float2(m, s);
}

__global__ void __launch_bounds__(BS_THREADS) beam_topk_kernel(StepArgs a) {
  __shared__ unsigned long long lists[BS_WARPS][32];
  __shared__ unsigned long long top[32];
  __shared__ float row_max, row_sum;
  pdl_wait();
  pdl_launch_dependents();
  unsigned long long step;
  if (!step_active(a, &step)) return;
  const int row = blockIdx.y, c = blockIdx.x, tid = threadIdx.x, K = 2 * a.nb;
  if (tid == 0) {
    const float2* st = a.stats + (long long)row * a.n_chunks;
    float M = -INFINITY;
    for (int j = 0; j < a.n_chunks; ++j) M = fmaxf(M, st[j].x);
    float s = 0.0f;
    for (int j = 0; j < a.n_chunks; ++j)
      if (st[j].x != -INFINITY) s = __fadd_rn(s, __fmul_rn(st[j].y, expf(st[j].x - M)));
    row_max = M;
    row_sum = s;
  }
  __syncthreads();
  const float M = row_max, sum = row_sum, bscore = a.st.beam_scores[row], pen = a.penalty;
  const float* x = a.logits + (long long)row * a.ld;
  const uint32_t* bits =
      a.st.presence ? a.st.presence + ((long long)(step & 1) * a.B * a.nb + row) * a.words : nullptr;
  const int i0 = c * BS_CHUNK, n = min(BS_CHUNK, a.V - i0);
  const uint32_t flat0 = (uint32_t)(row % a.nb) * (uint32_t)a.V + (uint32_t)i0;
  auto key_of = [&](int j) {
    const int i = i0 + j;
    float s = logf(expf(x[i] - M) / sum);
    // every product / sum rounded on its own (no FMA contraction), as the reference and the oracle round them: inputs
    // that tie there tie here, and the tie goes to the lower flat index
    if (bits && ((bits[i >> 5] >> (i & 31)) & 1u)) s = s < 0.0f ? __fmul_rn(s, pen) : __fdiv_rn(s, pen);
    return make_key(__fadd_rn(s, bscore), flat0 + (uint32_t)j);
  };
  block_topk(key_of, n, K, lists, top);
  if (tid < K) a.keys[((long long)row * a.n_chunks + c) * K + tid] = top[tid];
}

struct MergeSmem {
  unsigned long long lists[BS_WARPS][32];
  unsigned long long top[32];
  unsigned long long sib[BS_MAX_BEAMS * 2 * BS_MAX_BEAMS];  // diversity: each row's top 2*nb
  float cand_score[32];
  int cand_token[32], cand_beam[32];
  int slot_token[BS_MAX_BEAMS], slot_parent[BS_MAX_BEAMS];
  double hyp_score[BS_MAX_BEAMS + 1];
  int hyp_step[BS_MAX_BEAMS + 1], hyp_slot[BS_MAX_BEAMS + 1];
  int was_done, last;
};

// BeamHypotheses.add (utils.py:115-127) on the item's store, in insertion order.
__device__ void hyp_add(MergeSmem& sm, int& count, double& worst, int nb, double score, int step, int slot) {
  if (count < nb || score > worst) {
    sm.hyp_score[count] = score;
    sm.hyp_step[count] = step;
    sm.hyp_slot[count] = slot;
    ++count;
    if (count > nb) {
      // sorted((s, idx)): delete the lowest, the new worst is the second lowest
      int lo = 0;
      for (int i = 1; i < count; ++i)
        if (sm.hyp_score[i] < sm.hyp_score[lo]) lo = i;
      int second = lo == 0 ? 1 : 0;
      for (int i = 0; i < count; ++i)
        if (i != lo && sm.hyp_score[i] < sm.hyp_score[second]) second = i;
      worst = sm.hyp_score[second];
      for (int i = lo; i + 1 < count; ++i) {
        sm.hyp_score[i] = sm.hyp_score[i + 1];
        sm.hyp_step[i] = sm.hyp_step[i + 1];
        sm.hyp_slot[i] = sm.hyp_slot[i + 1];
      }
      --count;
    } else {
      worst = fmin(score, worst);
    }
  }
}

__global__ void __launch_bounds__(BS_THREADS) beam_merge_kernel(StepArgs a) {
  __shared__ MergeSmem sm;
  pdl_wait();
  pdl_launch_dependents();
  unsigned long long step;
  if (!step_active(a, &step)) {
    if (blockIdx.x == 0 && threadIdx.x == 0) a.st.state[3] = 0;  // nothing for the reorder to move
    return;
  }
  const int b = blockIdx.x, tid = threadIdx.x, nb = a.nb, K = 2 * nb, rows = a.B * nb;
  const b200mix_beam_state& st = a.st;
  const int t = (int)step;
  if (tid == 0) sm.was_done = st.done[b] != 0;
  __syncthreads();
  if (sm.was_done) {
    // BeamSearchScorer.process :208-219: pad, score 0, index 0; the item's cache / presence rows are left alone
    if (tid < nb) {
      const int r = b * nb + tid;
      st.next_ids[r] = a.pad;
      st.beam_scores[r] = 0.0f;
      st.tokens[(long long)t * rows + r] = a.pad;
      st.parents[(long long)t * rows + r] = 0;
    }
  } else {
    const unsigned long long* keys = a.keys + (long long)b * nb * a.n_chunks * K;
    if (a.diversity == 0.0f) {
      block_topk([&](int i) { return keys[i]; }, nb * a.n_chunks * K, K, sm.lists, sm.top);
      if (tid < K) {
        const uint32_t flat = key_index(sm.top[tid]);
        sm.cand_score[tid] = key_score(sm.top[tid]);
        sm.cand_token[tid] = (int)(flat % (uint32_t)a.V);
        sm.cand_beam[tid] = (int)(flat / (uint32_t)a.V);
      }
    } else {
      const int per_row = a.n_chunks * K;
      for (int j = 0; j < nb; ++j) {
        const unsigned long long* rk = keys + (long long)j * per_row;
        block_topk([&](int i) { return rk[i]; }, per_row, K, sm.lists, sm.top);
        if (tid < K) sm.sib[j * K + tid] = sm.top[tid];
        __syncthreads();
      }
      // diversified score = score - rank * diversity_rate (rank 1 .. 2*nb), position p = beam * 2*nb + rank - 1
      const float rate = a.diversity;
      block_topk(
          [&](int p) {
            const float d = __fsub_rn(key_score(sm.sib[p]), __fmul_rn((float)(p % K + 1), rate));  // two roundings
            return make_key(d, (uint32_t)p);
          },
          nb * K, K, sm.lists, sm.top);
      if (tid < K) {
        const int p = (int)key_index(sm.top[tid]);
        sm.cand_score[tid] = key_score(sm.sib[p]);
        sm.cand_token[tid] = (int)(key_index(sm.sib[p]) % (uint32_t)a.V);
        sm.cand_beam[tid] = p / K;
      }
    }
    __syncthreads();
    if (tid == 0) {
      // BeamSearchScorer.process :221-256 in fp64
      int count = st.hyp_count[b];
      double worst = st.hyp_worst[b];
      for (int i = 0; i < count; ++i) {
        sm.hyp_score[i] = st.hyp_score[b * nb + i];
        sm.hyp_step[i] = st.hyp_step[b * nb + i];
        sm.hyp_slot[i] = st.hyp_slot[b * nb + i];
      }
      const double len_pen = pow((double)(t + 5) / 6.0, a.length_penalty);
      float best = -INFINITY;
      for (int r = 0; r < K; ++r) best = fmaxf(best, sm.cand_score[r]);
      int filled = 0;
      for (int r = 0; r < K && filled < nb; ++r) {
        const int tok = sm.cand_token[r];
        if (a.eos >= 0 && tok == a.eos) {
          if (r >= nb) continue;
          hyp_add(sm, count, worst, nb, (double)sm.cand_score[r] / len_pen, t, sm.cand_beam[r]);
        } else {
          const int row = b * nb + filled;
          st.next_ids[row] = tok;
          st.beam_scores[row] = sm.cand_score[r];
          st.tokens[(long long)t * rows + row] = tok;
          st.parents[(long long)t * rows + row] = sm.cand_beam[r];
          sm.slot_token[filled] = tok;
          sm.slot_parent[filled] = sm.cand_beam[r];
          ++filled;
        }
      }
      // BeamHypotheses.is_done :129-142
      bool done = false;
      if (count >= nb) done = a.early_stopping ? true : worst >= (double)best / len_pen;
      for (int i = 0; i < count; ++i) {
        st.hyp_score[b * nb + i] = sm.hyp_score[i];
        st.hyp_step[b * nb + i] = sm.hyp_step[i];
        st.hyp_slot[b * nb + i] = sm.hyp_slot[i];
      }
      st.hyp_count[b] = count;
      st.hyp_worst[b] = worst;
      if (done) st.done[b] = 1;
    }
    __syncthreads();
    if (st.presence) {
      // child bitmap = parent bitmap + the new id, from the buffer of this step's parity into the other one
      const long long plane = (long long)rows * a.words;
      const uint32_t* src = st.presence + (long long)(t & 1) * plane;
      uint32_t* dst = st.presence + (long long)((t + 1) & 1) * plane;
      for (int j = 0; j < nb; ++j) {
        const uint32_t* s = src + (long long)(b * nb + sm.slot_parent[j]) * a.words;
        uint32_t* d = dst + (long long)(b * nb + j) * a.words;
        const int tok = sm.slot_token[j];
        for (int w = tid; w < a.words; w += BS_THREADS) d[w] = s[w] | (w == (tok >> 5) ? 1u << (tok & 31) : 0u);
      }
    }
  }
  // ---- last CTA to arrive: all-done flag, reorder length, step --------------------------------------------------
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    sm.last = atomicAdd(reinterpret_cast<unsigned long long*>(&st.state[1]), 1ull) == (unsigned long long)gridDim.x - 1;
  }
  __syncthreads();
  if (!sm.last) return;
  __threadfence();
  int all = 1;
  for (int i = tid; i < a.B; i += BS_THREADS)
    if (!*reinterpret_cast<volatile int32_t*>(&st.done[i])) all = 0;
  all = __syncthreads_and(all);
  if (tid == 0) {
    st.state[2] = all ? 1ull : 0ull;
    // generated positions [S, S + step) of the cache to reorder; none after the last selection, which no decode
    // step reads
    st.state[3] = step + 1 == (unsigned long long)a.max_new ? 0ull : step;
    st.state[1] = 0;
    st.state[0] = step + 1;
  }
}

struct ReorderArgs {
  void* const* layer_kv;  // [2 * L]: K_0, V_0, K_1, V_1, ...
  int nb, row_vecs, pos_per_cta;
  long long max_len, S, B;
  const int32_t* parents;
  const unsigned long long* state;
  const int32_t* done;
};

__global__ void __launch_bounds__(RO_THREADS) kv_reorder_kernel(ReorderArgs a) {
  extern __shared__ uint4 stage[];
  __shared__ int par[BS_MAX_BEAMS];
  __shared__ int moved;
  pdl_wait();
  pdl_launch_dependents();
  const long long n = (long long)a.state[3];
  const long long p0 = (long long)blockIdx.x * a.pos_per_cta;
  const int b = blockIdx.y, tid = threadIdx.x, nb = a.nb;
  if (p0 >= n || a.done[b]) return;
  const long long col = (long long)a.state[0] - 1;
  if (tid == 0) moved = 0;
  __syncthreads();
  if (tid < nb) {
    par[tid] = a.parents[col * a.B * nb + (long long)b * nb + tid];
    if (par[tid] != tid) atomicOr(&moved, 1);
  }
  __syncthreads();
  if (!moved) return;  // identity permutation: nothing to write
  const int np = (int)min((long long)a.pos_per_cta, n - p0);
  const int per_pos = nb * a.row_vecs, total = np * per_pos;
  for (int kv = 0; kv < 2; ++kv) {
    uint4* base = reinterpret_cast<uint4*>(a.layer_kv[2 * blockIdx.z + kv]);
    auto gidx = [&](int e) {  // element e of the staged block -> (position, beam, vector) in the cache
      const int p = e / per_pos, r = e - p * per_pos, j = r / a.row_vecs, v = r - j * a.row_vecs;
      return ((long long)(b * nb + j) * a.max_len + a.S + p0 + p) * a.row_vecs + v;
    };
    for (int e = tid; e < total; e += RO_THREADS) stage[e] = base[gidx(e)];
    __syncthreads();
    for (int e = tid; e < total; e += RO_THREADS) {
      const int p = e / per_pos, r = e - p * per_pos, j = r / a.row_vecs, v = r - j * a.row_vecs;
      if (par[j] != j) base[gidx(e)] = stage[p * per_pos + par[j] * a.row_vecs + v];
    }
    __syncthreads();
  }
}

int n_chunks_of(int64_t V) { return (int)((V + BS_CHUNK - 1) / BS_CHUNK); }

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int b200mix_beam_search_workspace_size(int64_t B, int64_t nb, int64_t V, int64_t* bytes) {
  B200_CHECK_ARG(bytes, "beam_search_workspace_size: null pointer");
  B200_CHECK_ARG(B >= 1 && nb >= 2 && nb <= BS_MAX_BEAMS && V >= 2 * nb && V <= (1ll << 20),
                 "beam_search_workspace_size: bad shape (B=%lld, nb=%lld, V=%lld)", (long long)B, (long long)nb,
                 (long long)V);
  const int64_t rows = B * nb, nc = n_chunks_of(V);
  *bytes = rows * nc * 2 * nb * 8 + rows * nc * 8;
  return 0;
}

extern "C" int b200mix_beam_search_step(const float* logits, int64_t ld, int64_t B, int64_t nb, int64_t V,
                                        const b200mix_beam_state* st, void* workspace, int64_t workspace_bytes,
                                        int64_t max_new, int64_t eos_id, int64_t pad_id, float penalty,
                                        float diversity_rate, double length_penalty, int32_t early_stopping,
                                        void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(logits && st && workspace, "beam_search_step: null pointer");
  B200_CHECK_ARG(st->state && st->next_ids && st->beam_scores && st->tokens && st->parents && st->hyp_score &&
                     st->hyp_step && st->hyp_slot && st->hyp_count && st->hyp_worst && st->done,
                 "beam_search_step: null pointer in the beam state");
  B200_CHECK_ARG(nb >= 2 && nb <= BS_MAX_BEAMS, "beam_search_step: num_beams=%lld must be in [2, %d]", (long long)nb,
                 BS_MAX_BEAMS);
  B200_CHECK_ARG(B >= 1 && B * nb <= 65535, "beam_search_step: B * num_beams = %lld must be in [1, 65535]",
                 (long long)(B * nb));
  B200_CHECK_ARG(V >= 2 * nb && V <= (1ll << 20), "beam_search_step: V=%lld must be in [2 * num_beams, 2^20]",
                 (long long)V);
  B200_CHECK_ARG(ld >= V, "beam_search_step: row stride %lld < V=%lld", (long long)ld, (long long)V);
  B200_CHECK_ARG(max_new >= 1 && max_new < (1ll << 31), "beam_search_step: max_new=%lld out of range",
                 (long long)max_new);
  B200_CHECK_ARG(eos_id >= -1 && eos_id < V, "beam_search_step: eos_id=%lld must be -1 or in [0, V)",
                 (long long)eos_id);
  B200_CHECK_ARG(pad_id >= 0 && pad_id < V, "beam_search_step: pad_id=%lld must be in [0, V)", (long long)pad_id);
  B200_CHECK_ARG(penalty > 0.0f && penalty <= FLT_MAX, "beam_search_step: repetition penalty must be > 0 (got %g)",
                 (double)penalty);
  B200_CHECK_ARG(penalty == 1.0f || st->presence, "beam_search_step: a repetition penalty needs the presence bitmap");
  B200_CHECK_ARG(diversity_rate >= 0.0f && diversity_rate <= FLT_MAX,
                 "beam_search_step: diversity_rate must be finite and >= 0 (got %g)", (double)diversity_rate);
  B200_CHECK_ARG(length_penalty == length_penalty && length_penalty >= -DBL_MAX && length_penalty <= DBL_MAX,
                 "beam_search_step: length_penalty must be finite");
  int64_t need = 0;
  b200mix_beam_search_workspace_size(B, nb, V, &need);
  B200_CHECK_ARG(workspace_bytes >= need, "beam_search_step: workspace of %lld bytes < %lld",
                 (long long)workspace_bytes, (long long)need);
  auto al = [](const void* p, int n) { return reinterpret_cast<uintptr_t>(p) % n == 0; };
  B200_CHECK_ARG(al(logits, 4) && al(workspace, 16) && al(st->state, 8) && al(st->next_ids, 8) &&
                     al(st->beam_scores, 4) && al(st->tokens, 8) && al(st->parents, 4) && al(st->hyp_score, 8) &&
                     al(st->hyp_step, 4) && al(st->hyp_slot, 4) && al(st->hyp_count, 4) && al(st->hyp_worst, 8) &&
                     al(st->done, 4) && al(st->presence, 4),
                 "beam_search_step: misaligned buffer");
  StepArgs a;
  a.logits = logits;
  a.ld = ld;
  a.B = (int)B;
  a.nb = (int)nb;
  a.V = (int)V;
  a.words = (int)((V + 31) / 32);
  a.n_chunks = n_chunks_of(V);
  a.st = *st;
  a.keys = reinterpret_cast<unsigned long long*>(workspace);
  a.stats = reinterpret_cast<float2*>(a.keys + B * nb * a.n_chunks * 2 * nb);
  a.max_new = max_new;
  a.eos = eos_id;
  a.pad = pad_id;
  a.penalty = penalty;
  a.diversity = diversity_rate;
  a.length_penalty = length_penalty;
  a.early_stopping = early_stopping != 0;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const dim3 grid((unsigned)a.n_chunks, (unsigned)(B * nb));
  B200_CUDA(launch_pdl(beam_stats_kernel, grid, dim3(BS_THREADS), 0, s, 1, a));
  B200_CUDA(launch_pdl(beam_topk_kernel, grid, dim3(BS_THREADS), 0, s, 1, a));
  B200_CUDA(launch_pdl(beam_merge_kernel, dim3((unsigned)B), dim3(BS_THREADS), 0, s, 1, a));
  return 0;
}

extern "C" int b200mix_kv_reorder(void* const* layer_kv, int64_t n_layers, int64_t B, int64_t nb, int64_t max_len,
                                  int64_t row_elems, int64_t S, int64_t max_new, const int32_t* parents,
                                  const uint64_t* state, const int32_t* done, void* stream) {
  if (int rc = ensure_device()) return rc;
  B200_CHECK_ARG(layer_kv && parents && state && done, "kv_reorder: null pointer");
  B200_CHECK_ARG(nb >= 2 && nb <= BS_MAX_BEAMS, "kv_reorder: num_beams=%lld must be in [2, %d]", (long long)nb,
                 BS_MAX_BEAMS);
  B200_CHECK_ARG(n_layers >= 1 && n_layers <= 65535 && B >= 1 && B <= 65535,
                 "kv_reorder: n_layers=%lld / B=%lld out of range", (long long)n_layers, (long long)B);
  B200_CHECK_ARG(row_elems >= 8 && row_elems % 8 == 0 && nb * row_elems * 2 <= RO_SMEM,
                 "kv_reorder: row of %lld bf16 must be a multiple of 8 with num_beams * row bytes <= %d",
                 (long long)row_elems, RO_SMEM);
  B200_CHECK_ARG(max_new >= 1 && S >= 0 && S + max_new <= max_len, "kv_reorder: S=%lld + max_new=%lld > max_len=%lld",
                 (long long)S, (long long)max_new, (long long)max_len);
  B200_CHECK_ARG(reinterpret_cast<uintptr_t>(layer_kv) % 8 == 0 && reinterpret_cast<uintptr_t>(parents) % 4 == 0 &&
                     reinterpret_cast<uintptr_t>(state) % 8 == 0 && reinterpret_cast<uintptr_t>(done) % 4 == 0,
                 "kv_reorder: misaligned buffer");
  ReorderArgs a;
  a.layer_kv = layer_kv;
  a.nb = (int)nb;
  a.row_vecs = (int)(row_elems / 8);
  a.pos_per_cta = (int)(RO_SMEM / (nb * row_elems * 2));
  a.max_len = max_len;
  a.S = S;
  a.B = B;
  a.parents = parents;
  a.state = reinterpret_cast<const unsigned long long*>(state);
  a.done = done;
  const dim3 grid((unsigned)((max_new + a.pos_per_cta - 1) / a.pos_per_cta), (unsigned)B, (unsigned)n_layers);
  const size_t smem = (size_t)a.pos_per_cta * nb * row_elems * 2;
  B200_CUDA(launch_pdl(kv_reorder_kernel, grid, dim3(RO_THREADS), smem, reinterpret_cast<cudaStream_t>(stream), 1, a));
  return 0;
}
