/*
 * b200mix — C ABI of the H100-native (sm_90a) hot path that replaces, for PaddleMIX's denoiser-forward /
 * ViT+LLM attention path, the arithmetic the reference delegates to paddlepaddle-gpu and to its Triton custom ops.
 *
 * Conventions (mirrors the ownership model of the reference's custom ops, paddlemix/triton_ops/triton_ops.py:641-693:
 * inputs are borrowed raw device pointers, work is enqueued on the caller's stream, no hidden synchronisation):
 *   - every pointer is a DEVICE pointer unless the name says host; the caller owns all buffers;
 *   - activations are bf16 row-major, images are NHWC ([B,H,W,C], the reference's data_format="NHWC" switch,
 *     ppdiffusers/models/unet_2d_condition.py:227,881-882); biases / modulation vectors / statistics are fp32;
 *   - Linear weights are [N_out, K_in] with K contiguous (torch layout; Paddle's [in,out] nn.Linear.weight,
 *     ppdiffusers/models/modeling_pytorch_paddle_utils.py:27-63, is transposed once at load by the Python shim);
 *     conv3x3 weights are [C_out, kh, kw, C_in];
 *   - every function returns 0 on success or a negative b200mix_status and never aborts;
 *     b200mix_last_error() returns a thread-local message for the last failure;
 *   - `stream` is a cudaStream_t passed as void*.
 * There is no CPU fallback: every entry point fails with B200MIX_ERR_NO_DEVICE when no sm_90 device is present.
 */
#ifndef B200MIX_H_
#define B200MIX_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum b200mix_status {
  B200MIX_OK = 0,
  B200MIX_ERR_INVALID = -1,   /* bad shape / alignment / argument */
  B200MIX_ERR_CUDA = -2,      /* a CUDA runtime/driver call failed */
  B200MIX_ERR_NO_DEVICE = -3, /* no sm_90 device visible */
  B200MIX_ERR_UNSUPPORTED = -4
} b200mix_status;

/* B200MIX_ACT_RELU is taken by b200mix_activation only; the GEMM epilogues cover NONE .. QUICK_GELU. */
enum { B200MIX_ACT_NONE = 0, B200MIX_ACT_SILU = 1, B200MIX_ACT_GELU_ERF = 2, B200MIX_ACT_GELU_TANH = 3, B200MIX_ACT_QUICK_GELU = 4,
       B200MIX_ACT_RELU = 5 };
enum { B200MIX_GLU_NONE = 0, B200MIX_GLU_GEGLU = 1, B200MIX_GLU_SWIGLU = 2 };

/* Fused GEMM epilogue, applied in this order on the fp32 accumulator of element (m, n):
 *   v = acc + bias[n] + row_add[(m / rows_per_group) * ld_row + n]
 *   v = act(v)
 *   glu != 0: columns are interleaved (2j = value, 2j+1 = gate); out[m, j] = value * gelu_erf(gate)   (GEGLU,
 *             ppdiffusers/models/activations.py:83-104) or silu(gate) * value (SwiGLU, modeling_qwen2_vl.py:492-493);
 *             the output then has N/2 columns
 *   v = v * row_gate[(m / rows_per_group) * ld_row + n]          (AdaLN-Zero gate, attention.py:196-214)
 *   v = (v + residual[r * ldr + n]) * out_scale                  (ResnetBlock2D output_scale_factor, resnet.py:806)
 *       with r = m, or m % residual_row_mod when residual_row_mod > 0 (a table shared by all groups, e.g. the
 *       cropped positional embedding of PatchEmbed, embeddings.py:186-247)
 */
typedef struct b200mix_epilogue {
  const float* bias;      /* [N] or NULL */
  const float* row_add;   /* [groups, ld_row] or NULL */
  const float* row_gate;  /* [groups, ld_row] or NULL */
  int64_t ld_row;
  int64_t rows_per_group; /* rows of the output sharing one row_add/row_gate row (H*W or sequence length) */
  const void* residual;   /* bf16 [M, ldr] or NULL */
  int64_t ldr;
  int32_t act;            /* B200MIX_ACT_* */
  int32_t glu;            /* B200MIX_GLU_* */
  int32_t out_fp32;       /* 0: bf16 output, 1: fp32 output */
  float out_scale;        /* 1.0f for none */
  int64_t residual_row_mod; /* 0: residual row = m */
  /* LayerNorm folded into the two Linear layers either side of it (BasicTransformerBlock: h = to_out(..) + h;
   * n = norm(h); q = to_q(n), attention.py:352-489). The PRODUCER of h passes stats_out = int64 [M][2], ZEROED by the
   * caller: its epilogue adds, per output row, the sum and the sum of squares of the bf16 values it stores, as 2^24
   * fixed point with integer atomics (integer adds commute: the totals are reproducible bit for bit).
   * The CONSUMER of LayerNorm(h) is called on h itself with the norm's affine folded into its weights,
   *   W'[n,k] = bf16(W[n,k] * gamma[k]),  ln_colsum[n] = sum_k W'[n,k],  bias'[n] = bias[n] + sum_k W[n,k] * beta[k],
   * passes ln_stats = that table, and rebuilds mean / rstd of every row in its epilogue:
   *   out[m,n] = rstd[m] * (acc[m,n] - mean[m] * ln_colsum[n]) + bias'[n]     (== Linear(LayerNorm(h)) algebraically;
   * h is not rounded a second time, so the result is closer to the fp32 reference than the two-kernel form).
   * ln_rms = 1: RMSNorm (no mean term). All NULL / 0 when unused.
   * Range: the int64 totals hold |sum x| and sum x^2 up to 2^63 / 2^24 = 5.5e11 per row (a 1280-wide row of RMS 2e4);
   * mean / variance are rebuilt in fp64 (E[x^2] - mean^2 cancels mean^2 / var, which fp32 would lose 2^-8 of at
   * |mean| / std = 2^8). acc - mean * ln_colsum is fp32 from the tensor cores and cancels |mean| / std: measured on an
   * H100 at |mean| / std = 2^8 the output stays within 6e-4 rms of fp64, under its own bf16 step, for every row bf16
   * can represent (|mean| / std < 2^8). Callers with rows outside that range keep b200mix_layernorm. */
  void* stats_out;
  const void* ln_stats;
  const float* ln_colsum;
  int32_t ln_rms;
  float ln_eps;
} b200mix_epilogue;

const char* b200mix_last_error(void);
const char* b200mix_version(void);
/* Select the device for the calling thread and verify it is sm_90. Replaces paddle.set_device / the implicit
 * place of paddle::Tensor in the reference ops. */
int b200mix_init(int device);
int b200mix_num_sms(void);
/* cudaMemsetAsync(ptr, 0, bytes) on `stream`: zeroes the row-statistics tables of b200mix_epilogue.stats_out. */
int b200mix_zero_bytes(void* ptr, int64_t bytes, void* stream);

/* ---- the path's only collective (SURVEY.md §8b, §8e) -------------------------------------------------------------
 * Images are sharded over ranks (one process per GPU, weights replicated, no per-step communication); the finished
 * latents are gathered once over NCCL. For contrast, the reference's on-path collective site does 4 scatters + 1
 * all_gather per step (pipelines/stable_diffusion_3/pipeline_stable_diffusion_3.py:803-839).
 *   b200mix_nccl_load(path)      dlopen the NCCL the caller names ("" / NULL: "libnccl.so.2" on the loader path)
 *   b200mix_nccl_unique_id(id)   rank 0: 128-byte ncclUniqueId, handed to the other ranks by the caller's launcher
 *   b200mix_comm_init(&comm, world, rank, id)   after b200mix_init(device); ncclCommInitRank
 *   b200mix_allgather_latents(comm, send, recv, bytes_per_rank, stream)   recv = [world * bytes_per_rank], rank order
 *   b200mix_comm_destroy(comm) */
int b200mix_nccl_load(const char* libnccl_path);
int b200mix_nccl_version(void);
int b200mix_nccl_unique_id(void* id128);
int b200mix_comm_init(void** comm, int32_t world_size, int32_t rank, const void* id128);
int b200mix_allgather_latents(void* comm, const void* send, void* recv, int64_t bytes_per_rank, void* stream);
int b200mix_comm_destroy(void* comm);

/* ---- dense contractions on wgmma tensor cores (TMA -> smem -> wgmma -> registers -> fused epilogue) ----------- */

/* C[M, N(/2 if glu)] = epilogue(A[M,K] @ W[N,K]^T). Replaces F.linear (ppdiffusers/models/lora.py:453-459) and
 * 1x1 conv on NHWC (lora.py:365-377). A, W bf16; lda/ldw/ldc in elements, multiples of 8. */
int b200mix_linear(const void* A, int64_t lda, const void* W, int64_t ldw, void* C, int64_t ldc, int64_t M, int64_t N,
                   int64_t K, const b200mix_epilogue* epi, void* stream);

/* Batched-strided Linear: for b < nbatch, C_b[rows,N] = epilogue(A_b[rows,K] @ W^T), X_b = X + b * x_bstride
 * (elements). Per-group epilogue vectors are indexed by b; r_bstride is the residual's batch stride. Lets the image
 * and text token ranges of SD3's joint [B, n_img+n_txt, *] buffers be produced / consumed in place
 * (JointAttnProcessor2_5 concat / split, attention_processor.py:934-975). */
int b200mix_linear_batched(const void* A, int64_t lda, int64_t a_bstride, const void* W, int64_t ldw, void* C,
                           int64_t ldc, int64_t c_bstride, int64_t rows, int64_t nbatch, int64_t N, int64_t K,
                           const b200mix_epilogue* epi, int64_t r_bstride, void* stream);

/* ---- weight-only int8 Linear (PaddleNLP quant_type="weight_only_int8": paddle.nn.quant.weight_quantize +
 * weight_only_linear; PaddleMIX triton_ops.py:363-563 weight_only_int8) ----------------------------------------------
 * b200mix_quantize_w8: W fp32 (w_is_fp32 = 1) or bf16 [N, K] row-major -> q int8 (N * K bytes, 16-byte aligned) and
 * scale fp32 [N]. Per row n: scale[n] = max_k |W[n,k]| / 127.0f and q[n,k] = clip(roundf(W[n,k] / scale[n]), -127, 127),
 * both IEEE fp32 divisions, roundf rounding half away from zero (paddle.round). A row that is all zero gets scale 0 and
 * q 0 (deliberately not 0 / 0 = NaN). Requires N % 16 == 0 and K % 64 == 0.
 * q is written in the device layout the GEMM reads, and this function is its only producer:
 *   q = [N / 16][K / 32][32 lanes][16 bytes]; byte 8 s + 2 r + e of lane l = 4 g + t holds element
 *   (row 16 tile + g + 8 (r & 1), k 32 blk + 16 s + 2 t + 8 (r >> 1) + e), s, e in {0, 1}, r in 0..3
 * (the A-operand fragments of two mma.m16n8k16 steps: one coalesced 512-byte load per warp and 16 x 32 block).
 *
 * b200mix_linear_w8: C[M, N(/2 if glu)] = epilogue(scale[n] * sum_k A[m,k] * q[n,k]); the scale multiplies the fp32
 * accumulator before the bias. A bf16 (16-byte aligned, lda % 8 == 0), q / scale from b200mix_quantize_w8.
 * Epilogue fields: bias, act, glu (interleaved rows as b200mix_linear), residual, out_fp32; any other field set returns
 * B200MIX_ERR_UNSUPPORTED. Requires N % 16 == 0 and K % 64 == 0 (B200MIX_ERR_INVALID otherwise).
 * Small M (decode) streams q through tensor cores; larger M expands bf16(q * scale) into `workspace` and runs
 * b200mix_linear. The workspace (16-byte aligned) must hold b200mix_linear_w8_workspace_size bytes; it is 0 for small M,
 * where workspace may be NULL. No allocation and no host synchronisation: CUDA-graph capturable. */
int b200mix_quantize_w8(const void* W, int32_t w_is_fp32, void* q, float* scale, int64_t N, int64_t K, void* stream);
int b200mix_linear_w8_workspace_size(int64_t M, int64_t N, int64_t K, int64_t* bytes);
int b200mix_linear_w8(const void* A, int64_t lda, const void* q, const float* scale, void* C, int64_t ldc, int64_t M,
                      int64_t N, int64_t K, const b200mix_epilogue* epi, void* workspace, int64_t workspace_bytes,
                      void* stream);

/* y[B,Ho,Wo,Cout] = epilogue(conv3x3(x[B,H,W,Cin], w[Cout,3,3,Cin], padding 1, stride 1|2)). Implicit GEMM without
 * im2col: each of the 9 taps is a shifted TMA box load with hardware zero fill at the borders.
 * Replaces F.conv2d in ResnetBlock2D / Downsample2D / Upsample2D / conv_out (resnet.py:271-294,169-218,728-808).
 * Cin must be a multiple of 64 (conv_in with Cin=4 is b200mix_conv3x3_small_cin). */
int b200mix_conv3x3(const void* x, const void* w, void* y, int64_t B, int64_t H, int64_t W, int64_t Cin, int64_t Cout,
                    int32_t stride, const b200mix_epilogue* epi, void* stream);

/* y[B,2H,2W,Cout] = epilogue(conv3x3(nearest_upsample_2x(x[B,H,W,Cin]), padding 1)) without materialising the upsampled
 * tensor: Upsample2D.forward (ppdiffusers/models/resnet.py:169-218: F.interpolate(scale_factor=2.0, mode="nearest") then
 * self.conv). Each output parity (y%2, x%2) is a 2x2 conv over the low-resolution input, so w4 holds the 3x3 filter
 * folded per parity: bf16 [Cout, 4 (py,px), 4 (a,b), Cin], tap (a,b) of parity (py,px) = sum of the taps of w[Cout,3,3,Cin]
 * that read the same input pixel (py = 0: a=0 <- ky 0, a=1 <- ky 1+2; py = 1: a=0 <- ky 0+1, a=1 <- ky 2; same in x),
 * summed in fp32 and rounded once. 4/9 of the plain conv's FLOPs and none of the 4x tensor's traffic. Cin % 64 == 0.
 * epilogue: bias / row_add (rows_per_group = 4*H*W) / activation / residual[B,2H,2W,Cout] / out_scale. */
int b200mix_conv3x3_up2x(const void* x, const void* w4, void* y, int64_t B, int64_t H, int64_t W, int64_t Cin,
                         int64_t Cout, const b200mix_epilogue* epi, void* stream);

/* conv3x3 stride 1 pad 1 for tiny Cin (UNet conv_in, unet_2d_condition.py:1064): x fp32 or bf16 NHWC [B,H,W,Cin],
 * w bf16 [Cout,3,3,Cin], bias fp32, y bf16 NHWC. CUDA-core kernel (K = 9*Cin = 36 is below one MMA k-block). */
int b200mix_conv3x3_small_cin(const void* x, int32_t x_fp32, const void* w, const float* bias, void* y, int64_t B,
                              int64_t H, int64_t W, int64_t Cin, int64_t Cout, void* stream);

/* y[B,Ho,Wo,Cout] = act(conv3x3(x[B,H,W,Cin], w[Cout,3,3,Cin], padding 1, stride 1|2) + bias), NHWC bf16 in / out,
 * 1 <= Cin <= 128, Cout % 8 == 0, Cout <= 256 (ControlNetConditioningEmbedding, controlnet.py:71-113). bias fp32 [Cout]
 * or NULL; act B200MIX_ACT_NONE or B200MIX_ACT_SILU; stride 2 needs even H and W (Ho = H/2, Wo = W/2).
 * Tensor-core implicit GEMM on mma.sync.m16n8k16 with K = 9 taps x Cin padded to 16 (csrc/conv_narrow.cu). */
int b200mix_conv3x3_narrow(const void* x, const void* w, const float* bias, void* y, int64_t B, int64_t H, int64_t W,
                           int64_t Cin, int64_t Cout, int32_t stride, int32_t act, void* stream);

/* Scaled dot-product attention, flash-style on wgmma (S=QK^T and O+=PV in registers, online softmax in registers).
 * Full signature of scaled_dot_product_attention_(query, key, value, attn_mask, dropout_p=0, is_causal, scale)
 * (ppdiffusers/patches/paddle_patch.py:414-424), semantics of its `math` branch (:445-461):
 *   softmax(q k^T * scale [+ attn_mask | causal mask]) v.
 * q/k/v/o are bf16 with head_dim contiguous; strides in elements for (batch, seq, head). D in {64, 128, 192}; heads
 * with other sizes are zero-padded by the shim at weight-load time. Hq % Hkv == 0 (GQA, modeling_qwen2_vl.py:497-506).
 * cu_seqlens (int32 device [nseq+1], may be NULL) switches on the varlen block-diagonal mode of the Qwen2-VL ViT
 * (modeling_qwen2_vl.py:354-381): then B must be 1 and both q and k are packed along seq. kv_lens (int32 device [B],
 * may be NULL) gives the number of valid keys per batch element (the block-diagonal text mask of STDiT2's
 * MultiHeadCrossAttention, Open-Sora layers/blocks.py:275-331); a batch element with 0 valid keys gets zeros. The K / V
 * rows between kv_lens[b] and Sk are still read (they take probability 0): they must hold FINITE values (a preallocated
 * KV cache is zero-filled once).
 * attn_mask (may be NULL): additive bias on the scaled scores, bf16 or fp32 (mask_fp32), element (b, h, q, k) at
 * attn_mask + b*m_sb + h*m_sh + q*m_sq + k (key stride 1; a stride of 0 broadcasts that dimension, so the
 * [B,1,1,Sk] key-padding bias (1 - m) * -10000 of unet_2d_condition.py:916-927 and the full [B,H,Sq,Sk] mask of
 * attention_processor.py:588-630 are both expressible). Like the reference, attn_mask is not combined with is_causal.
 * causal uses the bottom-right alignment (query i sees keys <= i + Sk - Sq) and requires Sq <= Sk. */
int b200mix_sdpa(const void* q, const void* k, const void* v, void* o, int64_t B, int64_t Hq, int64_t Hkv, int64_t Sq,
                 int64_t Sk, int64_t D, int64_t q_sb, int64_t q_ss, int64_t q_sh, int64_t k_sb, int64_t k_ss,
                 int64_t k_sh, int64_t v_sb, int64_t v_ss, int64_t v_sh, int64_t o_sb, int64_t o_ss, int64_t o_sh,
                 float scale, int32_t causal, const int32_t* cu_seqlens, int32_t nseq, const int32_t* kv_lens,
                 const void* attn_mask, int32_t mask_fp32, int64_t m_sb, int64_t m_sh, int64_t m_sq, void* stream);

/* ---- HBM-bound normalisation / modulation kernels (coalesced 16-byte accesses, fp32 statistics) -------------- */

/* GroupNorm (+ optional SiLU) over NHWC bf16; the input may be the channel-concatenation [x1 | x2] of two tensors
 * (skip connections, unet_2d_blocks.py:2353-2356) which is thereby never materialised. x2 may be NULL (C2 = 0).
 * Replaces nn.GroupNorm + nonlinearity (resnet.py:667-692,760-786; transformer_2d.py:161; unet_2d_condition.py:1193).
 * y bf16 [B,H,W,C1+C2]. Two launches: per-CTA partial sums of x - c and (x - c)^2 in fp32, exchanged as fixed-point
 * int64 (2^-24 / 2^-16 resolution) and added into 128-bit totals by the last CTA of each batch element (exact, so
 * bit-reproducible), then apply. The shift c is the group's mean over pixel 0 of the batch element. Range (tested on
 * the VAE decoder's groups of up to 8.4 M elements): |mean| / std up to 2^8 with pixel 0's group mean within a few std
 * of the group mean, RMS 1e-3 to 1e4; one CTA's partial must stay under 2^47 in sum (x - c)^2. `stats` = scratch of at least
 * 4096 + (4*num_sms + 2*B) * groups * 16 bytes that the caller ZERO-FILLS ONCE at allocation (its first 4 KB hold the
 * arrival counters, which every call leaves at zero); one scratch per concurrently used stream. */
int b200mix_groupnorm_nhwc(const void* x1, int64_t C1, const void* x2, int64_t C2, const float* gamma,
                           const float* beta, void* y, void* stats, int64_t stats_bytes, int64_t B, int64_t HW,
                           int32_t groups, float eps, int32_t silu, void* stream);

/* Row-wise LayerNorm family. For each row m of x[M,N] (bf16):
 *   r = x + gate[g]*delta (if delta given; also written to resid_out)            (fused_adaLN_scale_residual,
 *   y = LN(r) [*weight + bias] [*(1 + scale[g]) + shift[g]]                       triton_ops.py:702-755,981-1027)
 * with g = m / rows_per_group; gate/scale/shift fp32 [groups, ld_mod]. rms != 0 switches to RMSNorm
 * (x * rsqrt(mean(x^2)+eps) * weight, modeling_qwen2_vl.py:467-478). */
int b200mix_layernorm(const void* x, const void* delta, const float* gate, void* resid_out, void* y,
                      const float* weight, const float* bias, const float* scale, const float* shift, int64_t ld_mod,
                      int64_t rows_per_group, int64_t M, int64_t N, float eps, int32_t rms, void* stream);

/* Row softmax y[m, :] = softmax(x[m, :] * scale): fp32 scores [M, ldx] -> bf16 probabilities [M, ldy], N <= 51200.
 * The attention of the VAE decoder's mid block (one 512-wide head over H*W tokens, ppdiffusers/models/vae.py:232-241;
 * AttnProcessor, attention_processor.py:673-735) = score GEMM (fp32 out) -> this kernel -> PV GEMM. */
int b200mix_softmax_rows(const float* x, void* y, int64_t M, int64_t N, int64_t ldx, int64_t ldy, float scale,
                         void* stream);

/* ---- small elementwise kernels ------------------------------------------------------------------------------ */

/* Sinusoidal timestep embedding, fp32 math (embeddings.py:26-64): out[b, :] for t[b]; flip_sin_to_cos, shift, scale
 * as in the reference; out bf16 or fp32 [B, ld_out] written at column offset col0. */
int b200mix_timestep_embedding(const float* t, void* out, int32_t out_fp32, int64_t B, int64_t dim, int64_t ld_out,
                               int64_t col0, int32_t flip_sin_to_cos, float downscale_freq_shift, float scale,
                               float max_period, void* stream);

/* y = act(x) elementwise for bf16/fp32 vectors (SiLU on temb, resnet.py:772-776; ReLU = max(x, 0), the nn.ReLU of the
 * T2I-Adapter resnet blocks, models/adapter.py:450,571). act is any B200MIX_ACT_*; y may alias x. */
int b200mix_activation(const void* x, void* y, int64_t n, int32_t act, int32_t x_fp32, int32_t y_fp32, void* stream);

/* Nearest-neighbour x2 upsample NHWC bf16 (F.interpolate(scale_factor=2, mode="nearest"), resnet.py:197-199). */
int b200mix_upsample_nearest2x_nhwc(const void* x, void* y, int64_t B, int64_t H, int64_t W, int64_t C, void* stream);

/* Channel concat of two NHWC bf16 tensors (unet_2d_blocks.py:2353-2356), for the 1x1 shortcut input. */
int b200mix_concat_channels(const void* x1, int64_t C1, const void* x2, int64_t C2, void* y, int64_t rows,
                            void* stream);

/* Layout/dtype conversion: NCHW fp32|bf16 -> NHWC bf16 and back (pipelines hand NCHW latents to unet.forward). */
int b200mix_nchw_to_nhwc(const void* x, int32_t x_fp32, void* y, int64_t B, int64_t C, int64_t H, int64_t W,
                         void* stream);
int b200mix_nhwc_to_nchw(const void* x, void* y, int32_t y_fp32, int64_t B, int64_t C, int64_t H, int64_t W,
                         void* stream);

/* T2I-Adapter input, nn.PixelUnshuffle(f) + the cast to the model dtype (models/adapter.py:306,328): x fp32|bf16 NCHW
 * [B,C,H,W] -> y bf16 NHWC [B,H/f,W/f,C*f*f] with y[b,h,w,c*f*f + i*f + j] = x[b,c,h*f+i,w*f+j]. f is 8 or 16; H and W
 * must be multiples of f; x and y 16-byte aligned. Each input pixel is read once, each thread writes one 16-byte piece
 * (8 channels = 8 neighbouring pixels of one input row). */
int b200mix_pixel_unshuffle(const void* x, int32_t x_fp32, void* y, int64_t B, int64_t C, int64_t H, int64_t W, int32_t f,
                            void* stream);

/* nn.AvgPool2D(kernel_size=2, stride=2, ceil_mode=True) with Paddle's default exclusive=True (models/adapter.py:411,537)
 * on bf16 NHWC: y [B,ceil(H/2),ceil(W/2),C]; a window that overhangs an odd edge averages its valid pixels only. Sums
 * in fp32, rounded once. C % 8 == 0, x and y 16-byte aligned. */
int b200mix_avgpool2x2_nhwc(const void* x, void* y, int64_t B, int64_t H, int64_t W, int64_t C, void* stream);

/* T2I-Adapter residuals (MultiAdapter.forward, models/adapter.py:85-100, and the scale / tile / CFG concat of
 * pipeline_stable_diffusion_adapter.py:823-836) in one pass over bf16 row-major tensors:
 *   y[r, :] = sum_k weight[k] * x_k[r mod rows_k, :]     (r < rows_out, fp32 sum in k order, rounded once)
 * n inputs (1..8) given as host arrays of device pointers, row counts and weights; each x_k is [rows_k, row_elems].
 * row_elems % 8 == 0, every pointer 16-byte aligned; y must not alias an input. */
int b200mix_weighted_sum_rows(int32_t n, const void* const* x, const int64_t* rows_in, const float* weight, void* y,
                              int64_t rows_out, int64_t row_elems, void* stream);

/* y = a + r for an NHWC bf16 activation a [B,H,W,C]; r is NHWC bf16 (r_nchw = 0) or the caller's NCHW fp32|bf16 tensor
 * (r_nchw = 1). The ControlNet / T2I-Adapter residual adds of UNet2DConditionModel.forward:
 * down_block_additional_residuals, mid_block_additional_residual, down_intrablock_additional_residuals
 * (unet_2d_condition.py:1109-1155; unet_2d_blocks.py:1211-1213). y may alias a. */
int b200mix_add_residual_nhwc(const void* a, const void* r, int32_t r_fp32, int32_t r_nchw, void* y, int64_t B, int64_t C,
                              int64_t H, int64_t W, void* stream);

/* Fused classifier-free-guidance combine + DDIM step (scheduling_ddim.py:410-457), eta = 0, fp32 state, for every
 * prediction_type (0 = epsilon, 1 = sample, 2 = v_prediction; :424-443) with optional clip_sample (clip_sample_range > 0
 * clips the predicted x0, :446-452; <= 0: off):
 *   m = m_u + g*(m_c - m_u)  (pipeline_stable_diffusion.py:882-884; m_c NULL => m = m_u); m_u, m_c bf16 or fp32 (m_fp32)
 *   epsilon: x0 = (x - sb_t*m)/sa_t, eps = m;  sample: x0 = m, eps = (x - sa_t*x0)/sb_t;
 *   v_prediction: x0 = sa_t*x - sb_t*m, eps = sa_t*m + sb_t*x;   x_prev = sa_p*clip(x0) + sb_p*eps.
 * The four scalars sa_t = sqrt(alpha_prod_t), sb_t = sqrt(1 - alpha_prod_t) and sa_p, sb_p (the same for the previous
 * timestep) are computed on the host by the scheduler, bit-exactly as scheduling_ddim.py:410-457 does, and applied here
 * with the same operation order in fp32. */
int b200mix_ddim_step_ex(const void* m_u, const void* m_c, int32_t m_fp32, float guidance, const float* x, float* x_prev,
                         int64_t n, float sqrt_alpha_t, float sqrt_beta_t, float sqrt_alpha_prev, float sqrt_beta_prev,
                         int32_t prediction_type, float clip_sample_range, void* stream);

/* LCMScheduler.step (scheduling_lcm.py:468-545), fused CFG combine: x0 as in b200mix_ddim_step_ex, optional clip,
 * denoised = c_out*x0 + c_skip*x (boundary-condition scalings :453-459, computed on the host),
 * x_prev = sa_p*denoised + sb_p*noise (noise = the caller's randn, multi-step) or denoised (noise NULL: last step).
 * `denoised` (may be NULL) receives the denoised sample (LCMSchedulerOutput.denoised). */
int b200mix_lcm_step(const void* m_u, const void* m_c, int32_t m_fp32, float guidance, const float* x, const float* noise,
                     float* x_prev, float* denoised, int64_t n, float sqrt_alpha_t, float sqrt_beta_t, float c_skip,
                     float c_out, float sqrt_alpha_prev, float sqrt_beta_prev, int32_t prediction_type,
                     float clip_sample_range, void* stream);

/* Open-Sora IDDPM sampling step with learned-range variance and the reference's CFG (ppdiffusers/examples/Open-Sora:
 * schedulers/iddpm/__init__.py:97-114 forward_with_cfg, gaussian_diffusion.py:278-372 p_mean_variance, :409-485
 * p_sample; epsilon prediction, clip_denoised = False), one launch, fp32 state x [B, C, N] (N = T*H*W):
 *   model_out [2B, 2C, N] fp32 | bf16 (m_fp32), conditional rows [0, B) first; channel k < cfg_channel is guided,
 *     g = uncond + cfg_scale * (cond - uncond), every other channel comes from the conditional rows;
 *   eps = channels [0, C), v = channels [C, 2C);
 *   frac = (v + 1) / 2;  logvar = frac * max_log + (1 - frac) * min_log
 *   x0 = sqrt_recip_ac * x - sqrt_recipm1_ac * eps;  mean = coef1 * x0 + coef2 * x
 *   x_prev = mean + exp(0.5 * logvar) * noise  (add_noise != 0),  x_prev = mean  (add_noise == 0: respaced index 0)
 * The six scalars are the scheduler's fp64 tables rounded to fp32 (max_log = log(beta_t), min_log =
 * posterior_log_variance_clipped[t]). Every operation is rounded on its own in this order; exp is the fp64 exp rounded
 * to fp32. noise [B, C, N] fp32, or NULL: standard normals from Philox4x32-10 keyed by `seed`, four per element group
 * g (elements 4g .. 4g+3 of x):
 *   (r0..r3) = philox4x32_10(counter = (step, g mod 2^32, g div 2^32, 0), key = (seed mod 2^32, seed div 2^32)),
 *   u_k = (r_k + 0.5) 2^-32,  z_{2p} = fp32(sqrt(-2 ln u_{2p}) cos(2 pi u_{2p+1})),
 *   z_{2p+1} = fp32(sqrt(-2 ln u_{2p}) sin(2 pi u_{2p+1}))  (fp64 Box-Muller, p = 0, 1).
 * x_prev may alias x. x_dup (may be NULL) receives a second copy of x_prev: the unconditional half of the next step's
 * [2B, C, N] model input. */
int b200mix_iddpm_step(const void* model_out, int32_t m_fp32, const float* x, const float* noise, float* x_prev,
                       float* x_dup, int64_t B, int64_t C, int64_t n_per_channel, float cfg_scale, int32_t cfg_channel,
                       float sqrt_recip_alphas_cumprod, float sqrt_recipm1_alphas_cumprod, float posterior_mean_coef1,
                       float posterior_mean_coef2, float max_log, float min_log, int32_t add_noise, uint64_t seed,
                       int64_t step, void* stream);

/* rescale_noise_cfg (pipeline_stable_diffusion.py:69-80; pipeline_stable_diffusion_xl.py:1061-1067) in two launches:
 *   ratio[b] = std(eps_c[b]) / std(noise_cfg[b]),  noise_cfg = eps_u + g*(eps_c - eps_u)   (unbiased std over C,H,W)
 *   out = noise_cfg;  ratio != NULL: out = guidance_rescale * (noise_cfg*ratio[b]) + (1 - guidance_rescale) * noise_cfg
 * out is fp32 and feeds any scheduler step kernel with its CFG inputs left NULL. */
int b200mix_cfg_rescale_ratio(const void* eps_u, const void* eps_c, int32_t eps_fp32, float guidance, float* ratio,
                              int64_t B, int64_t n_per_sample, void* stream);
int b200mix_cfg_combine(const void* eps_u, const void* eps_c, int32_t eps_fp32, float guidance, const float* ratio,
                        float guidance_rescale, int64_t n_per_sample, float* out, int64_t n, void* stream);

/* FlowMatchEuler step (scheduling_flow_match_euler_discrete.py:244-275, s_churn = 0), fp32 state, same operation
 * order as the reference: denoised = x - v*sigma; derivative = (x - denoised)/sigma; x_prev = x + derivative*dt
 * with dt = sigma_next - sigma computed in fp32 on the host. */
int b200mix_euler_step(const void* v_u, const void* v_c, int32_t v_fp32, float guidance, const float* x, float* x_prev,
                       int64_t n, float sigma, float dt, void* stream);

/* EulerDiscreteScheduler (scheduling_euler_discrete.py:135-503; SDXL's default sampler), deterministic path
 * (s_churn = 0, epsilon prediction): its step IS b200mix_euler_step (pred = x - sigma*eps; derivative = (x - pred)/sigma;
 * x_prev = x + derivative*dt). scale_model_input (:218-241) divides the fp32 sample by (sigma^2 + 1) ** 0.5; the
 * host computes that denominator in fp32, this applies an IEEE fp32 division. */
int b200mix_scale_model_input(const float* x, float* y, int64_t n, float denom, void* stream);

/* EulerAncestralDiscreteScheduler.step ("Euler a", scheduling_euler_ancestral_discrete.py:268-357), fused with the CFG
 * combine, fp32 state, one rounding per operation in this order:
 *   m = m_u + g*(m_c - m_u)   (m_c NULL => m = m_u); m_u, m_c bf16 or fp32 (m_fp32)
 *   prediction_type 0 (epsilon):      x0 = x - sigma*m
 *   prediction_type 2 (v_prediction): x0 = m*c_out + x/s2p1   (c_out = -sigma/(sigma^2+1)^0.5, s2p1 = sigma^2+1)
 *   d = (x - x0)/sigma;  x_prev = x + d*dt;  x_prev = x_prev + z*sigma_up
 * The same arithmetic as b200mix_euler_step up to the noise term. The host computes in fp32, in the order of
 * :339-347, sigma_up = (sigma_to^2*(sigma_from^2 - sigma_to^2)/sigma_from^2)^0.5,
 * sigma_down = (sigma_to^2 - sigma_up^2)^0.5 and dt = sigma_down - sigma. z is noise[i] (fp32, x's element count) or,
 * with noise NULL, the Philox stream of b200mix_iddpm_step keyed by (seed, step): element group g = elements
 * 4g .. 4g+3 takes the four normals of philox4x32_10(counter = (step, g mod 2^32, g div 2^32, 0),
 * key = (seed mod 2^32, seed div 2^32)). x_prev may alias x. */
int b200mix_euler_ancestral_step(const void* m_u, const void* m_c, int32_t m_fp32, float guidance, const float* x,
                                 const float* noise, float* x_prev, int64_t n, int32_t prediction_type, float sigma,
                                 float c_out, float s2p1, float dt, float sigma_up, uint64_t seed, int64_t step,
                                 void* stream);

/* Host-computed fp32 scalars of one b200mix_unipc_step (see there). */
typedef struct {
  float alpha_t, sigma_t;       /* convert_model_output at the current sigma (_sigma_to_alpha_sigma_t) */
  float A_c, K_c, E_c, rc_last; /* UniC: sigma_t/sigma_s0, alpha_t*h_phi_1, alpha_t*B_h, rhos_c[-1] */
  float rc[2], rk_c[2];         /* UniC history terms k = 0, 1: rhos_c[k], rks[k] */
  float A_p, K_p, E_p;          /* UniP: sigma_t/sigma_s0, alpha_t*h_phi_1, alpha_t*B_h */
  float rp[2], rk_p[2];         /* UniP history terms k = 0, 1: rhos_p[k], rks[k] */
} b200mix_unipc_coeffs;

/* UniPCMultistepScheduler.step with predict_x0 = True, solver_type bh1 / bh2, orders 1-3
 * (scheduling_unipc_multistep.py:720-804, convert_model_output :368-437, UniC :567-701, UniP :438-565), one launch,
 * fp32 state, one rounding per operation in this order (c = *coeffs):
 *   m  = m_u + g*(m_c - m_u)   (m_c NULL => m = m_u); m_u, m_c bf16 or fp32 (m_fp32)
 *   m0 = x0 of m at the uncorrected sample x, as b200mix_ddim_step_ex with sa_t = c.alpha_t, sb_t = c.sigma_t
 *        (prediction_type 0 epsilon, 1 sample, 2 v_prediction)
 *   UniC (last_sample != NULL; m_prev = the previous step's m0):
 *     res = c.rc_last*(m0 - m_prev);  corr = sum over present k of c.rc[k]*((hc_k - m_prev)/c.rk_c[k]);
 *     res = corr + res (only if some hc_k is present);  x_c = (c.A_c*last_sample - c.K_c*m_prev) - c.E_c*res
 *   else x_c = x
 *   UniP: x_next = c.A_p*x_c - c.K_p*m0;  pred = sum over present k of c.rp[k]*((hp_k - m0)/c.rk_p[k]);
 *     x_next = x_next - c.E_p*pred (only if some hp_k is present)
 * Each sum runs over k = 0, 1 in that order: acc = t_0, then acc = acc + t_1. hc0 / hc1 are the x0 of the steps
 * before m_prev (most recent first), hp0 / hp1 those before m0 (hp0 = m_prev); a NULL pointer is an absent term and
 * is not read. Writes m_out = m0 (the history ring's next entry), x_corr = x_c (the next step's last_sample) and
 * x_next. Every tensor is fp32 with x's element count except m_u / m_c. x_next may alias x and x_corr may alias
 * last_sample; m_out aliases none of the inputs. */
int b200mix_unipc_step(const void* m_u, const void* m_c, int32_t m_fp32, float guidance, const float* x,
                       const float* last_sample, const float* m_prev, const float* hc0, const float* hc1,
                       const float* hp0, const float* hp1, float* x_next, float* x_corr, float* m_out, int64_t n,
                       int32_t prediction_type, const b200mix_unipc_coeffs* coeffs, void* stream);

/* DPMSolverMultistepScheduler.step for "dpmsolver++" / midpoint / epsilon prediction ("DPM-Solver++ 2M",
 * scheduling_dpmsolver_multistep.py:801-873), fused with the CFG combine, fp32 state:
 *   x0 = (x - sigma_cur*eps) / alpha_cur                                   (convert_model_output, :446-453)
 *   m_prev == NULL: x_next = A*x - C*x0                                     (first order, :548-553)
 *   else          : x_next = A*x - C*x0 - halfC*(inv_r0*(x0 - m_prev))      (second order midpoint, :633-640)
 * m_out receives x0 (next step's m_prev). The scalars A = sigma_t/sigma_s0, C = alpha_t*(exp(-h) - 1), halfC = 0.5*C,
 * inv_r0 = 1/r0 are computed on the host in fp32 like the reference's 0-d tensors; every operation is rounded
 * individually in the reference's order. */
int b200mix_dpmpp_2m_step(const void* eps_u, const void* eps_c, int32_t eps_fp32, float guidance, const float* x,
                          const float* m_prev, float* x_next, float* m_out, int64_t n, float sigma_cur, float alpha_cur,
                          float A, float C, float halfC, float inv_r0, void* stream);

/* The ancestral noise z of b200mix_ddim_eta_step and b200mix_dpmpp_2m_sde_step is noise[i] (fp32, x's element count)
 * or, with noise NULL, the Philox stream of b200mix_iddpm_step and b200mix_euler_ancestral_step keyed by
 * (seed, step): element group g = elements 4g .. 4g+3 takes the four normals of
 * philox4x32_10(counter = (step, g mod 2^32, g div 2^32, 0), key = (seed mod 2^32, seed div 2^32)), fp64 Box-Muller as
 * written at b200mix_iddpm_step. */

/* DDIMScheduler.step with eta > 0 (scheduling_ddim.py:410-475), fused with the CFG combine, fp32 state, one rounding
 * per operation in this order:
 *   m = m_u + g*(m_c - m_u)   (m_c NULL => m = m_u); m_u, m_c bf16 or fp32 (m_fp32)
 *   x0, eps from m as in b200mix_ddim_step_ex (prediction_type 0 epsilon, 1 sample, 2 v_prediction)
 *   clip_sample_range > 0: x0 = clip(x0, -range, range)                                  (:446-452)
 *   use_clipped_model_output != 0: eps = (x - sa_t*x0)/sb_t, from the clipped x0          (:449-451)
 *   x_prev = (sa_p*x0 + sb_p*eps) + std_dev_t*z                                           (:454-472)
 * The host computes in fp32, in the reference's order, std_dev_t = eta * variance^0.5 and
 * sb_p = (1 - alpha_prod_t_prev - std_dev_t^2)^0.5. z: see above. x_prev may alias x. */
int b200mix_ddim_eta_step(const void* m_u, const void* m_c, int32_t m_fp32, float guidance, const float* x,
                          const float* noise, float* x_prev, int64_t n, float sqrt_alpha_t, float sqrt_beta_t,
                          float sqrt_alpha_prev, float sqrt_beta_prev, float std_dev_t, int32_t prediction_type,
                          float clip_sample_range, int32_t use_clipped_model_output, uint64_t seed, int64_t step,
                          void* stream);

/* DPMSolverMultistepScheduler.step for "sde-dpmsolver++" / midpoint / epsilon prediction ("DPM-Solver++ 2M SDE",
 * scheduling_dpmsolver_multistep.py:802-880), fused with the CFG combine, fp32 state, one rounding per operation in
 * this order:
 *   x0 = (x - sigma_cur*eps) / alpha_cur                                   (convert_model_output, :446-453)
 *   x_next = A*x + B*x0                                                     (first order, :561-567)
 *   m_prev != NULL: x_next = x_next + halfB*(inv_r0*(x0 - m_prev))          (second order midpoint, :666-674)
 *   x_next = x_next + N*z
 * with A = sigma_t/sigma_s0*exp(-h), B = alpha_t*(1 - exp(-2h)), halfB = 0.5*B, inv_r0 = 1/r0 and
 * N = sigma_t*sqrt(1 - exp(-2h)) computed on the host in fp32 like the reference's 0-d tensors. m_out receives x0 (the
 * next step's m_prev). z: see above. x_next may alias x; m_out aliases none of the inputs. */
int b200mix_dpmpp_2m_sde_step(const void* eps_u, const void* eps_c, int32_t eps_fp32, float guidance, const float* x,
                              const float* noise, const float* m_prev, float* x_next, float* m_out, int64_t n,
                              float sigma_cur, float alpha_cur, float A, float B, float halfB, float inv_r0, float N,
                              uint64_t seed, int64_t step, void* stream);

/* SD3 / DiT patchify: x NCHW [B,C,H,W] (fp32|bf16) -> rows [B*(H/p)*(W/p), C*p*p] bf16 with the column order
 * (c, ph, pw) of a flattened Conv2D weight [D,C,p,p] (PatchEmbed.proj, embeddings.py:143-150), and its inverse for
 * the output head: rows [B*h*w, p*p*C] in (ph, pw, c) order -> NCHW [B,C,h*p,w*p] (transformer_sd3.py:350-356). */
int b200mix_patchify(const void* x, int32_t x_fp32, void* y, int64_t B, int64_t C, int64_t H, int64_t W, int32_t p,
                     void* stream);
int b200mix_unpatchify(const void* x, void* y, int32_t y_fp32, int64_t B, int64_t C, int64_t h, int64_t w, int32_t p,
                       void* stream);

/* Row gather / scatter on bf16 matrices with int64 device indices: the token-embedding lookup and the
 * `inputs_embeds[image_mask] = image_embeds` merge of Qwen2-VL (modeling_qwen2_vl.py:1443,1449-1452). dim % 8 == 0. */
int b200mix_gather_rows(const void* table, const int64_t* ids, void* out, int64_t n, int64_t dim, void* stream);
int b200mix_scatter_rows(const void* src, const int64_t* idx, void* dst, int64_t n, int64_t dim, void* stream);

/* ---- Open-Sora STDiT2 helpers (ppdiffusers/examples/Open-Sora/models) ----------------------------------------- */

/* out[b,g,:] = x[b,:] + table[g,:] (fp32): scale_shift_table[None] + t.reshape(B,6,C), stdit/stdit2.py:121-126. */
int b200mix_broadcast_add(const float* x, const float* table, float* out, int64_t B, int64_t G, int64_t N,
                          void* stream);
/* In-place RMSNorm over the first d channels of every head of x[rows, H, ld_head] (q_norm / k_norm = LlamaRMSNorm,
 * layers/blocks.py:46-68,214). */
int b200mix_head_rmsnorm_inplace(void* x, int64_t rows, int64_t H, int64_t d, int64_t ld_row, int64_t ld_head,
                                 const float* weight, float eps, void* stream);
/* Temporal self-attention of STDiT2Block (stdit2.py:160-171; Attention.forward, blocks.py:200-241): sequences of
 * length T <= 32 along the frame axis of the token-major qkv buffer [B, T, S, 3, H, d] (row = (b*T+t)*S+s), with
 * interleaved-pair RoPE (cos/sin fp32 [T, d/2], blocks.py:566-591) and optional q/k RMSNorm, out [B, T, S, H*d].
 * Even d <= 128; row strides ld_row >= 3*H*d and ld_out >= H*d, both even, on 4-byte aligned buffers. */
int b200mix_small_attention(const void* qkv, void* out, int64_t B, int64_t T, int64_t S, int64_t H, int64_t d,
                            int64_t ld_row, int64_t ld_out, const float* rope_cos, const float* rope_sin,
                            const float* q_norm_w, const float* k_norm_w, float eps, float scale, void* stream);
/* PatchEmbed3D with patch (1,p,p) as a row gather (blocks.py:94-164) and STDiT2.unpatchify (stdit2.py:450-474):
 * x [B,C,T,H,W] -> rows [B*T*(H/p)*(W/p), C*p*p] bf16;  rows [B*T*h*w, p*p*C] -> fp32 [B,C,T,h*p,w*p]. */
int b200mix_patchify3d(const void* x, int32_t x_fp32, void* y, int64_t B, int64_t C, int64_t T, int64_t H, int64_t W,
                       int32_t p, void* stream);
int b200mix_unpatchify3d(const void* x, float* y, int64_t B, int64_t C, int64_t T, int64_t h, int64_t w, int32_t p,
                         void* stream);

/* fp32 <-> bf16 casts (round-to-nearest-even). */
int b200mix_cast(const void* x, void* y, int64_t n, int32_t x_fp32, int32_t y_fp32, void* stream);

/* Rotary embedding applied in place on x (token stride ld_tok, head stride ld_head, first D dims of each head
 * rotated; bf16, rotate_half convention, fp32 math) with per-token cos/sin fp32 [T, D] (apply_rotary_pos_emb_vision, modeling_qwen2_vl.py:227-238; M-RoPE tables are gathered on the
 * host side by the shim exactly as apply_multimodal_rotary_pos_emb :179-224 does). */
int b200mix_rope_inplace(void* x, int64_t T, int64_t H, int64_t D, int64_t ld_tok, int64_t ld_head, const float* cos,
                         const float* sin, void* stream);

/* Single-token decode step, one launch per layer for what Qwen2VLAttention.forward does between the qkv projection and
 * the attention (modeling_qwen2_vl.py:573-596: apply_multimodal_rotary_pos_emb on q and k, then the cache append):
 * qkv bf16 [B, (heads + 2 * kv_heads) * D] (row stride ld_row): the q heads are rotated in place, the k heads are rotated
 * into row rows[b] of cache_k, the v heads are copied into row rows[b] of cache_v (caches bf16 [*, kv_heads * D];
 * rows int64 [B] on the device, so the step is CUDA-graph capturable); cos / sin fp32 [B, D]. */
int b200mix_decode_rope_cache(void* qkv, int64_t ld_row, int64_t B, int64_t heads, int64_t kv_heads, int64_t D,
                              const float* cos, const float* sin, const int64_t* rows, void* cache_k, void* cache_v,
                              void* stream);

/* ---- Token sampling (PaddleNLP GenerationMixin.greedy_search / sample, generation/utils.py:1028-1271) ------------- */

/* One generation step for B rows of fp32 logits (row b at logits + b * ld, V <= 2^20 columns), one CTA per row:
 *   1. repetition penalty (logits_process.py:104-110): l = l < 0 ? l * penalty : l / penalty for every id whose bit is
 *      set in the row's presence bitmap (uint32 [B, ceil(V / 32)], bit i of word i / 32);
 *   2. do_sample == 0: argmax of the penalised logits, lowest id on ties (temperature, top_k, top_p are ignored);
 *   3. do_sample != 0: p = softmax(l / temperature) in fp32 (IEEE division, accurate expf); top_k > 0 keeps
 *      p >= the k-th largest p (ties kept); top_p < 1 then keeps, in order of descending p with lower ids first among
 *      equal p, every id whose preceding mass is <= top_p (the top-k output is not renormalised; the first id is always
 *      kept); masses are summed as floor(p * 2^48) integers. Draw: Philox4x32-10 with key = seed and counter =
 *      (step, b, 0, 0), u = (x0 >> 8) * 2^-24; the token is the first kept id, in ascending id order, whose inclusive
 *      prefix mass exceeds u * (kept mass);
 *   4. (utils.py:1239-1259) a row already finished emits pad_id instead; finished[b] |= (token in eos_ids). The token
 *      is written to out[b * ld_out + step] (when step < max_new) and to next_ids[b], and its presence bit is set.
 * state (uint64 [4], zeroed before the first step): [0] = step, [1] = arrival counter (left at 0), [2] = 1 once every
 * row has finished, [3] = the step at which the last row finished. The kernel advances state[0], so the call can be
 * replayed in a CUDA graph. finished int32 [B]; eos_ids int64 [n_eos] (n_eos = 0: rows never finish); pad_id in
 * [0, V) when n_eos > 0. Requires temperature > 0, 0 < top_p <= 1, top_k >= 0, penalty > 0; 4-byte aligned logits /
 * presence / finished and 8-byte aligned state / out / next_ids / eos_ids. */
int b200mix_sample_tokens(const float* logits, int64_t ld, int64_t B, int64_t V, uint32_t* presence, int32_t* finished,
                          uint64_t* state, int64_t* out, int64_t ld_out, int64_t max_new, int64_t* next_ids,
                          const int64_t* eos_ids, int32_t n_eos, int64_t pad_id, int32_t do_sample, float temperature,
                          int32_t top_k, float top_p, float penalty, uint64_t seed, void* stream);

/* ---- Beam search (PaddleNLP GenerationMixin.beam_search, generation/utils.py:1484-1649) -------------------------- */

/* Device state of one beam-search call over B items of nb beams (rows = B * nb, row b * nb + j is beam j of item b).
 * Every buffer lives on the device; the step kernel reads and updates them, so a call can be replayed in a CUDA graph. */
typedef struct b200mix_beam_state {
  uint64_t* state;      /* [4] zeroed before step 0: [0] step, [1] arrival counter (left at 0), [2] 1 once every item is
                           done, [3] generated cache positions the following b200mix_kv_reorder moves (0: none,
                           also after the selection at step max_new - 1, whose cache no decode step reads) */
  int64_t* next_ids;    /* [rows] the chosen token per beam slot (what the next decode step embeds) */
  float* beam_scores;   /* [rows] running beam scores: 0 for beam 0, -1e6 for the others before step 0 (:1523-1526) */
  int64_t* tokens;      /* [max_new, rows] token chosen per slot at each step */
  int32_t* parents;     /* [max_new, rows] parent beam (within the item) of each slot at each step */
  double* hyp_score;    /* [B, nb] BeamHypotheses in insertion order: score (GNMT length penalty applied), */
  int32_t* hyp_step;    /* [B, nb]   number of generated tokens of the hypothesis (the step its eos was chosen), */
  int32_t* hyp_slot;    /* [B, nb]   beam slot whose history it ends, at that step */
  int32_t* hyp_count;   /* [B] entries in use */
  double* hyp_worst;    /* [B] worst_score, 1e6 before step 0 (:107) */
  int32_t* done;        /* [B] BeamSearchScorer._done */
  uint32_t* presence;   /* [2, rows, ceil(V / 32)] ping-pong bitmaps of the ids in each beam (buffer step & 1 is read,
                           the other written); NULL when penalty == 1 */
} b200mix_beam_state;

/* Bytes of the scratch buffer b200mix_beam_search_step needs for B items of nb beams over V tokens (into *bytes). */
int b200mix_beam_search_workspace_size(int64_t B, int64_t nb, int64_t V, int64_t* bytes);

/* One beam-search step (beam_search :1555-1621 with BeamSearchScorer.process :196-262 and BeamHypotheses :98-143) for
 * fp32 logits of B * nb rows (row r at logits + r * ld):
 *   1. score = log(exp(x - max) / sum) in fp32 (:1561-1562), repetition penalty (logits_process.py:104-110: score < 0 ?
 *      score * penalty : score / penalty on the ids present in the beam), + the running beam score (:1564);
 *   2. diversity_rate == 0: the item's top 2 * nb of its nb * V scores (:1569-1574); diversity_rate > 0: each row's top
 *      2 * nb, minus rank * diversity_rate (rank 1 .. 2 * nb, fp32), top 2 * nb of those (:1576-1598), whose
 *      undiversified scores go on. Ties: lower flat index (beam * V + token, or beam * 2 * nb + rank - 1) first;
 *   3. process in fp64: an eos_id candidate at rank < nb adds a hypothesis with score / ((step + 5) / 6)^length_penalty,
 *      one at rank >= nb is skipped, any other candidate fills the next slot; a done item emits pad_id, score 0, parent
 *      0; is_done with early_stopping or worst_score >= best candidate / ((step + 5) / 6)^length_penalty.
 * Writes next_ids, beam_scores, column `step` of tokens / parents, the hypothesis store, done, the child presence
 * bitmaps and advances state (steps at or past max_new, or after every item is done, change nothing but state[3]).
 * Scores are rounded after every operation (no fused multiply-add), as the reference rounds them.
 * eos_id = -1: no eos. Requires 2 <= nb <= 16, 2 * nb <= V <= 2^20, penalty > 0, finite diversity_rate >= 0 and
 * length_penalty, pad_id in [0, V), the workspace of b200mix_beam_search_workspace_size (16-byte aligned). */
int b200mix_beam_search_step(const float* logits, int64_t ld, int64_t B, int64_t nb, int64_t V,
                             const b200mix_beam_state* st, void* workspace, int64_t workspace_bytes, int64_t max_new,
                             int64_t eos_id, int64_t pad_id, float penalty, float diversity_rate, double length_penalty,
                             int32_t early_stopping, void* stream);

/* reorder_cache (:1480-1482, index_select of every cache tensor by the chosen parents) for the generated region only,
 * in place, all layers in one launch. layer_kv: device array [2 * n_layers] of bf16 cache bases (K_0, V_0, K_1, ...),
 * each [B * nb, max_len, row_elems]. Moves positions [S, S + state[3]) of every beam whose parent (column state[0] - 1 of
 * parents [max_new, B * nb]) is not itself; items with done[b] set are left alone. Prompt positions [0, S) are never
 * touched: they are the same in every beam of an item. Launched for max_new positions (CTAs past state[3] exit), so it
 * can be captured once and replayed. Requires row_elems a multiple of 8, nb * row_elems * 2 <= 32768 and every base in
 * layer_kv 16-byte aligned (rows are moved as 16-byte vectors; the table lives on the device, so this is not checked). */
int b200mix_kv_reorder(void* const* layer_kv, int64_t n_layers, int64_t B, int64_t nb, int64_t max_len,
                       int64_t row_elems, int64_t S, int64_t max_new, const int32_t* parents, const uint64_t* state,
                       const int32_t* done, void* stream);

/* ---- LoRA weight update (LoRACompatibleLinear._fuse_lora / LoRACompatibleConv._fuse_lora,
 * ppdiffusers/models/lora.py:117-165, :312-362) -------------------------------------------------------------------
 * One target: a device-layout bf16 weight, or a row slice of a batched one. For n < N, k < K:
 *   out[n, k] = bf16(base[n, k] + col_scale[k] * sum_j U[n, j] * D[j, k])     (col_scale null: 1)
 *   colsum[n] = colsum_base[n] + sum_k (out[n, k] - base[n, k])                (only when colsum is set)
 * base is the snapshot of the weight as loaded, so the result never depends on earlier LoRA states. An element (or a
 * colsum) whose update is exactly zero is copied from base bit for bit. U, D: fp32, row-major, contiguous. */
typedef struct b200mix_lora_item {
  void* out;                /* bf16 [N, ld_out] */
  const void* base;         /* bf16 [N, ld_base], must not overlap out */
  const float* U;           /* [N, R] */
  const float* D;           /* [R, K] */
  const float* col_scale;   /* [K] or null */
  float* colsum;            /* [N] or null */
  const float* colsum_base; /* [N]; required exactly when colsum is set */
  int64_t ld_out, ld_base, N, K, R;
} b200mix_lora_item;

#define B200MIX_LORA_MAX_RANK 512

int b200mix_lora_workspace_size(int32_t n_items, int64_t* bytes);

/* Rebuilds every item's target in one persistent launch over (item, 64-row tile) work units: U @ D on tensor cores
 * (mma.sync m16n8k8 tf32, operands rounded to tf32 with rna, fp32 accumulation over j in order), then one fp32 add
 * and one bf16 rounding per element. Each element and each colsum is produced by one thread / warp in a fixed order,
 * so the result is deterministic. items: host array, copied into `workspace` (16-byte aligned, at least
 * b200mix_lora_workspace_size bytes) on `stream`. Requires R a positive multiple of 8 and <= B200MIX_LORA_MAX_RANK,
 * K a positive multiple of 8, ld_out / ld_base multiples of 8 and >= K, out / base / U / D 16-byte aligned. */
int b200mix_lora_apply(const b200mix_lora_item* items, int32_t n_items, void* workspace, int64_t workspace_bytes,
                       void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200MIX_H_ */
