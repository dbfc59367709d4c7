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

enum { B200MIX_ACT_NONE = 0, B200MIX_ACT_SILU = 1, B200MIX_ACT_GELU_ERF = 2, B200MIX_ACT_GELU_TANH = 3, B200MIX_ACT_QUICK_GELU = 4 };
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
   * mean / variance are rebuilt in fp32 (E[x^2] - mean^2), accurate to ~1e-7 * mean^2 / var, i.e. below the bf16
   * resolution of h for every row bf16 can represent. Callers with rows outside that range keep b200mix_layernorm. */
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
 * y bf16 [B,H,W,C1+C2]. Two launches: per-CTA partial statistics in double, reduced in a fixed order by the last
 * CTA of each batch element (bit-reproducible), then apply. `stats` = scratch of at least
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

/* y = act(x) elementwise for bf16/fp32 vectors (SiLU on temb, resnet.py:772-776). */
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

/* y = a + r for an NHWC bf16 activation a [B,H,W,C]; r is NHWC bf16 (r_nchw = 0) or the caller's NCHW fp32|bf16 tensor
 * (r_nchw = 1). The ControlNet / T2I-Adapter residual adds of UNet2DConditionModel.forward:
 * down_block_additional_residuals, mid_block_additional_residual, down_intrablock_additional_residuals
 * (unet_2d_condition.py:1109-1155; unet_2d_blocks.py:1211-1213). y may alias a. */
int b200mix_add_residual_nhwc(const void* a, const void* r, int32_t r_fp32, int32_t r_nchw, void* y, int64_t B, int64_t C,
                              int64_t H, int64_t W, void* stream);

/* Fused classifier-free-guidance combine + DDIM step (eta = 0, epsilon prediction), fp32 state:
 *   eps = eps_u + g*(eps_c - eps_u)  (pipeline_stable_diffusion.py:882-884; eps_c NULL => eps = eps_u)
 *   x0 = (x - sqrt_beta_t*eps) / sqrt_alpha_t ; x_prev = sqrt_alpha_prev*x0 + sqrt_beta_prev*eps
 * The four scalars are computed on the host by the scheduler, bit-exactly as scheduling_ddim.py:410-457 does, and
 * applied here with the same operation order in fp32. eps inputs bf16 or fp32 (eps_fp32). */
int b200mix_ddim_step(const void* eps_u, const void* eps_c, int32_t eps_fp32, float guidance, const float* x,
                      float* x_prev, int64_t n, float sqrt_alpha_t, float sqrt_beta_t, float sqrt_alpha_prev,
                      float sqrt_beta_prev, void* stream);

/* DDIM step for every prediction_type (0 = epsilon, 1 = sample, 2 = v_prediction; scheduling_ddim.py:424-443) with
 * optional clip_sample (clip_sample_range > 0 clips the predicted x0, :446-452; <= 0: off), eta = 0, fused CFG combine:
 *   epsilon: x0 = (x - sb_t*m)/sa_t, eps = m;  sample: x0 = m, eps = (x - sa_t*x0)/sb_t;
 *   v_prediction: x0 = sa_t*x - sb_t*m, eps = sa_t*m + sb_t*x;   x_prev = sa_p*clip(x0) + sb_p*eps. */
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
 * interleaved-pair RoPE (cos/sin fp32 [T, d/2], blocks.py:566-591) and optional q/k RMSNorm, out [B, T, S, H*d]. */
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

#ifdef __cplusplus
}
#endif
#endif /* B200MIX_H_ */
