/*
 * vista_b200 — C-ABI of the H100-native (sm_90a) Vista denoising hot path.
 *
 * The reference (OpenDriveLab/Vista) is pure Python and has no FFI of its own; every kernel it runs
 * is a library call reached through PyTorch.  Each entry point below replaces one family of those
 * library call sites (reference file:line given per function, paths relative to the reference
 * root).  The binding a reference maintainer would add is a ctypes stub — see INTEGRATION.md.
 *
 * Conventions
 *   - plain C: raw device pointers, sizes, a cudaStream_t passed as void*; no torch types.
 *   - activations are TOKEN-MAJOR fp16: [tokens, channels] with an explicit row stride in
 *     elements ("ld").  A (B,C,H,W) reference tensor is stored as tokens = (b*H + h)*W + w,
 *     i.e. NHWC; the "(b t) s c" token layout of vwm/modules/video_attention.py:116 is the
 *     same memory.  Row strides let a tensor live inside a wider buffer (skip-concat, q|k|v).
 *   - every call is asynchronous on `stream`; the library keeps no global mutable state
 *     besides the last-error string.  Returns 0 on success, non-zero on error
 *     (message via b200v_last_error()).  There is NO CPU fallback.
 */
#ifndef VISTA_B200_H
#define VISTA_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

const char* b200v_last_error(void);
int b200v_version(void);
/* Fills sm count / compute capability of the current device. */
int b200v_device_info(int32_t* sm_count, int32_t* cc_major, int32_t* cc_minor);

/* ------------------------------------------------------------------------------------------------
 * Tap-GEMM on wgmma tensor cores (TMA-fed, register accumulators, fused epilogue).
 *   out[token, n] = epilogue( sum_{tap, c} A[token shifted by tap, c] * Wt[n, tap*cin + c] )
 * One kernel serves
 *   nn.Linear ................ vwm/modules/attention.py:275-282,88,120,579,603 (ntaps = 1)
 *   nn.Conv2d 3x3 pad 1 ...... vwm/modules/diffusionmodules/openaimodel.py:198,232,84; model.py:104,109,60
 *   nn.Conv2d 1x1 ............ openaimodel.py:241; model.py:114,152-155
 *   nn.Conv3d (3,1,1) ........ video_model.py:38-52; temporal_ae.py:25-37,83-88 (taps along frames)
 * Epilogue (fp32):  v = s_acc*(acc + bias[n]) + rowvec[(token/rv_div)%rv_mod, n];  v = act(v);
 *                   v += s_res1*res1[token,n] + s_res2*res2[token,n]
 *   act: 0 none, 1 SiLU, 2 GEGLU (value*gelu_erf(gate); weights/bias pre-permuted so a tile of
 *   tile_n columns holds tile_n/2 value columns followed by their gate columns; N counts the
 *   permuted columns, the output has N/2 columns) — vwm/modules/attention.py:85-93,
 *   3 GELU (erf form, nn.GELU() of the CLIP tower's mlp.c_fc; bias only, fp16 operands and output).
 * ---------------------------------------------------------------------------------------------- */
typedef struct b200v_gemm_desc {
  const void* a;        /* fp16/bf16 activations */
  int64_t lda;          /* row stride of A in elements (multiple of 8) */
  int64_t tokens;       /* number of A rows = NB*H*W */
  int32_t a_mode;       /* 0: linear (2-D), 1: image taps (4-D view c,w,h,b with zero padding), 2: image taps over the
                         * nearest-2x upsampled view of A — output pixel (f, y, x) of the NB x 2H x 2W result reads
                         * A pixel (f, floor((y + dh) / 2), floor((x + dw) / 2)), zero outside; the output has 4 tokens
                         * rows (token (f * 2H + y) * 2W + x).  The upsampled tensor is never written.  Epilogue: bias
                         * and fused statistics only (act 0, no rowvec / residuals / s_acc, fp16 operands and output) */
  int32_t W, H, NB;     /* a_mode 1: geometry of the view; a_mode 2: geometry of A (low resolution); a_mode 0: ignored */
  int32_t box_w, box_h, box_b; /* a_mode 1 / 2: token tile of A, box_w*box_h*box_b == 128 (a_mode 2: each box makes 4 tiles,
                                * one per output parity) */
  int32_t cin;          /* channels per tap (multiple of 64) */
  int32_t ntaps;        /* 1..9 */
  int32_t dh[9];        /* tap offsets along h and w */
  int32_t dw[9];
  const void* b;        /* weights [N, ntaps*cin], K contiguous, same dtype as A */
  int32_t N;            /* multiple of 8 */
  int32_t tile_n;       /* 32..256, multiple of 32 */
  int32_t bf16;         /* 0: fp16 operands, 1: bf16 operands */
  void* out;            /* fp16 (or fp32 if out_f32) [tokens, ldo] */
  int64_t ldo;
  int32_t out_f32;
  int32_t act;
  const float* bias;    /* [N] or NULL */
  const float* rowvec;  /* [rows, ld_rowvec] fp32 or NULL */
  int64_t ld_rowvec;
  int32_t rv_div, rv_mod;
  const void* res1;     /* same dtype as out (16-bit) or NULL */
  int64_t ld_res1;
  float s_res1;
  const void* res2;
  int64_t ld_res2;
  float s_res2;
  float s_acc;
  /* Optional: GroupNorm statistics of the output, fused into the epilogue (util.py:214-216 reads its input once more in
   * the reference; here the producer already has the values in registers).  stats != NULL: fp32 column partials — sum and
   * sum of squares of the stored values over each (128-token tile, 32-row quarter) — are written to
   * stats[((tile * 4 + quarter) * stats_ld + stats_col0 + n) * 2 + {0, 1}] for every output column n; b200v_groupnorm_
   * from_partials turns them into (mean, rstd).  Needs fp16 output, act 0, at most one residual, no rowvec with a
   * residual, and token tiles of 128 consecutive tokens (a_mode 0, or boxes of whole image rows / row segments). */
  float* stats;
  int64_t stats_ld;
  int32_t stats_col0;
  /* a_mode 1 only: the A view has h_pad extra rows of H before and after the H rows that produce output (extents
   * c, W, H + 2 h_pad, NB; `a` points at the first extra row).  Tap offsets are taken relative to the first OUTPUT row, so
   * a (3,1,1) convolution over frames reads its neighbours' boundary frames from the halo slots instead of zero padding:
   * the frame-sharded temporal convolution in ONE launch (openaimodel.py:190-193 across shards). */
  int32_t h_pad;
} b200v_gemm_desc;

int b200v_gemm(const b200v_gemm_desc* d, void* stream);

/* (mean, rstd) per (statistic, group) from the column partials b200v_gemm wrote (fixed summation order, fp64):
 * statistic s covers frames [s * frames_per_stat, (s + 1) * frames_per_stat), each of tokens_per_frame tokens
 * (a multiple of 128); mean_rstd [n_stats, groups, 2] fp32.  raw_sums (optional, [n_stats, groups, 2] fp64) receives
 * (sum, sum of squares) instead — the frame-sharded GroupNorm all-reduces those before finalising. */
int b200v_groupnorm_from_partials(const float* partials, int64_t stats_ld, int32_t n_stats, int32_t frames_per_stat,
                                  int32_t tokens_per_frame, int32_t C, int32_t groups, float eps, float* mean_rstd,
                                  double* raw_sums, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Spatial self-attention, head dim 64, non-causal:  softmax(Q K^T / 8) V  per (frame, head).
 * Replaces xformers.ops.memory_efficient_attention at vwm/modules/attention.py:401 (and the head
 * split / merge copies at :370-378, :409-414).  q/k/v are column slices of token-major buffers:
 * element (frame f, token t, head h, dim d) of q is q[(f*seq + t)*ld_q + h*64 + d].
 * ---------------------------------------------------------------------------------------------- */
/* Flash attention on wgmma (sm_90a): one 128-query tile per CTA, two consumer warpgroups of 64 query rows, K / V in a
 * 3-deep TMA ring, online softmax in registers, P fed to the P V MMA from registers.  The _v3 (short sequences) and _v7
 * (long sequences) entry points run the same kernel. */
int b200v_attention_spatial_v3(const void* q, int64_t ld_q, const void* k, int64_t ld_k, const void* v, int64_t ld_v,
                               void* out, int64_t ld_o, int32_t frames, int32_t seq, int32_t heads, void* stream);


int b200v_attention_spatial_v7(const void* q, int64_t ld_q, const void* k, int64_t ld_k, const void* v, int64_t ld_v,
                               void* out, int64_t ld_o, int32_t frames, int32_t seq, int32_t heads, void* stream);

/* Temporal self-attention over the T frames of each pixel (seq len T <= 32, head dim 64).
 * Replaces the batchified xformers call at vwm/modules/attention.py:384-399 reached from
 * vwm/modules/video_attention.py:127 and both "(b t) s c <-> (b s) t c" rearranges (:116,:140):
 * tokens stay in (b t) s order, the kernel strides over frames. */
int b200v_attention_temporal(const void* q, int64_t ld_q, const void* k, int64_t ld_k, const void* v, int64_t ld_v,
                             void* out, int64_t ld_o, int32_t nb, int32_t T, int32_t S, int32_t heads, void* stream);

/* Frame-sharded variant: queries / outputs are the Tq local frames (rows (b*Tq + t)*S + s), keys / values the T
 * frames of the whole clip whose row blocks start at token kv_frame_tok[b*T + t] of the k / v buffers (the
 * all-gathered K|V of every rank).  Replaces the same call sites when frames are sharded over GPUs. */
int b200v_attention_temporal_sharded(const void* q, int64_t ld_q, const void* k, int64_t ld_k, const void* v, int64_t ld_v,
                                     void* out, int64_t ld_o, int32_t nb, int32_t Tq, int32_t T, int32_t S, int32_t heads,
                                     const int64_t* kv_frame_tok, void* stream);

/* ------------------------------------------------------------------------------------------------
 * GroupNorm (32 groups) in two phases, fp32 partials / fp64 reduction, bit-reproducible:
 *   stats: per (frame, chunk of tokens, group) partial sums go to `partials`; the chunk length is chosen per
 *          shape and is never below b200v_groupnorm_chunk(), so
 *          frames * ceil(tokens_per_frame / b200v_groupnorm_chunk()) * groups * 2 doubles of scratch always
 *          suffice; the last block of each statistic
 *          (stat = frame / frames_per_stat, ticket in `counters`, which must be zero on first use and is
 *          left zero) reduces them in a fixed order and writes mean_rstd[stat, group, {mean, rstd}].
 *   apply: y = (x - mean) * rstd * gamma + beta, optional SiLU, fp16 out
 * frames_per_stat = 1 is the per-frame GroupNorm32 (vwm/modules/diffusionmodules/util.py:214-216),
 * frames_per_stat = T is the (C/32, T, H, W) statistic of the temporal ResBlock
 * (video_model.py:67-72 with openaimodel.py:195-199, dims=3).
 * ---------------------------------------------------------------------------------------------- */
int b200v_groupnorm_chunk(void);
/* the chunk length b200v_groupnorm_stats uses for this shape (exact scratch sizing) */
int b200v_groupnorm_chunk_for(int32_t frames, int32_t tokens_per_frame);
int b200v_groupnorm_stats(const void* x, int64_t ldx, int32_t frames, int32_t tokens_per_frame, int32_t C,
                          int32_t groups, int32_t frames_per_stat, float eps, double* partials, int32_t* counters,
                          float* mean_rstd, void* stream);
int b200v_groupnorm_apply(const void* x, int64_t ldx, void* y, int64_t ldy, int32_t frames, int32_t tokens_per_frame,
                          int32_t C, int32_t groups, int32_t frames_per_stat, const float* mean_rstd, const float* gamma,
                          const float* beta, int32_t silu, void* stream);

/* Frame-sharded mode (one clip spread over several GPUs): the temporal statistic spans frames held by other
 * ranks, so `b200v_groupnorm_sums` stops after the local fixed-order reduction and returns raw
 * sums[stat, group, {sum, sumsq}] (fp64); the caller adds the ranks' sums (NCCL) and calls
 * `b200v_groupnorm_finalize` with the global element count. */
int b200v_groupnorm_sums(const void* x, int64_t ldx, int32_t frames, int32_t tokens_per_frame, int32_t C, int32_t groups,
                         int32_t frames_per_stat, double* partials, int32_t* counters, double* sums, void* stream);
int b200v_groupnorm_finalize(const double* sums, int32_t n_stat_groups, double count, float eps, float* mean_rstd,
                             void* stream);

/* LayerNorm over C per token (eps 1e-5), optional fp32 row-vector added to the input first:
 *   y = LN(x + addvec[(token/av_div)%av_mod, :]).   nn.LayerNorm at attention.py:488-490,
 * video_attention.py:49,76,97,98; the add is `x_mix = x + emb` (video_attention.py:284-285). */
int b200v_layernorm(const void* x, int64_t ldx, void* y, int64_t ldy, int64_t tokens, int32_t C, const float* gamma,
                    const float* beta, float eps, const float* addvec, int64_t ld_addvec, int32_t av_div,
                    int32_t av_mod, void* stream);

/* Direct convolutions for the two thin ends of the UNet / decoder (CUDA cores; < 0.1 % of FLOPs):
 *   conv3x3_small_cin : Cin <= 8, e.g. input_blocks.0 (video_model.py:189), decoder conv_in (model.py:604)
 *   conv3x3_small_cout: Cout <= 4, e.g. out[2] (video_model.py:438), AE3DConv's Conv2d (temporal_ae.py:91) */
int b200v_conv3x3_small_cin(const void* x, int32_t cin, const float* w /* [cout,cin,3,3] */, const float* bias,
                            void* out, int64_t ldo, int32_t NB, int32_t H, int32_t W, int32_t cout, void* stream);
int b200v_conv3x3_small_cout(const void* x, int64_t ldx, int32_t cin, const float* w /* [cout,cin,3,3] */,
                             const float* bias, float* out /* [tokens, cout] fp32 */, int32_t NB, int32_t H, int32_t W,
                             int32_t cout, void* stream);

/* Data movement: stride-2 im2col for Downsample (openaimodel.py:129-136), nearest 2x upsample
 * (openaimodel.py:100; model.py:63). */
int b200v_im2col_s2(const void* x, int64_t ldx, void* out, int32_t NB, int32_t H, int32_t W, int32_t C, void* stream);
/* VAE-encoder Downsample (vwm/modules/diffusionmodules/model.py:69-83): pad right / bottom by one, stride 2, no other
 * padding: out[(b,ho,wo), tap*C + c] = x[b, 2ho+kh, 2wo+kw, c], Ho = (H-2)/2 + 1.  (Next row: the VAE encoder.) */
int b200v_im2col_s2_asym(const void* x, int64_t ldx, void* out, int32_t NB, int32_t H, int32_t W, int32_t C, void* stream);
int b200v_upsample2x(const void* x, int64_t ldx, void* out, int64_t ldo, int32_t NB, int32_t H, int32_t W, int32_t C,
                     void* stream);

/* Small fp32 helpers of the embedding path:
 *   timestep_embedding: out[i, :] = cos||sin(t[i] * freqs)   (util.py:141-165), fp16 out
 *   silu_f16: y = silu(x) fp32 -> fp16 (emb_layers' nn.SiLU, openaimodel.py:222-225)
 *   blend_emb: emb = e_cond*m + e_plain*(1-m) + label   (video_model.py:457-471) */
int b200v_timestep_embedding(const float* t, int32_t n, int32_t dim, float max_period, void* out_f16, int64_t ldo,
                             void* stream);
int b200v_blend_emb(const float* e_plain, const float* e_cond, const float* label, const float* mask, float* emb_f32,
                    void* silu_emb_f16, int32_t rows, int32_t dim, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Fused EDM / Euler sampler step around the UNet call (all fp32 state, NCHW latents (T,4,h,w)):
 *   prepare: x = x*(1-mask) + cond_frame*mask                       (sampling.py:105-106)
 *            unet_in[(2T),h,w,8] = [x*c_in(sigma) | concat]  fp16   (guiders.py:28-36, denoiser.py:33-35,
 *                                                                     wrappers.py:31), rows [uncond; cond]
 *            c_noise[2T] = 0.25*ln(sigma)                           (denoiser_scaling.py:58)
 *   update : D_u/c = net*c_out + x*c_skip; D = D_u + scale[t]*(D_c - D_u)   (guiders.py:23-26,68-74)
 *            x += (x - D)/sigma * (sigma_next - sigma)              (sampling_utils.py:46, sampling.py:85-88)
 *            and, when `final`, re-imposes the conditioning frames  (sampling.py:122-123)
 * sigma values are read from the device array `sigmas` at index *step_idx (device int); update
 * increments *step_idx so that a captured CUDA graph can be replayed for every step.
 *   update_2m: D as in update; then, with {a, b, c, e} = coefs[4 * *step_idx ..] (DPM-Solver++(2M),
 *            Lu et al. 2022, arXiv 2211.01095, Algorithm 2; a = s'/s, b = expm1(-h), h = ln(s/s'),
 *            c = 1 + 1/(2r), e = 1/(2r), r = h_prev/h; c = 1, e = 0 on a first-order row):
 *            x = a*x - b*(c*D - e*d_prev); d_prev = D             (d_prev is not read when e == 0)
 *            and, when `final`, re-imposes the conditioning frames
 *   update_action: action guidance (vista_b200.diffusion.ActionCFG, InstructPix2Pix eq. 3): D_img = the denoised value of
 *            row t of net_img (the conditional rows with the action slots of crossattn zeroed),
 *            D = D_u + scales[t]*(D_img - D_u) + action_scales[t]*(D_c - D_img); then the Euler step
 *            (coefs == d_prev == NULL) or the 2M step (both given), as in update / update_2m
 *   update_cond: the unguided step (guidance weight 1): net_c holds the T conditional rows only,
 *            D = c_skip*x + c_out*net_c; then the Euler step (coefs == d_prev == NULL) or the 2M step
 *            (both given, D written to d_prev), as in update_action
 * ---------------------------------------------------------------------------------------------- */
int b200v_sampler_prepare(float* x, const float* cond_frame, const float* mask,
                          const float* concat_u /* uncond rows (T,4,h,w) or NULL = zeros */,
                          const float* concat_c /* cond rows (T,4,h,w) or NULL = zeros */, const float* sigmas, const int32_t* step_idx,
                          void* unet_in_f16 /* [2T*h*w] rows of 8 fp16, row stride ld_in elements */, int64_t ld_in,
                          float* c_noise, int32_t T, int32_t h, int32_t w, void* stream);
int b200v_sampler_update(float* x, const float* net_out /* [2T*h*w, ld_net] fp32 token-major, 4 channels used */,
                         int64_t ld_net, const float* cond_frame, const float* mask, const float* scales /* [T] */, const float* sigmas, int32_t* step_idx,
                         int32_t num_steps, int32_t T, int32_t h, int32_t w, void* stream);
int b200v_sampler_update_2m(float* x, const float* net_out /* as in b200v_sampler_update */, int64_t ld_net,
                            const float* cond_frame, const float* mask, const float* scales /* [T] */,
                            const float* coefs /* [num_steps, 4] fp32 {a, b, c, e}, 16-byte aligned */,
                            float* d_prev /* (T,4,h,w) fp32, the previous step's D */, const float* sigmas,
                            int32_t* step_idx, int32_t num_steps, int32_t T, int32_t h, int32_t w, void* stream);
int b200v_sampler_update_action(float* x, const float* net_out /* as in b200v_sampler_update */, int64_t ld_net,
                                const float* net_img /* [T*h*w, ld_img] fp32 token-major, 4 channels used */,
                                int64_t ld_img, const float* cond_frame, const float* mask,
                                const float* scales /* [T] s_img */, const float* action_scales /* [T] s_act */,
                                const float* coefs /* as in update_2m, or NULL */, float* d_prev /* or NULL */,
                                const float* sigmas, int32_t* step_idx, int32_t num_steps, int32_t T, int32_t h,
                                int32_t w, void* stream);
int b200v_sampler_update_cond(float* x, const float* net_c /* [T*h*w, ld_net] fp32 token-major, 4 channels used */,
                              int64_t ld_net, const float* cond_frame, const float* mask,
                              const float* coefs /* as in update_2m, or NULL */, float* d_prev /* or NULL */,
                              const float* sigmas, int32_t* step_idx, int32_t num_steps, int32_t T, int32_t h,
                              int32_t w, void* stream);

/* VAE decoder helpers.
 *   softmax_rows : fp32 scores -> fp16 probabilities, one row per block (mid.attn_1 single-head d=512
 *                  attention, vwm/modules/diffusionmodules/model.py:158-170, done as GEMM-softmax-GEMM)
 *   time_mix_small: AE3DConv.time_mix_conv (3->3 channels, (3,1,1)), temporal_ae.py:83-97, writing NCHW
 *                  fp32 frames [out_frame0 + t]; frames with blend[t] != 0 are averaged with the existing
 *                  content and frames t < skip_frames are dropped — the 3-frame chunk-overlap rule of
 *                  DiffusionEngine.decode_first_stage (vwm/models/diffusion.py:166-170). */
int b200v_softmax_rows(const float* x, int64_t ld_in, void* y_f16, int64_t ld_out, int64_t rows, int32_t cols,
                       void* stream);
int b200v_time_mix_small(const float* x /* [T*HW, ldx] fp32, C channels used */, int64_t ldx,
                         const float* w /* [C,C,3] */, const float* bias,
                         float* out /* NCHW fp32 */, const int32_t* blend, int32_t T, int32_t HW, int32_t C,
                         int32_t out_frame0, int32_t skip_frames, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Callers' glue as device code (SURVEY.md 8f rows 2-4; csrc/glue.cu).
 *   time_mix_small_u8 : time_mix_small that ALSO stores every frame it produces the way the reference's output
 *       path does — clamp((x + 1) / 2, 0, 1) (sample_utils.py:374), 255 * s truncated to uint8, "t c h w -> t h w c"
 *       (sample_utils.py:96-126) — into out_u8 [frames, HW, C].  The fp32 NCHW `out` is only written for frames
 *       t >= keep_f32_from (the tail a later chunk blends with; < 0 = every frame) and read for blended frames.
 *   rollout_advance : between two rounds of the long-horizon rollout (sample_utils.py:318-365): optional
 *       sample[0] = z0 (first round, :336), samples_z[dst_frame0 + t] = sample[t] for t >= src_frame0 (:337,:362),
 *       filled = fill_latent(sample[-n_cond:], T, [0..n_cond-1]) (:350, :280-283; NULL = last round).
 *   ensemble_reward : reward_utils.py:318-337 — out2[0] = mean_i var_k(member_k[i]) (unbiased over the K members,
 *       fp32 per element as the reference, fp64 fixed-order sum), out2[1] = exp(-out2[0]).  members_dev = device
 *       array of K device pointers; partial >= b200v_ensemble_reward_scratch() doubles; ticket = zeroed uint32
 *       (self-resetting).
 * ---------------------------------------------------------------------------------------------- */
int b200v_time_mix_small_u8(const float* x, int64_t ldx, const float* w, const float* bias, float* out, uint8_t* out_u8,
                            const int32_t* blend, int32_t T, int32_t HW, int32_t C, int32_t out_frame0,
                            int32_t skip_frames, int32_t keep_f32_from, void* stream);
int b200v_rollout_advance(float* sample, const float* z0, float* samples_z, float* filled, int32_t T, int64_t frame_elems,
                          int32_t dst_frame0, int32_t src_frame0, int32_t n_cond, void* stream);
int b200v_ensemble_reward_scratch(void);
int b200v_ensemble_reward(const float* const* members_dev, int32_t K, int64_t n, double* partial, uint32_t* ticket,
                          float* out2, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Collectives of the frame-sharded step over NVLink peer memory (csrc/peer.cu; SURVEY.md 8e).  A "window" is device memory
 * of one rank that its peers map (CUDA IPC) and store into; flags inside the window order the traffic (system-scope
 * release / acquire), sequence numbers are device-resident counters bumped by the kernels, so the calls below are plain
 * stream-ordered launches that a CUDA graph can replay.
 *   peer_alloc / open / close / free : window lifetime; handle64 = 64-byte cudaIpcMemHandle_t to hand to the peers.
 *   peer_allreduce_f64 : data[n] (n <= b200v_peer_allreduce_max()) summed over `world` ranks in RANK ORDER (same bits on
 *       every rank).  windows_dev = device array [world] of window base pointers as mapped by THIS rank (own window at
 *       [rank]); slot_off / flag_off = byte offsets, identical on all ranks, of 2 * world * max doubles and 2 * 16 uint32.
 *   peer_put : `rows` rows of row_bytes (multiple of 16) from src (pitch src_pitch) to each of n_dst (<= 8) destinations
 *       (pitch dst_pitch), then flag[d] = next sequence number of `counter` (release, after a system fence; last block by
 *       `ticket`, a zeroed uint32 that resets itself).
 *   peer_wait : spin (one thread per flag, bounded) until the n LOCAL flags reach the next sequence number of `counter`.
 * ---------------------------------------------------------------------------------------------- */
int b200v_peer_alloc(int64_t bytes, void** ptr, void* handle64);
int b200v_peer_open(const void* handle64, void** ptr);
int b200v_peer_close(void* ptr);
int b200v_peer_free(void* ptr);
int b200v_peer_allreduce_max(void);
int b200v_peer_allreduce_f64(double* data, int32_t n, void* const* windows_dev, int64_t slot_off, int64_t flag_off, int32_t rank,
                             int32_t world, uint32_t* counter, void* stream);
int b200v_peer_put(const void* src, int64_t src_pitch, int64_t rows, int64_t row_bytes, void* const* dsts_dev, int64_t dst_pitch,
                   uint32_t* const* flags_dev, int32_t n_dst, uint32_t* counter, uint32_t* ticket, void* stream);
int b200v_peer_wait(const uint32_t* const* flags_dev, int32_t n, uint32_t* counter, void* stream);

/* ------------------------------------------------------------------------------------------------
 * CLIP ViT-H/14 image tower of the conditioner (FrozenOpenCLIPImageEmbedder, vwm/modules/encoders/modules.py:251-399;
 * csrc/clip.cu).  The linear layers, LayerNorms and the token assembly run on b200v_gemm / b200v_layernorm.
 *   clip_preprocess : x (n,3,H,W) fp32 NCHW in [-1, 1] -> out [n*257, ldo] fp16 patch rows of the patch-embedding GEMM:
 *       FrozenOpenCLIPImageEmbedder.preprocess (modules.py:293-305) = kornia.geometry.resize to 224 x 224 (bicubic,
 *       align_corners, Gaussian anti-alias blur when antialias and the image shrinks), (x + 1) / 2, CLIP mean / std;
 *       row b*257 + 1 + 16 py + px holds patch (py, px) of image b with K index c*196 + 14 dy + dx (the flattening of
 *       conv1.weight [width, 3, 14, 14]); row b*257 (the class-token slot) and columns 588 .. ldo-1 are zero, so the
 *       GEMM with a row vector (rv_mod 257) of class embedding + positional embedding yields the tower's input tokens.
 *       Arithmetic fp32; out_f32 = 1 stores fp32 rows instead of fp16.
 *   attention_d80   : softmax(Q K^T / sqrt(80)) V per (image, head), head width 80 (the tower's nn.MultiheadAttention);
 *       q / k / v element (image b, token t, head h, dim d) at q[(b*seq + t)*ld_q + h*80 + d] (column blocks of the fused
 *       in-proj output), merged-head output likewise.  fp32 softmax and accumulation.
 * ---------------------------------------------------------------------------------------------- */
int b200v_clip_preprocess(const float* x, int32_t n, int32_t H, int32_t W, int32_t antialias, void* out, int64_t ldo,
                          int32_t out_f32, void* stream);
int b200v_attention_d80(const void* q, int64_t ld_q, const void* k, int64_t ld_k, const void* v, int64_t ld_v, void* out,
                        int64_t ld_o, int32_t batch, int32_t seq, int32_t heads, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Sinusoidal scalar embedders of the conditioner (ConcatTimestepEmbedderND, vwm/modules/encoders/modules.py:402-425;
 * csrc/cond.cu).  One launch writes every slot of `table` for all `rows` into column slices of the fp32 output
 * [rows, ldo] (`vector`, or the action columns of `crossattn`): for slot s and value j of row r,
 *   out[r, dst_col + j*outdim + k]          = cos(values[r, value_col + j] * freqs[freq_off + k])   k < outdim/2
 *   out[r, dst_col + j*outdim + outdim/2 + k] = sin(...)                                            (util.py:155-162)
 * — the "(b d) d2 -> b (d d2)" layout of modules.py:420-422; an odd outdim has a zero last column.  `zero` slots are
 * written with zeros and read nothing (force_zero_embeddings, modules.py:152-153).  values: fp32 [rows, ld_values];
 * freqs: fp32 frequency table, computed on the host with the reference's expression.  Full-precision sincosf.
 * ---------------------------------------------------------------------------------------------- */
#define B200V_SINUSOID_MAX_SLOTS 16
typedef struct b200v_sinusoid_slot {
  int32_t value_col;     /* first column of this slot's values in `values` */
  int32_t num_features;  /* values per row */
  int32_t outdim;        /* embedding width per value */
  int32_t dst_col;       /* first output column */
  int32_t zero;          /* 1: write zeros */
  int32_t freq_off;      /* first of the outdim/2 frequencies in `freqs` */
} b200v_sinusoid_slot;
typedef struct b200v_sinusoid_table {
  int32_t n_slots;
  b200v_sinusoid_slot slot[B200V_SINUSOID_MAX_SLOTS];
} b200v_sinusoid_table;
int b200v_sinusoid_embed(const float* values, int64_t ld_values, int32_t rows, const b200v_sinusoid_table* table,
                         const float* freqs, float* out, int64_t ldo, void* stream);

/* Layout converters at the boundary: NCHW fp32 <-> token-major (NHWC) fp16/fp32. */
int b200v_nchw_to_tokens(const float* x, void* out_f16, int64_t ldo, int32_t NB, int32_t C, int32_t H, int32_t W,
                         void* stream);
int b200v_tokens_to_nchw(const void* x, int32_t x_is_f32, int64_t ldx, float* out, int32_t NB, int32_t C, int32_t H,
                         int32_t W, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Camera frames in (sample.py:174-201, load_img; csrc/ingest/ingest.cu).
 *   frames_u8_resize : T uint8 RGB frames (NHWC, src + t*frame_stride + y*row_stride + 3*x) -> out fp32 (T, 3, out_h,
 *       out_w) = Image.crop((crop_x, crop_y, crop_x + crop_w, crop_y + crop_h)).resize((out_w, out_h), LANCZOS), then
 *       ToTensor and x * 2 - 1 (u8 / 255.0f correctly rounded, * 2, - 1), bit for bit Pillow's 8-bit resampler.  Per
 *       axis the host's tables (vista_b200/ingest.py lanczos_tables): bounds [out][2] = (first input index within the
 *       crop, count), weights [out][ksize] int32 in 22-bit fixed point.  A pass whose size is unchanged is skipped, as
 *       Pillow skips it, and its tables may be NULL.  The horizontal pass runs first, over the cropped rows
 *       [y_first, y_first + y_rows) the vertical pass reads (all crop_h rows when the height is unchanged), into
 *       scratch (T, y_rows, out_w, 3) uint8 (unused, may be NULL, when the width is unchanged).  Two launches, no
 *       allocation.
 * ---------------------------------------------------------------------------------------------- */
int b200v_frames_u8_resize(const uint8_t* src, int64_t frame_stride, int64_t row_stride, int32_t T, int32_t src_h,
                           int32_t src_w, int32_t crop_x, int32_t crop_y, int32_t crop_w, int32_t crop_h, int32_t out_h,
                           int32_t out_w, const int32_t* xbounds, const int32_t* xweights, int32_t xksize,
                           const int32_t* ybounds, const int32_t* yweights, int32_t yksize, int32_t y_first,
                           int32_t y_rows, uint8_t* scratch, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VISTA_B200_H */
