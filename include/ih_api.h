/* libimagharmony_sm90.so -- C ABI of the H100-native SDXL / IMAGHarmony denoise hot path.
 *
 * The reference (muzishen/IMAGHarmony) has no FFI of its own: its operator boundary is the diffusers
 * attention-processor protocol (ip_adapter/attention_processor.py:364-371) and the nn.Module calls inside the
 * diffusers UNet it drives from ip_adapter/custom_pipelines.py:338-345.  Each entry point below names the reference
 * call site(s) whose arithmetic it replaces.  The Python host (imagharmony_b200/ops.py) binds these with ctypes.
 *
 * Conventions
 *   - all tensors are fp16 ("__half") device pointers unless stated; activations are NHWC / [rows, channels].
 *   - `stream` is a cudaStream_t passed as void*; nothing here allocates, synchronises or keeps state except an
 *     internally locked TMA-descriptor cache.
 *   - return 0 on success, <0 on error; ih_last_error() returns a thread-local description.
 */
#ifndef IH_API_H
#define IH_API_H

#ifdef __cplusplus
extern "C" {
#endif

#define IH_API_VERSION 2

/* epilogue flags for ih_gemm_f16 */
#define IH_EPI_NONE 0
#define IH_EPI_GEGLU 1 /* out[:, j] = (acc[:, j] + b[j]) * gelu_erf(acc[:, F + j] + b[F + j]),  N = 2F */
#define IH_EPI_SILU 2  /* out = silu(acc + bias) */
#define IH_EPI_GELU 4  /* out = gelu_erf(acc + bias) */
#define IH_EPI_QUICK_GELU 8 /* out = x * sigmoid(1.702 x), x = acc + bias  (CLIP-L text tower MLP, scope row f2) */
/* out = relu(alpha * acc + bias + residual).  Unlike SILU / GELU / QUICK_GELU, which act on acc + bias BEFORE the
 * residual is added, ReLU acts AFTER it: the tiny autoencoder's block output relu(conv(x) + x) is one launch.  Not
 * combinable with the other flags; ih_conv2d_scaled_f16 accepts it too.  NaN propagates as in torch.relu (NaN and +inf
 * pass through, negatives and -inf become 0; the sign of a zero is unspecified). */
#define IH_EPI_RELU 16

const char* ih_last_error(void);
int ih_version(void);
long long ih_launch_count(void); /* kernels launched by this library since the last reset */
void ih_launch_count_reset(void);

/* out[M,N] = epi(A[M,K] @ W[N,K]^T + bias[N] + rowbias[row / rows_per_group, N]) + residual[M,N]
 * Replaces nn.Linear: attention_processor.py:292,299-300,320 (AttnProcessor2_0 to_q/to_k/to_v/to_out),
 * :396,410-411,432-433,453 (IPAttnProcessor2_0 incl. to_k_ip/to_v_ip), and the diffusers proj_in/proj_out/FF/1x1
 * conv layers reached through custom_pipelines.py:338-345.  tile_n: 0 = auto, else 64/128/160/192/256 (384 and
 * 512 mean 192 and 256).  With IH_EPI_GEGLU tile_n counts the weight rows of a tile, value and gate halves together:
 * 128/192/256 (64/96/128 outputs per tile); the 192-row GEGLU tile cannot write stats_out.
 * tile_n = IH_TILE_PINGPONG forces the ping-pong kernel (128x128 tiles, one per MMA warpgroup; GEGLU: 64 outputs per
 * tile), which the automatic choice takes where it is faster.  It supports bias, LayerNorm folding and GEGLU only, and
 * its outputs are bitwise equal to the other tiles'. */
#define IH_TILE_PINGPONG 1
int ih_gemm_f16(const void* a, long long lda, const void* w, const void* bias, const void* rowbias,
                int rows_per_group, long long ld_rowbias, const void* residual, long long ldr, void* out,
                long long ldo, int M, int N, int K, int epilogue, int tile_n, void* stream);

/* ih_gemm_f16 with LayerNorm folded in (BasicTransformerBlock norm1/2/3 -> attn / FF projections).
 *   stats_out != NULL : additionally write, per output row, (sum, sum of squares) of the fp16 values stored as
 *                       float [ceil(N/64), M, 2]: partial sums whose total over slots is the row's (one writer per
 *                       slot, every slot written; deterministic).  160-column tiles (tile_n = 160, or the automatic
 *                       choice) need N % 320 == 0 here; the automatic choice respects that.
 *   ln_stats  != NULL : `a` holds the RAW (un-normalised) rows; `w` is the weight pre-multiplied by the LayerNorm gamma
 *                       with every row centred (w[n,k] = W[n,k] gamma[k] - mean_k(W[n,:] gamma)), so that
 *                       a w^T = (a - mean(a)) (W gamma)^T; `bias` = W beta + b.  The epilogue applies
 *                       out = rstd[m] * acc + bias[n], rstd rebuilt from the producer's slabs
 *                       ln_stats [ln_slabs, M, 2] over the K features with epsilon ln_eps. */
int ih_gemm_ln_f16(const void* a, long long lda, const void* w, const void* bias, const void* rowbias,
                   int rows_per_group, long long ld_rowbias, const void* residual, long long ldr, void* out,
                   long long ldo, int M, int N, int K, int epilogue, int tile_n, const void* ln_stats, int ln_slabs,
                   float ln_eps, void* stats_out, void* stream);

/* out = epi(alpha * (A W^T) + bias) + residual: ih_gemm_f16 with an output scale.  Used by the VAE decoder's SCALED
 * RESIDUAL STREAM (scope row f1): the reference upcasts the SDXL VAE to fp32 because its activations overflow fp16
 * (custom_pipelines.py:366-371); here the residual stream is stored as 2^-k * x (GroupNorm is scale-invariant, every
 * conv / linear that writes the stream scales its output and bias by 2^-k), which is exact in real arithmetic. */
int ih_gemm_scaled_f16(const void* a, long long lda, const void* w, const void* bias, const void* residual,
                       long long ldr, void* out, long long ldo, int M, int N, int K, int epilogue, float alpha,
                       void* stream);

/* One-shot hint for the NEXT ih_gemm_* / ih_conv2d_* launch of the calling thread: while it runs, an idle warp of every
 * CTA prefetches a slice of `weights` (the weight matrix of the kernel that will follow it) into L2
 * (cp.async.bulk.prefetch.L2).  Inside a denoise step every layer's weights come from HBM; this hides the first round
 * trips of the following launch.  A pure performance hint: results never depend on it. */
void ih_gemm_prefetch_next(const void* weights, long long bytes);

/* Debug aid: CTA 0 of later GEMM / conv launches writes %globaltimer stamps into this device buffer (>= 16 uint64);
 * NULL disables.  Not used on the product path. */
void ih_gemm_set_trace(void* device_buffer);

/* 3x3 convolution, padding 1, stride 1|2, NHWC activations, weight [Cout, 9*Cin] (tap-major: (ky*3+kx)*Cin + c).
 * out = conv(x) + bias[Cout] + rowbias[b*ld_rowbias + c] + residual.  Replaces diffusers ResnetBlock2D / Downsample2D /
 * Upsample2D nn.Conv2d (custom_pipelines.py:338-345 -> unet forward). */
int ih_conv2d_f16(const void* x, const void* w, const void* bias, const void* rowbias, long long ld_rowbias,
                  const void* residual, void* out, int B, int Hin, int Win, int Cin, int Cout, int ksize, int stride,
                  int tile_n, void* stream);
/* 3x3 conv (stride 1, pad 1) with a FUSED 1x1 shortcut convolution over one or two further NHWC sources:
 *   out = conv3x3(x) + [sc0 | sc1] Wsc^T + bias + rowbias        w = [Cout, 9*Cin + Csc0 + Csc1] (3x3 taps, then Wsc)
 * i.e. diffusers ResnetBlock2D `conv2(h) + conv_shortcut(cat(hidden, skip))` as ONE launch: the shortcut's K blocks
 * accumulate into the same accumulator tile and the channel concat of the up-blocks is never materialised.  Csc0, Csc1 % 64 == 0;
 * sc1 may be NULL. */
int ih_conv2d_shortcut_f16(const void* x, const void* w, const void* bias, const void* rowbias, long long ld_rowbias,
                           const void* sc0, int Csc0, const void* sc1, int Csc1, void* out, int B, int H, int W, int Cin,
                           int Cout, void* stream);
/* out = alpha * conv(x) + bias + residual (3x3, pad 1): the VAE decoder's scaled residual stream, see ih_gemm_scaled_f16.
 * epilogue: IH_EPI_NONE, or IH_EPI_RELU for relu(alpha * conv(x) + bias + residual) (the tiny autoencoder's convs). */
int ih_conv2d_scaled_f16(const void* x, const void* w, const void* bias, const void* residual, void* out, int B, int Hin,
                         int Win, int Cin, int Cout, int stride, float alpha, void* stream, int epilogue);

/* out = alpha * conv(x) + bias: 3x3 conv, stride 2, padded by one zero row / column at the BOTTOM and RIGHT only
 * (Ho = Hin / 2, Wo = Win / 2; Hin, Win even).  Replaces [3P] diffusers Downsample2D(padding=0) of the VAE encoder
 * (`F.pad(x, (0, 1, 0, 1))` then Conv2d(stride 2, padding 0)); alpha serves the encoder's scaled residual stream.
 * Same weight layout and tile_n values as ih_conv2d_f16. */
int ih_conv2d_down_f16(const void* x, const void* w, const void* bias, void* out, int B, int Hin, int Win, int Cin,
                       int Cout, int tile_n, float alpha, void* stream);

/* Multi-head attention, head_dim 64, softmax scale 1/8, no mask.
 *   q: [B, Nq, *] rows with ldq elements per row, head h at columns [h*64, h*64+64) (same for k, v, out).
 *   Self attention (n_ip == 0): out = softmax(q k^T / 8) v over Nk keys.
 *   Decoupled IP cross attention (n_ip > 0): keys/values are the concatenation [text (Nk - n_ip) ; ip (n_ip)];
 *     out = softmax_text(q k_t^T/8) v_t + ip_scale * softmax_ip(q k_ip^T/8) v_ip   (two separate softmaxes).
 * Replaces F.scaled_dot_product_attention at attention_processor.py:312-314 (self), :423-425 (text branch),
 * :440-442 + :450 (IP branch and the scale*ip axpy).  Nk <= 128 uses the single-block path.
 *   workspace: NULL, or a caller-owned scratch buffer (>= ih_attention_workspace_bytes(...) bytes, no initialisation
 *     needed).  With it the long self-attention shapes (Nk > 128, n_ip == 0) cut the query tiles that would otherwise
 *     form a nearly empty last wave into KV parts that share one wave and are merged by a second small kernel
 *     (flash-decoding style, fixed merge order: deterministic).  Without it every query tile is processed whole. */
int ih_attention_ws_f16(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv,
                        void* out, long long ldo, int B, int H, int Nq, int Nk, int n_ip, float ip_scale,
                        void* workspace, long long workspace_bytes, void* stream);
long long ih_attention_workspace_bytes(int B, int H, int Nq, int Nk, int n_ip);

/* Test aid: 0 (default) = split only when the cost model predicts a gain, 1 = split every partial last wave (at
 * least 2 parts, even where they overflow into one more wave). */
void ih_attention_set_split_policy(int policy);
/* Test / A-B aid: the kernel of the multi-block path (Nk > 128).  0 (default) = the persistent warp-specialised
 * kernel, 1 = the two-CTA-per-SM kernel that also serves Nk <= 128.  Rows processed whole are bit-identical between
 * the two; the KV-split plan (and so the rows of split units) follows the selected kernel's residency. */
void ih_attention_set_kernel(int kernel);

/* GroupNorm over NHWC [B, HW, C] (optionally the channel-concatenation of two tensors x0 [.., C0] and x1 [.., C1]),
 * fp32 partial sums reduced in double, optional fused SiLU.  stats_ws: ih_groupnorm_workspace_bytes(B, groups) bytes,
 * zero-initialised ONCE by the caller (the kernels leave its ticket counters at zero again) and not shared by
 * concurrently running calls.  C = C0 + C1 <= 4096 with C0, C1 multiples of 8, groups divides C (and groups <= C / 2
 * when C > 1024), 1 <= B <= 1024.  Replaces nn.GroupNorm (+ nn.SiLU) in diffusers ResnetBlock2D / Transformer2DModel. */
long long ih_groupnorm_workspace_bytes(int B, int groups);
int ih_groupnorm_f16(const void* x0, int C0, const void* x1, int C1, const void* gamma, const void* beta, void* out,
                     void* stats_ws, int B, int HW, int groups, float eps, int silu, void* stream);

/* LayerNorm over the last dim of [rows, C], fp32 statistics. Replaces nn.LayerNorm in BasicTransformerBlock. */
int ih_layernorm_f16(const void* x, const void* gamma, const void* beta, void* out, int rows, int C, float eps,
                     void* stream);

/* Small-M linear (M <= 64 rows): out[m, n] = act_out(W[n,:] . act_in(x[m,:]) + b[n]) * out_scale + addend[m, n];
 * act: 0 none, 1 SiLU.
 * Time / added-condition embeddings and the 17 time_emb_proj layers (diffusers), ImageProjModel / HarmonyAttention
 * linears (ip_adapter.py:41-48, train.py:243-266). */
int ih_linear_small_f16(const void* x, long long ldx, const void* w, const void* bias, const void* addend,
                        long long ld_add, void* out, long long ldo, int M, int N, int K, int act_in, int act_out,
                        float out_scale, void* stream);

/* Small generic attention on CUDA cores: out = softmax(q k^T / scale) v, head dims dqk / dv <= 128, Nk <= 1024,
 * B*H*Nq a multiple of 4.  HarmonyAttention's Cross_Attention (attention_processor.py:35-56; head_dim 40, v_dim 64,
 * scale = sqrt(40) is a divisor as in the reference), once per generate(). */
int ih_attention_small_f16(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv,
                           void* out, long long ldo, int B, int H, int Nq, int Nk, int dqk, int dv, float scale,
                           void* stream);

/* Sinusoidal embedding (flip_sin_to_cos, shift 0): out[i, :] = [cos(t_i f), sin(t_i f)], f = 10000^(-j/half). t fp32.
 * step_i32 == NULL: t_i = t_f32[i]; else every row uses t_f32[*step_i32] (device-resident step counter, so the
 * timestep of custom_pipelines.py:325 can live inside a replayed CUDA graph). */
int ih_sinusoid_f16(const void* t_f32, const void* step_i32, void* out, long long ldo, int n, int dim, void* stream);

/* out[i] = a[i] + b[i % period]: residual / positional-embedding adds of the Resampler (resampler.py:128-131,143-144). */
int ih_add_bcast_f16(const void* a, const void* b, void* out, long long n, long long period, void* stream);
/* out[b, :] = mean_n x[b, n, :]  -- Resampler masked_mean with an all-ones mask (resampler.py:137-138,150-158). */
int ih_mean_tokens_f16(const void* x, void* out, int B, int n, int D, void* stream);

/* In-place row softmax of an fp16 matrix [rows, cols] (row stride ld elements, fp32 statistics), cols <= 32768, over
 * the first valid_cols columns of every row (valid_cols = cols: the whole row); the padding columns are written as 0.
 * With two ih_gemm_f16 calls it forms the single-head, head_dim-512 attention of the VAE decoder mid block
 * ([3P] diffusers AutoencoderKL, called at custom_pipelines.py:373). */
int ih_softmax_rows_masked_f16(void* x, long long ld, long long rows, int cols, int valid_cols, void* stream);

/* Nearest-neighbour 2x upsample NHWC [B,H,W,C] -> [B,2H,2W,C]. */
int ih_upsample2x_f16(const void* x, void* out, int B, int H, int W, int C, void* stream);

/* Channel concat of two NHWC tensors: out[.., :C0] = x0, out[.., C0:] = x1. rows = B*H*W. */
int ih_concat_f16(const void* x0, int C0, const void* x1, int C1, void* out, long long rows, void* stream);

/* conv_in on the tensor-core GEMM: im2col of the NCHW latent into A [B*H*W, Kpad] (k = ci*9 + ky*3 + kx, zero padded),
 * to be multiplied with the OIHW weight flattened (and zero padded) to [Cout, Kpad] by ih_gemm_f16. */
int ih_im2col3x3_nchw_f16(const void* x_nchw, void* out, int B, int Cin, int H, int W, int Kpad, void* stream);
/* The same patch matrix for the channel concatenation of x0 [B,C0,H,W] and x1 [B,C1,H,W] (NCHW fp16) without forming it:
 * column k = ci*9 + ky*3 + kx reads x0 for ci < C0 and x1 channel ci - C0 otherwise (conv_in of the 9-channel
 * inpainting UNet: latents | mask | masked-image latents).  Kpad % 8 == 0 and Kpad >= (C0 + C1) * 9. */
int ih_im2col3x3_nchw_cat_f16(const void* x0, int C0, const void* x1, int C1, void* out, int B, int H, int W, int Kpad,
                              void* stream);
/* conv_out on ih_conv2d_f16 with Cout padded to 16: gather NHWC [B, HW, ldc] channels [0, C) into NCHW [B, C, HW]. */
int ih_nhwc_to_nchw_f16(const void* x, long long ldc, void* out, int B, long long HW, int C, void* stream);

/* Image-to-image initial latents ([3P] diffusers StableDiffusionXLImg2ImgPipeline.prepare_latents with fp16 latents):
 *   z = posterior sample of the VAE encoder's moments (mean + exp(0.5 clamp(logvar, -30, 20)) * eps),
 *   out = fp16(fp16(scaling_factor * fp16(z)) + fp16(noise * fp16(sigma)))   (EulerDiscreteScheduler.add_noise).
 * moments: NHWC fp16 [B_moments, HW, ldc] (mean = channels [0, C), logvar = [C, 2C)); eps: NCHW [B_eps, C, HW], fp32
 * (eps_f32 = 1: the fp32 posterior of an upcast VAE) or fp16 (eps_f32 = 0: fp16 posterior, fp16 rounding after every
 * op); noise, out: NCHW fp16 [B, C, HW].  Image b reads moments[b % B_moments] and eps[b % B_eps] (the torch.cat tiling
 * of encoded latents); B must be a multiple of both.  eps and noise are drawn by the caller from its generators. */
int ih_vae_posterior_noise_f16(const void* moments, long long ldc, const void* eps, int eps_f32, const void* noise,
                               void* out, int B, int B_moments, int B_eps, long long HW, int C, float scaling_factor,
                               float sigma, void* stream);

/* One scheduler transition (custom_pipelines.py:332-334,348-357):
 *   eps = u + g (c - u)  (fp16 tensor arithmetic, rounded like the reference's);
 *   x <- fp16( x + ((x - (x - sigma_i eps)) / sigma_i) (sigma_{i+1} - sigma_i) )   (fp32 inside, Euler, [3P] diffusers);
 *   model_in <- cat([x, x]) / sqrt(sigma_{i+1}^2 + 1)  (next step's scaled CFG input); step counter i += 1.
 * noise_pred: [2n,4,H,W] fp16 (uncond half first), latents: [n,4,H,W] fp16, model_in: [2n,4,H,W] fp16.
 * sigmas: device fp32 [T+1]; step: device int32 (read, then incremented). n_per_image = 4*H*W. */
int ih_euler_cfg_step(const void* noise_pred, void* latents, void* model_in, const void* sigmas, void* step,
                      float guidance, long long n_per_image, int n_images, void* stream);

/* ---- scope row f2: conditioning encoders (CLIP towers the reference loads at ip_adapter.py:81-84 and calls at
 * :163-164 (image) and through encode_prompt :292-319 (text)); arithmetic = [3P] transformers CLIPEncoderLayer. ---- */

/* softmax(q k^T * scale (+ causal mask)) v, any head dims that are multiples of 8 (<= 256), fp32 softmax.
 * q [B*Nq, >= H*dqk], k [B*Nk, >= H*dqk], v [B*Nk, >= H*dv], out [B*Nq, >= H*dv]; causal: key j visible iff j <= i.
 * Replaces CLIPAttention (text: causal, head_dim 64; ViT-bigG vision: head_dim 104). */
int ih_attention_generic_f16(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv,
                             void* out, long long ldo, int B, int H, int Nq, int Nk, int dqk, int dv, float scale,
                             int causal, void* stream);

/* out[r, :] = tok_emb[ids[r], :] + pos_emb[r % T, :]   (CLIPTextEmbeddings); ids int32 device [rows]. */
int ih_embed_tokens_f16(const void* ids_i32, const void* tok_emb, const void* pos_emb, void* out, int rows, int T, int C,
                        int vocab, void* stream);

/* PNS judge front end: image NCHW fp16 in [-1, 1] (VAE output) -> area-averaged S x S -> [0, 1] -> CLIP mean / std
 * normalisation -> patch rows [B*(S/P)^2, Kpad], k = c*P*P + py*P + px (flattened patch_embedding conv weight layout).
 * mean3 / std3: HOST pointers to 3 floats. */
int ih_resize_patchify_f16(const void* img_nchw, void* out, int B, int C, int Hin, int Win, int S, int P, int Kpad,
                           const float* mean3, const float* std3, void* stream);

/* General scheduler transition: the loop options the reference accepts beyond the default CFG path.
 *   use_cfg = 0 : guidance_scale <= 1 (custom_pipelines.py:223 do_classifier_free_guidance False): noise_pred and
 *                 model_in are [n,4,H,W]; eps = noise_pred (:332,:348 skipped).
 *   guidance_rescale > 0 (:352-354, [3P] diffusers rescale_noise_cfg): eps <- r * eps * (std(c) / std(eps)) + (1 - r) * eps
 *                 with the per-image unbiased std over all non-batch elements, fp16 rounding points of the fp16 tensors.
 * Otherwise identical to ih_euler_cfg_step (which stays the fast path for the default call). */
int ih_euler_step_ex(const void* noise_pred, void* latents, void* model_in, const void* sigmas, void* step,
                     float guidance, float guidance_rescale, long long n_per_image, int n_images, int use_cfg,
                     void* stream);

/* Inpainting transition ([3P] diffusers StableDiffusionXLInpaintPipeline, 4-channel UNet): the transition of
 * ih_euler_step_ex (same use_cfg / guidance_rescale options and rounding points), then, on the fp16 Euler result x of
 * step i = *step, the blend with the image outside the mask before latents and model_in are written:
 *   proper = fp16(img + fp16(noise * fp16(sigma[i+1])))  if i + 1 < *blend_end,  else img;
 *   x <- fp16(fp16(fp16(1 - m) * proper) + fp16(m * x)),  m = mask[b, pixel] over the 4 channels;
 *   model_in <- x / sqrt(sigma[i+1]^2 + 1) (duplicated with CFG); step counter i += 1.
 * image_latents, noise: [n,4,H,W] fp16 (tiled to the batch), mask: [n,1,H,W] fp16, n_per_image = 4*H*W; blend_end:
 * device int32, the absolute schedule index where the loop ends (read at every step, so one graph serves every
 * denoising_end). */
int ih_euler_inpaint_step(const void* noise_pred, void* latents, void* model_in, const void* sigmas, void* step,
                          float guidance, float guidance_rescale, long long n_per_image, int n_images, int use_cfg,
                          const void* image_latents, const void* noise, const void* mask, const void* blend_end,
                          void* stream);

/* Multistep-solver transition with the use_cfg / guidance_rescale options and CFG rounding points of ih_euler_step_ex.
 * `solver` picks the scheduler; step i = *step reads row i of its coefficient table `coeffs`, computed on the host
 * with torch fp32 0-dim arithmetic.  Both write latents and model_in <- latents (unscaled, duplicated with CFG) and
 * advance the step counter; loop_begin is a device int32, the first schedule index of the loop (only read), whose step
 * has no history.  prev_x0, last_sample, prev_x0_2: [n,C,H,W] fp16 buffers the solver keeps between steps.
 *
 * IH_SOLVER_DPMPP_2M ([3P] diffusers DPMSolverMultistepScheduler: dpmsolver++, midpoint, epsilon prediction):
 * coeffs fp32 [T, IH_DPM_COEFFS]
 *   {sigma_s, 1/alpha_s, sigma_t/sigma_s, c = alpha_t*(exp(-h)-1), 0.5*c, 1/r0, first, 0}
 * (VP sigmas, h = lambda_t - lambda_s, r0 = h_prev / h).  With eps the guided prediction and x the fp16 latents:
 *   x0 = fp16(fp16(x - fp16(sigma_s*eps)) * (1/alpha_s));
 *   x  <- fp16(fp32(ratio*x) - fp16(c*x0) [- fp16(0.5c * fp16(1/r0 * fp16(x0 - prev_x0)))])
 * where the bracket (second order) is dropped iff i == *loop_begin or first != 0.  prev_x0 <- x0.  last_sample and
 * prev_x0_2 must be null.
 *
 * IH_SOLVER_UNIPC_BH2 ([3P] diffusers UniPCMultistepScheduler: bh2, solver_order 2, predict_x0, epsilon prediction):
 * coeffs fp32 [T, IH_UNIPC_COEFFS]
 *   {sigma_s, 1/alpha_s, p_ratio, p_c, 1/rk_p, p, c_ratio, c_c, 1/rk_c, rho0, rho1, c, 0, 0, 0, 0}
 * with the predictor's scalars from sigma_i -> sigma_{i+1} and the corrector's from sigma_{i-1} -> sigma_i (ratio =
 * sigma_t/sigma_s0 of VP sigmas, c = alpha_t*expm1(-h), rk = (lambda_{s_k} - lambda_s0)/h, rho = fp16 rhos_c) and the
 * orders p = min(2, T-i, i+1), c = p(i-1) (0 at i = 0).  The corrector of order c rewrites x from last_sample,
 * prev_x0 (and prev_x0_2 when c == 2) and x0; then prev_x0_2 <- prev_x0 <- x0, last_sample <- x, and the predictor
 * of order p steps x to the latents (SURVEY A.9).  A loop starting at b = *loop_begin lowers the orders to
 * p <= i - b + 1 and c <= i - b.  last_sample and prev_x0_2 are required. */
#define IH_SOLVER_DPMPP_2M 0
#define IH_SOLVER_UNIPC_BH2 1
#define IH_DPM_COEFFS 8
#define IH_UNIPC_COEFFS 16
int ih_dpm_solver_step(const void* noise_pred, void* latents, void* model_in, void* prev_x0, const void* coeffs,
                       void* step, const void* loop_begin, float guidance, float guidance_rescale, long long n_per_image,
                       int n_images, int use_cfg, void* stream, int solver, void* last_sample, void* prev_x0_2);

/* Euler Ancestral transition ([3P] diffusers EulerAncestralDiscreteScheduler, epsilon prediction) with the use_cfg /
 * guidance_rescale options and CFG rounding points of ih_euler_step_ex.  Step i = *step reads row i of coeffs, fp32
 * [T, IH_EULER_A_COEFFS] computed on the host:
 *   {sigma_i, 1/sigma_i, dt = sigma_down - sigma_i, sigma_up, 1/sqrt(sigma_{i+1}^2 + 1), fp16(sigma_{i+1}),
 *    1/sqrt(sigma_i^2 + 1), 0}
 * and row i of step_noise, fp16 [T, n, 4, H, W] drawn by the caller.  With eps the guided prediction, x the latents:
 *   x0 = x - fp16(sigma*eps);  x <- fp16(fp32(fp32((x - x0) * (1/sigma)) * dt) + x + fp16(noise * sigma_up))
 * (fp32 sums left to right).  With image_latents, blend_noise, mask and blend_end (all or none) the inpainting blend of
 * ih_euler_inpaint_step follows, re-noising with fp16(sigma_{i+1}).  Writes latents and
 * model_in <- fp16(x * (1/sqrt(sigma_{i+1}^2 + 1))) (duplicated with CFG); step counter i += 1. */
#define IH_EULER_A_COEFFS 8
int ih_euler_ancestral_step(const void* noise_pred, void* latents, void* model_in, const void* coeffs,
                            const void* step_noise, void* step, float guidance, float guidance_rescale,
                            long long n_per_image, int n_images, int use_cfg, const void* image_latents,
                            const void* blend_noise, const void* mask, const void* blend_end, void* stream);
/* The first model input of an Euler Ancestral loop in the same convention: model_in = fp16(latents * coeffs[*step, 6])
 * (duplicated when duplicate != 0), i.e. diffusers' scale_model_input as ATen evaluates it. */
int ih_euler_ancestral_scale_input(const void* latents, void* model_in, const void* coeffs, const void* step,
                                   long long total, int duplicate, void* stream);

/* model_in = cat([latents, latents]) / sqrt(sigma[*step]^2 + 1)   (custom_pipelines.py:332-334, first step); with
 * duplicate = 0, model_in = latents / sqrt(...) for the no-CFG loop (custom_pipelines.py:332 else-branch). */
int ih_scale_model_input_ex(const void* latents, void* model_in, const void* sigmas, const void* step, long long total,
                            int duplicate, void* stream);

/* 3x3 conv, pad 1, stride 1 or 2, for the small channel counts of the ControlNet conditioning embedding ([3P] diffusers
 * ControlNetConditioningEmbedding: 3/16/32/96 input channels, which the implicit-GEMM conv cannot take).
 *   out[b, yo, xo, co] = fp16(act(bias[co] + sum_{tap, ci} x[b, yo*stride + ky - 1, xo*stride + kx - 1, ci] w[co, tap, ci]))
 * with fp32 accumulation, act = SiLU when silu = 1.  x is read through the element strides (sb, sh, sw, sc), so NCHW
 * and NHWC inputs both work; w is tap-major [Cout, 9 * Cin] (ops.pack_conv3x3_weight); bias may be NULL; out is NHWC
 * [B, Ho, Wo, Cout] contiguous with Ho = ceil(H / stride), Wo = ceil(W / stride). */
int ih_conv3x3_small_f16(const void* x, long long sb, long long sh, long long sw, long long sc, const void* w,
                         const void* bias, void* out, int B, int H, int W, int Cin, int Cout, int stride, int silu,
                         void* stream);

/* ControlNet residual injection ([3P] diffusers UNet2DConditionModel with down_block_additional_residuals /
 * mid_block_additional_residual): for each entry k, in place on rows [skip_row0, skip_row0 + rows) of `skip`
 * ([*, channels] contiguous fp16),  skip = fp16(skip + fp16(residual * scale[k]))  with residual [rows, channels]
 * contiguous fp16 and scale a device fp32 vector of n_entries values.  One launch for all entries; the entries are
 * copied into the kernel's arguments (a captured graph keeps them), the scales are read from device memory at run
 * time.  channels must be a multiple of 8 and both pointers 16-byte aligned. */
#define IH_CN_MAX_RESIDUALS 16
typedef struct IhCnResidual {
  void* skip;
  const void* residual;
  long long rows;
  long long skip_row0;
  int channels;
} IhCnResidual;
int ih_controlnet_add_residuals_f16(const IhCnResidual* entries, int n_entries, const void* scale, void* stream);

/* Multi-ControlNet residual injection ([3P] diffusers MultiControlNetModel, whose nets' scaled residuals are summed in
 * fp16 in net order before the UNet adds them): for each entry e, in place on rows [skip_row0, skip_row0 + rows) of
 * `skip` ([*, channels] contiguous fp16),
 *   acc = fp16(r_0 * s_0[e]);  acc = fp16(acc + fp16(r_k * s_k[e])) for k = 1 .. n_nets - 1;  skip = fp16(skip + acc)
 * with r_k = residual[k] ([rows, channels] contiguous fp16) and s_k = scales[k], net k's device fp32 vector of
 * n_entries values.  One launch for all entries and nets; entries and scale pointers are copied into the kernel's
 * arguments, the scale values are read from device memory at run time.  n_nets = 1 computes exactly what
 * ih_controlnet_add_residuals_f16 computes (which stays the faster single-net path).  channels must be a multiple of 8
 * and every pointer 16-byte aligned. */
#define IH_CN_MAX_NETS 8
typedef struct IhCnMultiResidual {
  void* skip;
  long long rows;
  long long skip_row0;
  int channels;
  const void* residual[IH_CN_MAX_NETS];
} IhCnMultiResidual;
int ih_controlnet_add_residuals_multi_f16(const IhCnMultiResidual* entries, int n_entries, const void* const* scales,
                                          int n_nets, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* IH_API_H */
