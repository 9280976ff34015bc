/* lb200.h -- C ABI of liblb200.so: the H100-native (sm_90a) backend of the
 * latentblending branch-tree denoising hot path.
 *
 * The reference (lunarring/latentblending @ fd5916a) has no FFI: its operator
 * seam is the duck-typed ``DiffusersHolder`` Python object.  Every entry point
 * below names the reference call it replaces (file:line under
 * /root/reference/latentblending/).  INTEGRATION.md shows the ctypes stub a
 * maintainer of the reference would add.
 *
 * Conventions
 *  - plain C types only; every ``dev`` pointer is a device pointer on the
 *    context's CUDA device; ``stream`` is a ``cudaStream_t`` passed as void*.
 *  - all calls enqueue asynchronously on ``stream``; no host sync, no
 *    allocation inside hot calls (the caller owns every buffer, including the
 *    workspaces whose sizes the *_workspace_bytes calls report).
 *  - return 0 on success, non-zero on error; lb_last_error() describes the
 *    last failure on the calling thread.
 *  - fp16 means IEEE binary16 (``__half``).  Activations are NHWC
 *    ([batch*height*width, channels] row-major); latents are NCHW like the
 *    reference's ``[1,4,h,w]`` tensors.
 *  - bf16 means bfloat16 (``__nv_bfloat16``: fp32's 8-bit exponent, 8-bit
 *    significand).  The VAE-decoder ops also exist in bf16: the stock SDXL
 *    VAE's activations exceed fp16's range (the reference decodes it in fp32
 *    when its config sets force_upcast, diffusers_holder.py:128-139), bf16's
 *    range is fp32's, and bf16 wgmma runs at the fp16 rate.  lb_gemm takes its
 *    types from its mode flags (LB_GEMM_BF16); every other op with a bf16
 *    variant takes a trailing ``int dtype`` (LB_DTYPE_F16 or LB_DTYPE_BF16, the
 *    element type of its 16-bit tensors; any other value is an error):
 *    lb_groupnorm, lb_conv_in, lb_upsample_nearest, lb_latent_prep,
 *    lb_softmax_rows, lb_postprocess_u8, lb_nhwc_to_nchw, lb_image_conv_in and
 *    lb_add_noise_rows.  A bf16 call keeps
 *    the fp16 call's layouts, strides, alignment rules and fp32 arithmetic;
 *    only the stored element type differs, except where an entry point says
 *    otherwise.
 */
#ifndef LB200_H
#define LB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LB_ABI_VERSION 4

/* element type of the ops that exist in both 16-bit formats (lb_op.dtype, the trailing ``dtype`` arguments) */
enum { LB_DTYPE_F16 = 0, LB_DTYPE_BF16 = 1 };

typedef struct lb_ctx lb_ctx;

int         lb_abi_version(void);
const char* lb_last_error(void);
/* one context per device; not thread-safe per context */
int lb_ctx_create(int device, lb_ctx** out);
int lb_ctx_destroy(lb_ctx* ctx);
int lb_ctx_sm_count(lb_ctx* ctx);

/* ---- K1: latent mixing ----------------------------------------------------
 * lb_slerp_rows: ``rows`` independent whole-row spherical interpolations
 *   out[r] = slerp(p0[r], p1[r], fract)   (fp64 arithmetic, result cast
 *   fp64->fp32->dtype, exactly utils.py:47-71).
 * Replaces: utils.py:29-71 interpolate_spherical; the 30-iteration parental
 * mix loop blending_engine.py:442-450 (rows = steps x branches; the None rows
 * are simply not passed); the in-loop crossfeed diffusers_holder.py:322-324
 * (rows = 1).
 *   dtype: 0 = fp16, 1 = fp32.  n = elements per row; row r starts at
 *   base + r*stride_{0,1,out} elements.  fract_rows_dev (device, fp64[rows])
 *   overrides ``fract`` per row when non-NULL.
 *   workspace_dev: lb_slerp_workspace_bytes(rows, n) bytes (may be NULL when
 *   that returns 0).
 */
size_t lb_slerp_workspace_bytes(int64_t rows, int64_t n);
int lb_slerp_rows(lb_ctx* ctx, const void* p0_dev, const void* p1_dev, void* out_dev,
                  int64_t rows, int64_t n, int64_t stride0, int64_t stride1, int64_t stride_out,
                  int dtype, double fract, const double* fract_rows_dev,
                  void* workspace_dev, void* stream);

/* lb_lerp: out = (1-f)*p0 + f*p1 elementwise, per-op rounding in ``dtype``
 * like torch (utils.py:97 on the 4-tuple text embeddings,
 * blending_engine.py:643-654). */
int lb_lerp(lb_ctx* ctx, const void* p0_dev, const void* p1_dev, void* out_dev,
            int64_t n, int dtype, double fract, void* stream);

/* ---- K9: scheduler arithmetic around the UNet ------------------------------
 * lb_scale_model_input: x_in[b] = fp16(x / divisor) for b < batch (CFG
 * duplicate, diffusers_holder.py:328-330; divisor = sqrt(sigma^2+1) in fp32).
 */
int lb_scale_model_input(lb_ctx* ctx, const void* latents_dev, void* out_dev,
                         int64_t n, int batch, float divisor, void* stream);

/* lb_cfg_euler_step: classifier-free-guidance combine + Euler(-ancestral) step
 * + trajectory store, with the reference's per-op fp16 roundings reproduced:
 *   eps = u + g*(t-u)                        diffusers_holder.py:347-349
 *   x'  = x + ((x-(x-sigma*eps))/sigma)*dt   diffusers_holder.py:356 (Euler)
 *   x'' = x' + noise*sigma_up                (ancestral only; noise may be NULL)
 * eps_dev holds [2,n] (uncond, text) when use_cfg else [1,n]; eps_text_dev (optional) points at the text half when
 * it is not adjacent to the unconditional one (the two CFG halves computed on two GPUs and exchanged per step).
 * Writes the new latents to out_dev and, if non-NULL, a clone to traj_dev
 * (``list_latents_out.append(latents.clone())``, diffusers_holder.py:359).
 * scaled_next_dev (optional): the NEXT step's model input, fp16(x'' / next_divisor) replicated scaled_batch times
 * (the next iteration's diffusers_holder.py:328-330) -- saves the separate lb_scale_model_input launch whenever the
 * next step has no crossfeed mix in between.
 */
int lb_cfg_euler_step(lb_ctx* ctx, const void* latents_dev, const void* eps_dev, const void* eps_text_dev,
                      const void* noise_dev, void* out_dev, void* traj_dev,
                      int64_t n, int use_cfg, float guidance, float sigma, float dt,
                      float sigma_up, void* scaled_next_dev, int scaled_batch, float next_divisor,
                      void* stream);

/* lb_cfg_lcm_step: the same CFG combine, trajectory store and fused next-step input as lb_cfg_euler_step, with the
 * step of diffusers 0.25.0 LCMScheduler (epsilon prediction; LCM-LoRA / LCM-SDXL), every op rounded to fp16:
 *   x0  = (x - sqrt_beta*eps) * inv_sqrt_alpha    sqrt(1-alpha_t), 1/sqrt(alpha_t): the CUDA stack divides by a CPU
 *                                                 scalar as a multiply by its fp32 reciprocal
 *   den = c_out*x0 + c_skip*x                     c_skip = .25/(s^2+.25), c_out = s/sqrt(s^2+.25), s = t*scaling
 *   x'  = sqrt_alpha_prev*den + sqrt_beta_prev*noise   when noise_dev is non-NULL (every step but the last), else den
 * LCM's scale_model_input is the identity, so the fused next-step input is written with next_divisor = 1.
 */
int lb_cfg_lcm_step(lb_ctx* ctx, const void* latents_dev, const void* eps_dev, const void* eps_text_dev,
                    const void* noise_dev, void* out_dev, void* traj_dev,
                    int64_t n, int use_cfg, float guidance, float sqrt_beta, float inv_sqrt_alpha, float c_skip,
                    float c_out, float sqrt_alpha_prev, float sqrt_beta_prev, void* scaled_next_dev, int scaled_batch,
                    float next_divisor, void* stream);

/* lb_cfg_dpm_step: the same CFG combine, trajectory store and fused next-step input, with the step of diffusers
 * 0.25.0 DPMSolverMultistepScheduler (dpmsolver++ / sde-dpmsolver++, epsilon prediction, first order or the multistep
 * second order, midpoint or heun), every op rounded to fp16, the scalars unrounded fp32 (CPU scalars in the
 * reference's stack):
 *   x0 = (x - sigma_s*eps) * inv_alpha_s          convert_model_output; 1/alpha_s as an fp32 reciprocal multiply
 *   D1 = inv_r0 * (x0 - x0_prev)                  second order only (x0_prev_dev non-NULL)
 *   x' = c_x*x + c_0*x0 + c_1*D1 + c_n*noise      left to right; the D1 term only with x0_prev_dev, the noise term
 *                                                 only with noise_dev (sde-dpmsolver++)
 * The host folds the solver variant and the signs of subtracted terms into c_x, c_0, c_1, c_n.  x0_prev_dev NULL
 * selects first order: the term is skipped, so a history that was never written may hold anything.  x0_out_dev
 * (required) receives x0, the branch's history for its next step; it may alias x0_prev_dev.  DPM's
 * scale_model_input is the identity, so the fused next-step input is written with next_divisor = 1.
 */
int lb_cfg_dpm_step(lb_ctx* ctx, const void* latents_dev, const void* eps_dev, const void* eps_text_dev,
                    const void* noise_dev, const void* x0_prev_dev, void* x0_out_dev, void* out_dev, void* traj_dev,
                    int64_t n, int use_cfg, float guidance, float sigma_s, float inv_alpha_s, float inv_r0,
                    float c_x, float c_0, float c_1, float c_n, void* scaled_next_dev, int scaled_batch,
                    float next_divisor, void* stream);

/* ---- K7 / K4: tensor-core GEMM and implicit-GEMM convolution ----------------
 * out[M,N] = epilogue( conv_taps(a0)[M, taps*a0_c] | a1[M, a1_c] ) x w[N, K]^T ),
 * fp16 operands, fp32 accumulation in registers (wgmma), M = B*H*W rows of an
 * NHWC activation.  taps = 1: Linear / 1x1 conv; taps = 9: 3x3 conv, stride 1,
 * zero padding 1 (weights pre-packed [N][ky][kx][a0_c]).  a1 (optional) is a
 * second 1x1 input appended along K (the resnet shortcut conv folded into
 * conv2).  Epilogue mode 0: + bias[n] + bias2[b][n] (time-embedding projection)
 * + res[row][n]; mode 1: GEGLU, N accumulators -> N/2 outputs (weight rows
 * interleaved per 128-column tile: 64 value rows then their 64 gate rows).
 * Replaces the cuBLAS / cuDNN calls under pipe.unet(...)
 * (diffusers_holder.py:336-344).  Constraints: a0_c, a1_c multiples of 64;
 * N multiple of 8; 16-byte aligned bases; any B, H, W with B*H*W < 2^31.
 * M tiling: 128-row tiles are either a box of pixels (tw x th x tb: 128 x 1 x 1 when W >= 128; needs W, and H when
 * H*W < 128, to be powers of two below that) or pixel runs (tile m = rows [128m, 128m+128) of the flattened NHWC
 * order, loaded with TMA im2col; any W and H).  By default the one with fewer tiles is used and a tie keeps the box;
 * LB_GEMM_TILE_BOX / LB_GEMM_TILE_RUNS force one (forcing the box on a shape it cannot tile is an error).  Both give
 * bit-identical results.
 */
typedef struct lb_gemm_desc {
    const void* a0; int64_t a0_ld; int32_t a0_c;
    const void* a1; int64_t a1_ld; int32_t a1_c;
    int32_t B, H, W;
    int32_t taps;
    const void* w; int64_t w_ld;
    int32_t N;
    const void* bias;
    const void* bias2; int64_t bias2_ld;
    const void* res; int64_t res_ld;
    void* out; int64_t out_ld;
    int32_t mode;     /* low byte: 0 = linear epilogue, 1 = GEGLU; flags: LB_GEMM_STATIC_W, LB_GEMM_RELU,
                         LB_GEMM_TILE_BOX, LB_GEMM_TILE_RUNS, LB_GEMM_BF16, LB_GEMM_OUT_F16, LB_GEMM_D2S2 */
} lb_gemm_desc;
/* mode flag: `w` is not written by the kernel that precedes this one on the stream (true for model weights, false
 * when an activation is passed as the B operand): its first tiles may be fetched before the previous kernel ends. */
#define LB_GEMM_STATIC_W 0x100
/* mode flag (linear epilogue): out = max(out, 0) -- the AlexNet convolutions of the LPIPS metric */
#define LB_GEMM_RELU 0x200
/* mode flags: force the pixel-box (LB_GEMM_TILE_BOX) or the pixel-run (LB_GEMM_TILE_RUNS) M tiling instead of the
 * automatic choice; at most one of them */
#define LB_GEMM_TILE_BOX 0x400
#define LB_GEMM_TILE_RUNS 0x800
/* mode flag: a0, a1, w, bias, bias2, res and out are bf16 instead of fp16 (fp32 accumulation as in fp16; the output
 * is rounded to bf16).  Linear epilogue only: GEGLU is rejected.  The VAE decoder of a checkpoint whose activations
 * overflow fp16 runs on it. */
#define LB_GEMM_BF16 0x1000
/* mode flag, only with LB_GEMM_BF16: bf16 operands, fp16 output (the VAE attention scores, whose fp16 rounding is 8x
 * finer than bf16's and whose magnitudes stay far inside fp16's range; lb_softmax_rows reads them as fp16) */
#define LB_GEMM_OUT_F16 0x2000
/* mode flag: nearest-2x upsample followed by a 3x3 conv as ONE GEMM over the low-resolution map (the upsampling
 * convolutions of the tiny VAE decoder, AutoencoderTiny).  taps = 9 over a B x H x W map a0 with N = 4 * Co: the weight
 * rows are four phase filters, row p * Co + c with p = 2a + b, each a 3x3 filter over LOW-resolution taps (the original
 * filter's taps summed onto the low-resolution pixel they read after upsampling; see latentblending_b200/taesd.py).
 * Accumulator column p * Co + c of low-resolution pixel (img, y, x) is stored at output pixel (img, 2y + a, 2x + b),
 * channel c, of the NHWC output [4*B*H*W rows, row stride out_ld]: the upsampled input is never materialised.
 * fp16, linear epilogue (+ bias[N], LB_GEMM_RELU); rejected with res, bias2, a1, GEGLU or LB_GEMM_BF16, with
 * taps != 9 and with N % 32 != 0 (so Co % 8 == 0). */
#define LB_GEMM_D2S2 0x4000
int lb_gemm(lb_ctx* ctx, const lb_gemm_desc* desc, void* stream);

/* ---- K8: fused attention, head_dim 64 ----------------------------------------
 * out[b, s, h*64+d] = softmax(Q K^T * scale) V per (batch, head); Q/K/V are
 * column slices of row-major [B*S, ld] fp16 buffers: head h of Q lives in
 * columns [q_col0 + 64h, q_col0 + 64h + 64) etc., so a fused QKV projection
 * ([.., 3C]) or a fused cross-attention KV projection ([B*77, 2C]) is consumed
 * in place.  Replaces F.scaled_dot_product_attention (diffusers AttnProcessor2_0)
 * under pipe.unet(...), diffusers_holder.py:336-344.  No mask, no dropout.
 */
typedef struct lb_attn_desc {
    const void* q; int64_t q_ld; int32_t q_col0;
    const void* k; int64_t k_ld; int32_t k_col0;
    const void* v; int64_t v_ld; int32_t v_col0;
    void* out; int64_t out_ld;
    int32_t B, heads, Sq, Skv, head_dim;
    float scale;
} lb_attn_desc;
int lb_attention(lb_ctx* ctx, const lb_attn_desc* desc, void* stream);

/* ---- K5 / K6: normalisation -----------------------------------------------------
 * lb_groupnorm: torch.nn.GroupNorm(groups, C, eps) over an NHWC activation
 * [B*HW, C] (row stride ld), optionally followed by SiLU; fp32 statistics.
 * lb_layernorm: torch.nn.LayerNorm(C, eps) over rows.  Both replace the norm
 * layers inside pipe.unet(...) (diffusers_holder.py:336-344).
 * The GroupNorm workspace (lb_groupnorm_workspace_bytes) must be ZERO-FILLED once after allocation: it holds
 * per-batch "last block" counters which every call leaves at zero again; it may be shared by successive calls on
 * one stream.  Results do not depend on the batch size (row chunking is a function of HW only).
 * lb_groupnorm in bf16: the same fp32 statistics and fixed-order reduction; the output is rounded to bf16 after the
 * affine and again after SiLU.
 */
size_t lb_groupnorm_workspace_bytes(lb_ctx* ctx, int B, int HW, int groups);
int lb_groupnorm(lb_ctx* ctx, const void* x, int64_t ld, int B, int HW, int C, int groups,
                 const void* gamma, const void* beta, float eps, int silu,
                 void* out, int64_t ldo, void* workspace, void* stream, int dtype);
int lb_layernorm(lb_ctx* ctx, const void* x, int64_t ld, int64_t rows, int C,
                 const void* gamma, const void* beta, float eps, void* out, int64_t ldo, void* stream);

/* ---- K3 / K2: embeddings and the boundary convolutions ------------------------------
 * lb_embed_inputs: sinusoidal timestep features [B,dim_t] and the text_time
 *   added-condition vector [B, pooled + 6*dim_a] (diffusers get_timestep_embedding,
 *   flip_sin_to_cos, freq_shift 0).
 * lb_linear_small: out = act_out(act_in(x) W^T + bias) (+ addend) for M <= 16 rows
 *   (time_embedding, add_embedding, all resnet time_emb_proj in one launch);
 *   act: 0 none, 1 SiLU.
 * lb_conv_in: the 4->C0 3x3 convolution at the NCHW latent boundary.  ``act``
 *   chooses an input transform and an output activation:
 *   act 0: none (in_scale unused); x, w_packed, bias and out of type ``dtype``;
 *   act 1: the tiny VAE decoder's input stage (AutoencoderTiny:
 *          decoder(latents / scaling_factor), whose first steps are
 *          tanh(z / 3) * 3, Conv2d(4, C, 3, padding=1), ReLU).  Each input v
 *          becomes h(h(tanh(h(h(v * in_scale) / 3))) * 3), h = rounding to
 *          fp16 (the fp16 roundings of the reference's ``/ scaling_factor``,
 *          ``/ 3``, ``tanh`` and ``* 3``; in_scale = 1 / scaling_factor), then
 *          the 3x3 conv + bias, then max(., 0).  fp16 only.
 * lb_upsample_nearest: F.interpolate(size=(Ho, Wo), mode="nearest") of an H x W
 *   map for Ho in {2H-1, 2H} and Wo in {2W-1, 2W} (any other size is an error):
 *   Ho = 2H, Wo = 2W is the nearest 2x of Upsample2D; the cropped sizes are the
 *   Upsample2D of an up block whose skip level has an odd side (diffusers'
 *   forward_upsample_size, latent sides not divisible by 2^(levels-1)).  Output
 *   pixel (yo, xo) is input pixel (yo >> 1, xo >> 1), i.e. nearest 2x cropped to
 *   Ho x Wo.  C and both row strides multiples of 8.
 * lb_im2col_s2: patch matrix of the stride-2 Downsample2D convs (then lb_gemm);
 *   its output is ceil(H/2) x ceil(W/2), so any H and W.
 */
int lb_embed_inputs(lb_ctx* ctx, float t, const void* text_embeds, const void* time_ids, int B,
                    int dim_t, int pooled, int dim_a, void* temb_in, void* add_in, void* stream);
int lb_linear_small(lb_ctx* ctx, const void* x, int64_t ldx, int M, int K, const void* w, int64_t ldw,
                    const void* bias, const void* addend, int64_t ldadd, int act_in, int act_out,
                    void* out, int64_t ldo, int N, void* stream);
int lb_conv_in(lb_ctx* ctx, const void* x_nchw, int B, int Cin, int H, int W, const void* w_packed,
               const void* bias, int Cout, void* out, int64_t ldo, int act, float in_scale, void* stream, int dtype);
int lb_upsample_nearest(lb_ctx* ctx, const void* x, int64_t ld, int B, int H, int W, int C, void* out, int64_t ldo,
                        int Ho, int Wo, void* stream, int dtype);
/* lb_conv_in_add: lb_conv_in (act 0, fp16) followed by the addition of a per-pixel addend shared by every image of
 *   the batch: out row r = h(h(conv + bias) + addend[r mod H*W]) (h = fp16 rounding).  An SDXL ControlNet's
 *   ``conv_in(x) + controlnet_cond_embedding(image)`` in one launch: the embedding [H*W, Cout] (row stride ld_add,
 *   a multiple of 8) is computed once per control image and serves every batch row of every step. */
int lb_conv_in_add(lb_ctx* ctx, const void* x_nchw, int B, int Cin, int H, int W, const void* w_packed,
                   const void* bias, int Cout, void* out, int64_t ldo, const void* addend, int64_t ld_add,
                   void* stream);
int lb_im2col_s2(lb_ctx* ctx, const void* x, int64_t ld, int B, int H, int W, int C, void* out, void* stream);

/* ---- ControlNet conditioning embedding (diffusers 0.25 ControlNetConditioningEmbedding) ----------------------
 * lb_cond_conv: direct 3x3 convolution, zero padding 1, stride 1 or 2, of an NHWC map x [B*H*W rows, row stride
 *   ld_x] into NHWC fp16 out [B*Ho*Wo, Cout] (row stride ldo), Ho = floor((H - 1) / stride) + 1 (likewise Wo);
 *   fp32 accumulation, y = h(acc + bias), then y = h(silu(y)) when silu = 1 (h = fp16 rounding).  Weights are packed
 *   [ky][kx][Cin][Cout] fp16.  in_u8 = 1: x is a uint8 image (1 to 8 channels, ld_x in bytes) and every input u is
 *   read as h(u / 255) (the control image's VaeImageProcessor scaling, no normalisation to [-1, 1]); in_u8 = 0: x is
 *   fp16 with Cin a multiple of 8 up to 256.  Cout a multiple of 8.  Meant for the small channel counts of the
 *   embedding at full image resolution (3 -> 16 -> 32 -> 96 -> 256), where K = 9*Cin does not suit lb_gemm.
 */
int lb_cond_conv(lb_ctx* ctx, const void* x, int64_t ld_x, int B, int H, int W, int Cin, int in_u8,
                 const void* w_packed, const void* bias, int Cout, int stride, int silu, void* out, int64_t ldo,
                 void* stream);

/* ---- VAE encoder and img2img start (diffusers 0.25 AutoencoderKL.encode, scheduler.add_noise) ------------------
 * lb_image_conv_in: the encoder's conv_in on a uint8 image: lb_cond_conv's direct 3x3 pad-1 stride-1 convolution of
 *   x [B*H*W pixels, ld_x bytes apart, Cin <= 8 channels] into NHWC out [B*H*W, Cout] (row stride ldo), with
 *   VaeImageProcessor.preprocess fused into the read: every input u becomes r(2 (u / 255) - 1), fp32 arithmetic and
 *   one rounding r to ``dtype``.  Weights [ky][kx][Cin][Cout] and bias of type ``dtype``, fp32 accumulation,
 *   y = r(acc + bias).  Cout a multiple of 8.
 * lb_im2col_s2_pad01: the patch matrix of Downsample2D(padding=0): F.pad(x, (0, 1, 0, 1)) then a 3x3 stride-2 conv
 *   without padding; like lb_im2col_s2 (out [B*Ho*Wo, 9*C], column (ky*3 + kx)*C + c, then lb_gemm with taps = 1),
 *   with Ho = floor((H - 2) / 2) + 1 (likewise Wo) and H, W >= 2.  It copies 2-byte elements: fp16 and bf16 alike.
 * lb_add_noise_rows: out[r] = add_noise(x0, noise, coeffs[r]) for r < rows, fp16 [rows, n] rows n elements apart:
 *   the forward-diffused rows of a trajectory that starts part-way down the schedule, and its start latent.  coeffs
 *   (device, fp16 [rows][2]) holds each row's (a, b); with h = fp16 rounding and x = h(x0):
 *     form 0:  h(x + h(noise * b))              Euler / Euler-ancestral: x0 + noise * sigma
 *     form 1:  h(h(a * x) + h(b * noise))       LCM, DPM-Solver++: alpha_t * x0 + sigma_t * noise
 *   (scheduler.add_noise on fp16 CUDA tensors, diffusers 0.25.0).  x0 is fp16 or bf16 (``dtype``), noise fp16.
 *   nonfinite_count_dev (optional, device int) is incremented by the number of non-finite x0 elements; rows may be 0,
 *   and then the call only counts.
 */
int lb_image_conv_in(lb_ctx* ctx, const void* img_u8, int64_t ld_x, int B, int H, int W, int Cin,
                     const void* w_packed, const void* bias, int Cout, void* out, int64_t ldo, void* stream,
                     int dtype);
int lb_im2col_s2_pad01(lb_ctx* ctx, const void* x, int64_t ld, int B, int H, int W, int C, void* out, void* stream);
int lb_add_noise_rows(lb_ctx* ctx, const void* x0, const void* noise, const void* coeffs_dev, int form, int64_t n,
                      int rows, void* out, int* nonfinite_count_dev, void* stream, int dtype);

/* ---- SDXL T2I-Adapter (diffusers 0.25 T2IAdapter "full_adapter_xl", StableDiffusionXLAdapterPipeline) -----------
 * lb_add_rows_bcast: dst[b*rows + r, c] = h(dst[b*rows + r, c] + src[r, c]) for b < B, r < rows, c < C (fp16, fp32
 *   add, h = one fp16 rounding: torch's fp16 ``+=``).  The adapter's per-image state, shared by every batch row (the
 *   CFG halves, every lockstep job), added in place to a UNet skip or the mid-block output.  dst and src are row-major
 *   with row strides ld_dst / ld_src (multiples of 8, >= C); C a multiple of 8; bases 16-byte aligned.
 * lb_pixel_unshuffle_u8: F.pixel_unshuffle(image, r) of a uint8 image [H, W, Cimg] (contiguous, 8-byte aligned base)
 *   fused with the adapter input's scaling: out [(H/r)*(W/r), r*r*Cimg] fp16 (contiguous), element (i*r + j)*Cimg + c
 *   of output pixel (y, x) = fp16(float(img[y*r + i, x*r + j, c]) / 255).  The columns are in (i, j, c) order, a
 *   permutation of torch's (c, i, j): the consumer's weights are permuted to match.  H, W multiples of r; r*Cimg a
 *   multiple of 8.
 * lb_avgpool2_ceil: AvgPool2d(2, stride 2, ceil_mode=True) of an NHWC fp16 map [H*W, C] (row stride ld) into
 *   [ceil(H/2)*ceil(W/2), C] (row stride ldo): the fp32 sum of the window's in-bounds pixels in row-major order
 *   divided by their count, one fp16 rounding (torch's avg_pool2d).  C and the strides multiples of 8.
 */
int lb_add_rows_bcast(lb_ctx* ctx, void* dst, int64_t ld_dst, const void* src, int64_t ld_src, int B, int64_t rows,
                      int C, void* stream);
int lb_pixel_unshuffle_u8(lb_ctx* ctx, const void* img_u8, int H, int W, int Cimg, int r, void* out, void* stream);
int lb_avgpool2_ceil(lb_ctx* ctx, const void* x, int64_t ld, int H, int W, int C, void* out, int64_t ldo,
                     void* stream);

/* ---- VAE decoder helpers (SURVEY section 8f next #1; latent2image, diffusers_holder.py:114-143) ----
 * lb_latent_prep: post_quant_conv(latents / scaling_factor) as a per-pixel CxC fp32 matrix (scale folded in).
 * lb_softmax_rows: row softmax of an fp16 matrix (the VAE mid-block single-head attention, head dim 512,
 *   runs as lb_gemm(Q,K) -> lb_softmax_rows -> lb_gemm(P,V^T)).  Any cols; row strides multiples of 8, bases
 *   16-byte aligned.
 * lb_postprocess_u8: (x/2+0.5).clamp(0,1)*255 -> uint8 NHWC (VaeImageProcessor.postprocess).  nonfinite_count_dev
 *   (optional, device int) is incremented by the number of NaN/Inf pixels: the decoder runs in fp16 where the reference
 *   upcasts the stock SDXL VAE to fp32 because it "overflows in float16" (diffusers_holder.py:128-133); an overflow
 *   anywhere upstream reaches the image as Inf/NaN and is reported instead of silently producing a black frame.
 * With LB_DTYPE_BF16 (the bf16 decoder of a VAE that overflows fp16):
 *   lb_latent_prep: fp16 latents in, bf16 out;
 *   lb_softmax_rows: fp16 scores in (lb_gemm with LB_GEMM_BF16 | LB_GEMM_OUT_F16), bf16 probabilities out; in
 *     place too (out == x, ldo == ld: every element is read before the same thread overwrites its 2 bytes);
 *   lb_postprocess_u8: bf16 image in; non-finite pixels are still counted.
 */
int lb_latent_prep(lb_ctx* ctx, const void* x_nchw, int B, int C, int64_t hw, const void* w_f32,
                   const void* bias_f32, void* out_nchw, void* stream, int dtype);
int lb_softmax_rows(lb_ctx* ctx, const void* x, int64_t ld, int64_t rows, int cols, void* out, int64_t ldo,
                    void* stream, int dtype);
int lb_postprocess_u8(lb_ctx* ctx, const void* img_nchw, int B, int C, int64_t hw, void* out_u8_nhwc,
                      int* nonfinite_count_dev, void* stream, int dtype);
/* lb_nhwc_to_nchw: the first C (<= 8) columns of NHWC rows [B*hw, ld] -> NCHW [B, C, hw].  The C0 -> 4 (UNet eps) and
 * C0 -> 3 (VAE RGB) output convolutions run as lb_gemm with an 8-row zero-padded weight matrix (N = 8); this puts the
 * result back into the reference's [B,C,H,W] tensor layout. */
int lb_nhwc_to_nchw(lb_ctx* ctx, const void* x, int64_t ld, int B, int C, int64_t hw, void* out_nchw, void* stream,
                    int dtype);

/* ---- LPIPS-AlexNet branch-placement metric (SURVEY section 8f next #2; blending_engine.py:744-758, lpips==0.1.4) ----
 * The five AlexNet convolutions run on lb_gemm (LB_GEMM_RELU) over patch matrices:
 * lb_lpips_im2col_u8: conv1's patch matrix [Ho*Wo, out_cols] straight from the uint8 HxWx3 device frame with the
 *   reference's input arithmetic fused: ((2*u/255 - 1) - shift[c]) / scale[c] (blending_engine.py:750-755 + lpips
 *   ScalingLayer); column (ky*k + kx)*3 + c, zero columns up to out_cols, zero padding outside the frame.
 * lb_im2col: generic NHWC fp16 patch matrix [Ho*Wo, k*k*C], column (ky*k + kx)*C + c.
 * lb_maxpool3s2: MaxPool2d(3, stride 2) on an NHWC map.
 * lb_lpips_tap: one tap of the distance: mean over pixels of sum_c lin[c] * (a_c/(|a|+1e-10) - b_c/(|b|+1e-10))^2,
 *   written to (accumulate = 0) or added to (accumulate = 1) the device scalar out_scalar; deterministic.
 */
int lb_lpips_im2col_u8(lb_ctx* ctx, const void* frame_u8, int H, int W, int k, int stride, int pad,
                       const float* shift3, const float* scale3, void* out, int64_t out_cols, void* stream);
int lb_im2col(lb_ctx* ctx, const void* x, int64_t ld, int H, int W, int C, int k, int stride, int pad, void* out,
              void* stream);
int lb_maxpool3s2(lb_ctx* ctx, const void* x, int64_t ld, int H, int W, int C, void* out, int64_t ldo, void* stream);
size_t lb_lpips_tap_workspace_bytes(lb_ctx* ctx);
int lb_lpips_tap(lb_ctx* ctx, const void* feat_a, const void* feat_b, int64_t ld, int64_t rows, int C,
                 const float* lin_w, int accumulate, float* out_scalar, void* workspace, void* stream);

/* ---- frame fill of write_movie_transition (SURVEY section 8f next #3; blending_engine.py:684-706, utils.py:105-178) ----
 * out[t] = uint8( fl32(w0[t] * frames[left[t]]) + fl32(w1[t] * frames[left[t] + 1]) ), t < T, over frames of n bytes
 * (n % 16 == 0): numpy's float32 blend (w0 = float32(1 - f), w1 = float32(f), no FMA contraction) and its truncating
 * uint8 cast; w1 == 0 copies the key frame.  left / w0 / w1 are device arrays of length T.
 */
int lb_frames_lerp_u8(lb_ctx* ctx, const void* frames_u8, int64_t n, const int* left_idx_dev, const float* w0_dev,
                      const float* w1_dev, int T, void* out_u8, void* stream);

/* ---- UNet executor ---------------------------------------------------------------
 * A program is a flat list of the ops above over static device buffers (one
 * SDXL UNet forward for a fixed batch/height/width lowers to ~1.7k records).
 * lb_program_create validates every record and pre-encodes the TMA descriptors;
 * lb_program_run replays it on ``stream`` (``t`` = the timestep fed to
 * LB_OP_EMBED_INPUTS).  Replaces the module walk of pipe.unet(...)
 * (diffusers_holder.py:336-344).
 * lb_op.dtype: the ``dtype`` argument of the record's call for the kinds whose entry point takes one (above); it must
 * be 0 for every other kind (a GEMM takes its types from its mode flags).  Kinds 8 and 18 are retired.
 * LB_OP_CONV_IN_ADD (lb_conv_in_add) and LB_OP_COND_CONV (lb_cond_conv) use the ``conv`` member: CONV_IN_ADD reads
 * x, B, Cin, H, W, w, bias, Cout, out, ld_out, addend, ld_add (act must be 0); COND_CONV reads x, ld_x, B, Cin, H, W,
 * w, bias, Cout, out, ld_out, stride, in_u8 and act as lb_cond_conv's ``silu``.
 * LB_OP_IMAGE_CONV_IN (lb_image_conv_in) uses the ``conv`` member's x, ld_x, B, Cin, H, W, w, bias, Cout, out and
 * ld_out, with lb_op.dtype; LB_OP_IM2COL_S2_PAD01 (lb_im2col_s2_pad01) uses ``resample`` like LB_OP_IM2COL_S2.
 * LB_OP_ADD_ROWS_BCAST (lb_add_rows_bcast) uses ``aux``: out = dst, ld_out = ld_dst, x = src, ld_x = ld_src, B,
 * n = rows, C.  LB_OP_PIXEL_UNSHUFFLE_U8 (lb_pixel_unshuffle_u8) uses ``patch``: x = image, H, W, C = Cimg, k = r, out.
 * LB_OP_AVGPOOL2_CEIL (lb_avgpool2_ceil) uses ``patch`` like LB_OP_MAXPOOL3S2: x, ld_x, H, W, C, out, ld_out.
 */
enum {
    LB_OP_GEMM = 1, LB_OP_ATTENTION = 2, LB_OP_GROUPNORM = 3, LB_OP_LAYERNORM = 4, LB_OP_EMBED_INPUTS = 5,
    LB_OP_LINEAR_SMALL = 6, LB_OP_CONV_IN = 7, LB_OP_UPSAMPLE_NEAREST = 9, LB_OP_IM2COL_S2 = 10,
    LB_OP_LATENT_PREP = 11, LB_OP_SOFTMAX_ROWS = 12, LB_OP_POSTPROCESS_U8 = 13,
    LB_OP_LPIPS_IM2COL_U8 = 14, LB_OP_IM2COL = 15, LB_OP_MAXPOOL3S2 = 16, LB_OP_NHWC_TO_NCHW = 17,
    LB_OP_CONV_IN_ADD = 19, LB_OP_COND_CONV = 20, LB_OP_IMAGE_CONV_IN = 21, LB_OP_IM2COL_S2_PAD01 = 22,
    LB_OP_ADD_ROWS_BCAST = 23, LB_OP_PIXEL_UNSHUFFLE_U8 = 24, LB_OP_AVGPOOL2_CEIL = 25
};
typedef struct lb_op {
    int32_t kind;
    int32_t dtype;      /* LB_DTYPE_F16 (0) or LB_DTYPE_BF16, see above */
    union {
        lb_gemm_desc gemm;
        lb_attn_desc attn;
        struct { const void* x; int64_t ld_x; int64_t rows; /* HW per batch (GN) or total rows (LN) */
                 int32_t B, C, groups, silu; float eps; const void* gamma; const void* beta;
                 void* out; int64_t ld_out; void* workspace; } norm;
        struct { const void* text_embeds; const void* time_ids; int32_t B, dim_t, pooled, dim_a;
                 void* temb_in; void* add_in; } embed;
        struct { const void* x; int64_t ldx; int32_t M, K; const void* w; int64_t ldw; const void* bias;
                 const void* addend; int64_t ldadd; int32_t act_in, act_out; void* out; int64_t ldo; int32_t N; } lin;
        /* CONV_IN (act, in_scale: lb_conv_in's); CONV_IN_ADD and COND_CONV, see above */
        struct { const void* x; int64_t ld_x; int32_t B, Cin, H, W; const void* w; const void* bias;
                 int32_t Cout; void* out; int64_t ld_out; int32_t act; float in_scale;
                 const void* addend; int64_t ld_add; int32_t stride, in_u8; } conv;
        /* UPSAMPLE_NEAREST: output Ho x Wo (see lb_upsample_nearest); IM2COL_S2 and IM2COL_S2_PAD01: Ho, Wo unused */
        struct { const void* x; int64_t ld_x; int32_t B, H, W, C; void* out; int64_t ld_out; int32_t Ho, Wo; } resample;
        /* LATENT_PREP: x,w,bias,out,B,C,n=h*w; SOFTMAX_ROWS: x,ld_x,out,ld_out,n=rows,C=cols;
         * POSTPROCESS_U8: x,out,B,C,n=h*w, w = optional device int counter of non-finite pixels;
         * NHWC_TO_NCHW: x,ld_x,out,B,C,n=h*w */
        struct { const void* x; int64_t ld_x; const void* w; const void* bias; void* out; int64_t ld_out;
                 int64_t n; int32_t B, C; } aux;
        /* LPIPS_IM2COL_U8 (x = uint8 frame, C = out_cols, f = shift[3], scale[3]); IM2COL; MAXPOOL3S2 (k/stride/pad unused) */
        struct { const void* x; int64_t ld_x; int32_t H, W, C, k, stride, pad; void* out; int64_t ld_out;
                 float f[6]; } patch;
    } u;
} lb_op;
typedef struct lb_program lb_program;
int     lb_program_create(lb_ctx* ctx, const lb_op* ops, int64_t n_ops, lb_program** out);
int     lb_program_run(lb_program* prog, float t, void* stream);
/* replay mode of lb_program_run: 1 = one CUDA-graph launch per run (captured on the second run, every launch keeps its
 * programmatic-dependent-launch edge), 0 = not captured yet, -1 = direct launches (capture unavailable or LB_NO_GRAPH) */
int     lb_program_is_graph(lb_program* prog);
/* profiling aid: replay only the ops whose kind bit (1u << LB_OP_*) is set in kind_mask */
int     lb_program_run_kinds(lb_program* prog, float t, uint32_t kind_mask, void* stream);
int64_t lb_program_count_kinds(lb_program* prog, uint32_t kind_mask);
int64_t lb_program_num_launches(lb_program* prog);
int     lb_program_destroy(lb_program* prog);

/* Reads and clears the device-side protocol-error flag the pipelined kernels
 * set before trapping (0 = no error).  Synchronises the device: debug only. */
int lb_ctx_error_flag(lb_ctx* ctx, int* out_code);

#ifdef __cplusplus
}
#endif
#endif /* LB200_H */
