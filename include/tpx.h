/* libtpx_b200 — C ABI of the H100-native 3DTopia-XL denoising hot path (DiT step, sampler update, VAE decode).
 *
 * The reference has NO C/FFI interface for this path: its boundary is a set of Python objects resolved by
 * dva/io.py:22-28 (`load_from_config`).  Each entry point below therefore cites the reference *Python*
 * interface it stands behind; the Python mirror of those interfaces (3dtopia-xl_b200/{dit,diffusion,vae}.py)
 * is a thin ctypes caller of this header.  INTEGRATION.md shows the binding a maintainer adds.
 *
 * Conventions: plain pointers and sizes only; every pointer named *dev* / documented "device" is a CUDA
 * device pointer on the current device; `stream` is a cudaStream_t passed as void* (NULL = legacy default
 * stream); all work is enqueued asynchronously on that stream, no host synchronisation, no allocation
 * inside hot calls (workspaces are caller-allocated, sizes from *_workspace_bytes); functions return 0 or a
 * negative TPX_ERR_* code and never throw; tpx_last_error() gives the thread-local message.
 * Handles are not thread-safe; distinct handles are independent.  Device code is sm_90a only: every entry
 * that launches work fails with TPX_ERR_CUDA on any other device — there is no CPU or other-arch fallback.
 */
#ifndef TPX_B200_H
#define TPX_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TPX_VERSION 100 /* 0.1.0 */

enum { TPX_OK = 0, TPX_ERR_ARG = -1, TPX_ERR_CUDA = -2, TPX_ERR_SHAPE = -3, TPX_ERR_STATE = -4, TPX_ERR_KEY = -5 };
enum { TPX_DTYPE_F32 = 0, TPX_DTYPE_F16 = 1 };

int tpx_version(void);
const char* tpx_last_error(void);
/* 0 if the current device can run the kernels (compute capability 9.0), else TPX_ERR_CUDA. */
int tpx_device_check(void);
/* Measurement hooks (bench.py): total kernels launched by this library so far; and an optional mode that brackets
 * every launch with a CUDA event pair on its stream.  profile_end synchronises the device and returns, per kernel
 * class, the summed device time (ms) and launch count.  Classes: 0 wgmma GEMM, 1 attention, 2 LayerNorm+modulate,
 * 3 GEMV/embedders, 4 CFG/sampler, 5 implicit-GEMM conv, 6 GroupNorm, 7 other VAE. */
#define TPX_PROF_NCLASS 8
int64_t tpx_launch_count(void);
int tpx_profile_begin(void);
int tpx_profile_end(float* ms_by_class, int64_t* launches_by_class);

/* ------------------------------------------------------------------------------------------------------------
 * DiT  — models/dit_crossattn.py:111-213 (class DiT), constructor kwargs as in configs/inference_dit.yml:52-62
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct tpx_dit tpx_dit;
typedef struct tpx_dit_config {
    int32_t seq_length;         /* N   (2048) */
    int32_t in_channels;        /* 68  */
    int32_t out_channels;       /* 136 = 2*in (learn_sigma) */
    int32_t condition_channels; /* 768 */
    int32_t hidden_size;        /* 1152 */
    int32_t depth;              /* 28 */
    int32_t num_heads;          /* 16 */
    int32_t mlp_hidden;         /* 4608 */
} tpx_dit_config;

/* DiT.__init__ (dit_crossattn.py:115-156): allocates the packed fp16 parameter store on the current device. */
int tpx_dit_create(const tpx_dit_config* cfg, tpx_dit** out);
void tpx_dit_destroy(tpx_dit* h);
/* nn.Module.load_state_dict (inference.py:262, sd['ema']): one call per reference key
 * ("blocks.3.crossattn.to_q.weight", "final_layer.linear.bias", "null_cond_embedding", ...).  `dev_ptr` is a
 * contiguous device tensor of dtype TPX_DTYPE_*; shape is checked against the module tree.  Unknown key -> TPX_ERR_KEY. */
int tpx_dit_set_weight(tpx_dit* h, const char* ref_key, const void* dev_ptr, int dtype, const int64_t* shape, int ndim, void* stream);
/* Read a parameter back from the packed store (fp16 values, written as `dtype`) into dst_dev (same element count as the key's
 * reference shape).  Lets the host mirror drop its copy of the checkpoint after ingestion (SURVEY.md §8f-4) and still answer
 * state_dict() / move between devices. */
int tpx_dit_get_weight(tpx_dit* h, const char* ref_key, void* dst_dev, int dtype, void* stream);
/* Call once after the last set_weight: checks every required key arrived, derives the per-block constant of the
 * all-null cross-attention (proj(to_v(null_cond_embedding)), SURVEY §8a a8). */
int tpx_dit_finalize(tpx_dit* h, void* stream);

/* Bytes of the persistent conditioning store for `n_cross` sequences with `M` context tokens, and of the per-call
 * scratch for `n_seq` sequences (n_seq = 2*B under CFG). */
size_t tpx_dit_cond_bytes(const tpx_dit* h, int n_cross, int M);
size_t tpx_dit_workspace_bytes(const tpx_dit* h, int n_seq);
/* Hoist of MemEffCrossAttention.to_k/to_v (attention.py:106-107) for all blocks: they depend only on the context y,
 * so they are computed once per image instead of once per step.  y: device fp32 [n_cross, M, condition_channels]. */
int tpx_dit_set_cond(tpx_dit* h, const float* y_dev, int n_cross, int M, void* cond_ws, size_t cond_bytes, void* stream);

/* DiT.forward (dit_crossattn.py:184-202) when use_cfg == 0, DiT.forward_with_cfg (:204-213) when use_cfg != 0.
 *   x   device fp32 [B, N, in_channels];  t  device int64 [B] (ORIGINAL-schedule timesteps);
 *   out device fp16 [B, N, out_channels].
 * use_cfg == 0 : B sequences, all attend to the stored context (set_cond n_cross == B).
 * use_cfg == 1 : batch [x;x], context [y;null]; the null half uses the derived constant (n_cross == B).
 * use_cfg == 2 : same, but the null half runs real cross-attention (set_cond was given [y;null], n_cross == 2B);
 *                exists so tests can check the constant identity on the device. */
int tpx_dit_forward(tpx_dit* h, const float* x_dev, const int64_t* t_dev, int B, int use_cfg, float cfg_scale, void* out_f16_dev, void* ws,
                    size_t ws_bytes, void* stream);
/* Hoist of TimestepEmbedder (models/utils.py:27-64) and of every adaLN_modulation Linear (dit_crossattn.py:40-43,54 and :66-69,75)
 * out of the sampling loop: they depend only on the timestep, and a sampling loop visits a fixed list of them
 * (SpacedDiffusion.timestep_map, respace.py:73-87; gaussian_diffusion.py:674-685 feeds the same t to the whole batch).
 * tpx_dit_set_timesteps computes the [K, 28*9*D + 2*D] fp16 modulation rows of K original-schedule timesteps (host int64 array)
 * into caller memory `ts_ws` (256-B aligned, tpx_dit_timesteps_bytes(h, K) bytes, must stay alive and untouched while used) with
 * the same kernels and the same per-element arithmetic a forward uses, 8 timesteps per pass over the 669 MB of adaLN weights.
 * tpx_dit_forward_step is tpx_dit_forward for a batch whose B samples all sit at timestep `t`: it reads the row of `t` from that
 * table instead of running the timestep MLP and the adaLN pass (results are bit-identical to tpx_dit_forward).  `t` must be one
 * of the K values (TPX_ERR_STATE otherwise); loading a weight invalidates the table. */
size_t tpx_dit_timesteps_bytes(const tpx_dit* h, int K);
int tpx_dit_set_timesteps(tpx_dit* h, const int64_t* t_host, int K, void* ts_ws, size_t ts_bytes, void* stream);
int tpx_dit_forward_step(tpx_dit* h, const float* x_dev, int64_t t, int B, int use_cfg, float cfg_scale, void* out_f16_dev, void* ws, size_t ws_bytes,
                         void* stream);
/* Debug / parity.  tpx_dit_debug_stage runs tpx_dit_forward's schedule (same arguments, same launches) up to a stop and returns,
 * leaving the workspace as it stands: TPX_DIT_STAGE_EMBED after the token embedding (`block` is ignored), or after the gated GEMM
 * that adds block `block`'s CROSS, SELF or MLP branch to the residual stream.  A bad stage or block is TPX_ERR_ARG.
 * tpx_dit_debug_tap copies the leading `count` (1..n_seq) sequences or samples of one buffer of the workspace `ws` carved for n_seq
 * sequences into dst_dev:
 *   RESIDUAL  fp32 [count, N, hidden]   the residual stream;
 *   ATTN_OUT  fp16 [count, N, hidden]   the attention output before proj, head j in columns [j*Dh, (j+1)*Dh), after a CROSS stop
 *                                       (the first n_cross sequences hold it) or a SELF stop;
 *   MOD       fp16 [count, 28*9*D + 2*D] the modulation rows of the batch's samples (a forward given device timesteps);
 *   PRE_CFG   fp16 [count, N, out_channels] the [cond; uncond] output before guidance, after a full forward with use_cfg != 0. */
enum { TPX_DIT_STAGE_EMBED = 0, TPX_DIT_STAGE_CROSS = 1, TPX_DIT_STAGE_SELF = 2, TPX_DIT_STAGE_MLP = 3 };
enum { TPX_DIT_TAP_RESIDUAL = 0, TPX_DIT_TAP_ATTN_OUT = 1, TPX_DIT_TAP_MOD = 2, TPX_DIT_TAP_PRE_CFG = 3 };
int tpx_dit_debug_stage(tpx_dit* h, const float* x_dev, const int64_t* t_dev, int B, int use_cfg, int block, int stage, void* ws, size_t ws_bytes,
                        void* stream);
int tpx_dit_debug_tap(const tpx_dit* h, const void* ws, int n_seq, int which, int count, void* dst_dev, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Sampler update — models/diffusion/gaussian_diffusion.py:255-338 (p_mean_variance, LEARNED_RANGE variance),
 * :531-578 (ddim_sample), :397-440 (p_sample).  Coefficients are the float64 tables evaluated at the step and
 * rounded to fp32 exactly like _extract_into_tensor (:880-892); the host mirror computes them.
 * pred_xstart = sqrt_ab * x - sqrt_1mab * model_out (one rounding per op): with (sqrt(ab), sqrt(1-ab)) this is VELOCITY (:340-344, the
 * released model), with (sqrt(1/ab), sqrt(1/ab-1)) EPSILON (:346-351), with (0, -1) START_X (:319-320); clip != 0 clamps it to [-1, 1]
 * (process_xstart, :310-315).
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct tpx_sampler_coefs {
    float sqrt_ab, sqrt_1mab, sqrt_recip_ab, sqrt_recipm1_ab;
    float c_x0, c_eps, sigma, nonzero; /* DDIM: sqrt(ab_prev), sqrt(1-ab_prev-sigma^2), sigma, (t != 0) */
    float coef1, coef2, min_log, max_log; /* DDPM: posterior mean coefficients, log-variance range */
    int32_t clip;
} tpx_sampler_coefs;
/* x, noise (may be NULL), x_prev, pred_x0: device fp32 [n]; model_out: device [n/C tokens, 2C] fp16 or fp32. */
int tpx_sampler_step(int ddim, const float* x_dev, const void* model_out_dev, int model_out_dtype, const float* noise_dev, int64_t n, int C,
                     const tpx_sampler_coefs* k, float* x_prev_dev, float* pred_x0_dev, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Sample -> decode glue (SURVEY §8a a13 / a15) — inference.py:328-332,343-348 ; app.py:119-123,134-139
 * ---------------------------------------------------------------------------------------------------------- */
/* a13: sample device fp32 [T, C] (T = batch * num_prims, C = 68).  With per-channel statistics (mean/std device fp32 [C]):
 * v = sample * inv_nf * std + mean, one rounding per op as the reference's eager CUDA ops (x / python_float = x * fp32(1/nf));
 * without (mean == std == NULL): srt = sample[:, 0:4], z = sample[:, 4:] * inv_nf (inference.py:337).
 * Outputs: srt device fp32 [T, 4] = (scale, xyz), z device fp32 [T, C-4] = the [T,1,4,4,4] latents VAE.decode takes. */
int tpx_latent_split(const float* sample_dev, const float* mean_dev, const float* std_dev, float inv_nf, int64_t T, int C, float* srt_dev,
                     float* z_dev, void* stream);
/* a15: decoded device [T, F] (F = 6 * vox, NCDHW per primitive = channel-major; dtype fp32 or fp16) -> out device fp32 [T, 4 + F] =
 * [srt | sdf/5 | (rgb+1)/2 | (mat+1)/2], the PrimSDF / ray-marcher layout (models/primsdf.py:28-33).  srt_fix != 0 applies
 * srt[:, 0] = srt[:, 0] / 10 + 0.05 (checkpoints without per-channel statistics, inference.py:343-344). */
int tpx_primvolume_pack(const float* srt_dev, const void* decoded_dev, int decoded_dtype, int64_t T, int F, int vox, int srt_fix, float* out_dev,
                        void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * VAE decoder — models/vae3d_dib.py:391-440 (class VAE), :330-387 (Decoder)
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct tpx_vae tpx_vae;
typedef struct tpx_vae_config {
    int32_t latent_channels; /* 1 */
    int32_t out_channels;    /* 6 */
    int32_t ch_mid;          /* up_channels[0] = 256 */
    int32_t ch_out;          /* up_channels[1] = 32 */
    int32_t attn_heads;      /* 8 */
} tpx_vae_config;
int tpx_vae_create(const tpx_vae_config* cfg, tpx_vae** out);
void tpx_vae_destroy(tpx_vae* h);
/* load_state_dict(sd['model_state_dict']) (inference.py:258): decoder.* / post_quant_conv.* keys are consumed,
 * encoder.* / quant_conv.* keys are accepted and ignored (return 1). */
int tpx_vae_set_weight(tpx_vae* h, const char* ref_key, const void* dev_ptr, int dtype, const int64_t* shape, int ndim, void* stream);
int tpx_vae_finalize(tpx_vae* h, void* stream);
size_t tpx_vae_workspace_bytes(const tpx_vae* h, int P);
/* VAE.decode (vae3d_dib.py:437-440): z device [P,1,4,4,4] (dtype z_dtype) -> out device [P,6,8,8,8] (dtype out_dtype). */
int tpx_vae_decode(tpx_vae* h, const void* z_dev, int z_dtype, void* out_dev, int out_dtype, int P, void* ws, size_t ws_bytes, void* stream);
/* Debug / parity: run the decode schedule through `stage` (the same launches tpx_vae_decode makes up to that point) and copy that
 * stage's activation, channels-last fp16 [P, S^3, C], into tap_f16_dev.  Stages (Decoder.forward, vae3d_dib.py:369-387):
 *   0 conv_in [P,64,256]; 1, 3 mid_block res 0 / 1 and 2 its attention [P,64,256]; 4, 5 up_blocks.0 res 0 / 1 [P,64,256];
 *   6 up_blocks.0 upsample [P,512,256]; 7, 8 up_blocks.1 res 0 (with its 1x1 shortcut) / 1 [P,512,32]; 9 norm_out + SiLU [P,512,32].
 * The decoder's output after stage 9 is tpx_vae_decode's. */
enum {
    TPX_VAE_STAGE_CONV_IN = 0, TPX_VAE_STAGE_MID_RES0 = 1, TPX_VAE_STAGE_MID_ATTN = 2, TPX_VAE_STAGE_MID_RES1 = 3, TPX_VAE_STAGE_UP0_RES0 = 4,
    TPX_VAE_STAGE_UP0_RES1 = 5, TPX_VAE_STAGE_UPSAMPLE = 6, TPX_VAE_STAGE_UP1_RES0 = 7, TPX_VAE_STAGE_UP1_RES1 = 8, TPX_VAE_STAGE_NORM_OUT = 9
};
int tpx_vae_debug_stage(tpx_vae* h, const void* z_dev, int z_dtype, int P, int stage, void* tap_f16_dev, void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * VAE encoder — models/vae3d_dib.py:431-435 (VAE.encode), :270-327 (Encoder), :147-184 (DownBlock), :428 (quant_conv).
 * A handle of its own, so the decoder handle's keys, return codes and workspace are untouched.  The config is tpx_vae_config with
 * out_channels = the encoder's in_channels (6), ch_out / ch_mid = down_channels (32 / 256), latent_channels 1, attn_heads 8.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct tpx_vae_encoder tpx_vae_encoder;
int tpx_vae_encoder_create(const tpx_vae_config* cfg, tpx_vae_encoder** out);
void tpx_vae_encoder_destroy(tpx_vae_encoder* h);
/* encoder.* / quant_conv.* keys are consumed (the stride-2 downsample weight is repacked for its space-to-depth input);
 * decoder.* / post_quant_conv.* keys are accepted and ignored (return 1). */
int tpx_vae_encoder_set_weight(tpx_vae_encoder* h, const char* ref_key, const void* dev_ptr, int dtype, const int64_t* shape, int ndim, void* stream);
int tpx_vae_encoder_finalize(tpx_vae_encoder* h, void* stream);
size_t tpx_vae_encoder_workspace_bytes(const tpx_vae_encoder* h, int P);
/* VAE.encode up to the posterior's parameters (vae3d_dib.py:431-433): x device [P,6,8,8,8] (dtype x_dtype) -> moments device
 * [P,2,4,4,4] (dtype out_dtype) = quant_conv(encoder(x)); channel 0 is the mean, 1 the (unclamped) log-variance. */
int tpx_vae_encode(tpx_vae_encoder* h, const void* x_dev, int x_dtype, void* moments_dev, int out_dtype, int P, void* ws, size_t ws_bytes, void* stream);
/* Debug / parity: run the encode schedule through `stage` and copy that stage's channels-last fp16 activation [P, S^3, C] into
 * tap_f16_dev.  Stages (Encoder.forward, vae3d_dib.py:310-327): 0 conv_in, 1 / 2 down_blocks.0 res 0 / 1 [P,512,32];
 * 3 down_blocks.0 downsample [P,64,32]; 4 / 5 down_blocks.1 res 0 (with its 1x1 shortcut) / 1, 6 mid_block res 0, 7 its attention,
 * 8 mid_block res 1, 9 norm_out + SiLU [P,64,256].  conv_out + quant_conv after stage 9 give tpx_vae_encode's output. */
enum {
    TPX_VAE_ENC_STAGE_CONV_IN = 0, TPX_VAE_ENC_STAGE_DOWN0_RES0 = 1, TPX_VAE_ENC_STAGE_DOWN0_RES1 = 2, TPX_VAE_ENC_STAGE_DOWNSAMPLE = 3,
    TPX_VAE_ENC_STAGE_DOWN1_RES0 = 4, TPX_VAE_ENC_STAGE_DOWN1_RES1 = 5, TPX_VAE_ENC_STAGE_MID_RES0 = 6, TPX_VAE_ENC_STAGE_MID_ATTN = 7,
    TPX_VAE_ENC_STAGE_MID_RES1 = 8, TPX_VAE_ENC_STAGE_NORM_OUT = 9
};
int tpx_vae_encode_debug_stage(tpx_vae_encoder* h, const void* x_dev, int x_dtype, int P, int stage, void* tap_f16_dev, void* ws, size_t ws_bytes,
                               void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Per-kernel entry points (unit parity tests; each is one launch of one hot-path kernel)
 * ---------------------------------------------------------------------------------------------------------- */
/* out[M,N] fp16 = act(A[M,K] W[N,K]^T + bias) ; act: 0 none (optionally * post_scale, re-rounded), 1 GELU-tanh.  tile_n: 0 = auto.
 * For the three linear entries: K % 8 == 0 and N % 8 == 0 (any K tail is zero-filled by the TMA, K = 32 included); lda, ldo, ldx are
 * row strides in elements with 16-B aligned rows, and only columns < K of A and [M, N] of the output are touched.  An explicit tile_n
 * with no kernel for the epilogue (128 / 144 / 192 / 256 for every epilogue; 32 for tpx_linear with act 0 only) is TPX_ERR_SHAPE, before any
 * launch. */
int tpx_linear(const void* A_f16, int lda, const void* W_f16, const void* bias_f16, void* out_f16, int ldo, int M, int N, int K, int act,
               float post_scale, int tile_n, void* stream);
/* xres[M,N] fp32 += h(gate[(row/rows_per_batch)%gate_batches, :] * h(A W^T + bias))   (DiTBlock residual, dit_crossattn.py:55-57) */
int tpx_linear_gated(const void* A_f16, int lda, const void* W_f16, const void* bias_f16, const void* gate_f16, int gate_bstride, int gate_batches,
                     int rows_per_batch, float* xres, int ldx, int M, int N, int K, int tile_n, void* stream);
/* Column-split + head-split store: col -> (which = col / split_cols, head, d); row -> (b = row / n_seq_tokens, n);
 * out{which}[b, head, n, DhP] (zero padded).  post_scale applies to which == 0 (attention.py:105).  The column group
 * `transposed_which` (-1 = none) is stored transposed as [b, head, DhP, transposed_ld] (tokens contiguous, transposed_ld >= n_seq_tokens):
 * the V operand layout of tpx_attention_tc.  M must be a whole number of sequences.  Its token columns [n_seq_tokens, transposed_ld):
 * when Dh % 24 == 0 and n_seq_tokens % 32 == 0 (the 24-column bulk-store epilogue) every output is cleared first, so they are zero;
 * otherwise they are left as the caller had them (tpx_attention_tc only needs them finite). */
int tpx_linear_heads(const void* A_f16, int lda, const void* W_f16, const void* bias_f16, void* out0, void* out1, void* out2, int M, int N, int K,
                     int split_cols, int H, int Dh, int DhP, int n_seq_tokens, float post_scale, int tile_n, int transposed_which, int transposed_ld,
                     void* stream);
/* y = LN(x; eps) * h(1 + scale) + shift -> fp16   (modulate(norm(x), shift, scale), utils.py:19-20) */
int tpx_ln_modulate(float* x, int rows, int D, float eps, const void* shift_f16, const void* scale_f16, int mod_bstride, int rows_per_batch,
                    int mod_batches, void* out_f16, const void* pre_gate_f16, const void* pre_const_f16, int pre_row0, void* stream);
/* memory_efficient_attention contract (attention.py:54,109): q [B,H,Nq,DhP], k/v [B,H,Nk,DhP] -> out [B,Nq,H*Dh].  Padding: q k^T runs
 * over all DhP columns, so q and k columns d >= Dh must be zero; v columns d >= Dh never reach the output (any value, NaN included). */
int tpx_attention(const void* q, const void* k, const void* v, void* out, int B, int H, int Nq, int Nk, int Dh, int DhP, float scale, void* stream);
/* Same contract on the wgmma path (Dh == 72, the released model's head size, or 64): q,k [B,H,N,80]; vT = V transposed
 * [B,H,80,NkPad], NkPad % 8 == 0.  q / k columns d >= Dh must be zero (q k^T runs over all 80); vT rows d >= Dh and key columns
 * >= Nk only have to be finite. */
int tpx_attention_tc(const void* q, const void* k, const void* vT, void* out, int B, int H, int Nq, int Nk, int NkPad, int Dh, float scale, void* stream);
/* out = h(uncond + h(s * h(cond - uncond)))  over [cond; uncond] halves of n_half elements (dit_crossattn.py:210-213) */
int tpx_cfg_combine(const void* both_f16, int64_t n_half, float s, void* out_f16, void* stream);
/* GroupNorm(groups, eps, affine) [+ SiLU] on a channels-last fp16 volume [P, S3, C]  (vae3d_dib.py:109,112,131-139) */
int tpx_groupnorm_silu(const void* x_f16, const void* gamma_f16, const void* beta_f16, int P, int S3, int C, int groups, float eps, int apply_silu,
                       void* out_f16, void* stream);
/* 3x3x3 / pad 1 convolution as implicit GEMM on a channels-last fp16 volume [P,S,S,S,C] (S in {4,8});
 * W_f16 is [Cout, 27*C] with k = tap*C + c, tap = (kz*3+ky)*3+kx;  out [P,S,S,S,Cout] fp16 = (conv + bias (+ resid)) * alpha. */
int tpx_conv3d_k3(const void* x_f16, const void* W_f16, const void* bias_f16, const void* resid_f16, float alpha, void* out_f16, int P, int S, int C,
                  int Cout, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * PrimSDF point query — models/primsdf.py:52-109 (PrimSDF.forward = prim_weight + grid_sample_feat), the consumer of
 * the decoded voxels (SURVEY.md §8f-1).  x device fp32 [n,3]; srt device fp32 [K,4] = (scale, tx, ty, tz), 16-B aligned;
 * feat device fp32 [K, dim_feat*S^3] channel-major (inference.py:347); out device fp32 [n, dim_feat]:
 * column 0 = sdf, 1..3 = rgb clipped to [0,1], 4..5 = roughness/metallic clipped.  inference != 0 applies the
 * nearest-voxel SDF approximation to points no primitive covers (primsdf.py:82-101).
 * ---------------------------------------------------------------------------------------------------------- */
int tpx_primsdf_query(const float* x_dev, const float* srt_dev, const float* feat_dev, int64_t n, int K, int S, int dim_feat, int inference,
                      float* out_dev, void* stream);
/* Grid-binned version of the same query (the survey's binned gather, models/primsdf.py:104-109 / inference.py:108-116): a 32^3
 * grid over the primitives' bounding box holds, per cell, the ascending lists of primitives whose box meets the cell and of the
 * primitives that can be the nearest centre for a point of the cell; tpx_primsdf_grid_build derives them from srt on the device
 * (rebuild whenever srt changes), tpx_primsdf_query_grid walks the lists of the point's cell.  Results are identical to
 * tpx_primsdf_query (same arithmetic in the same order); points outside the grid and over-full lists take the exhaustive loop.
 * grid_ws: 256-B aligned device memory of tpx_primsdf_grid_bytes(cap_entries) bytes (8 M entries cover the shipped 2048 boxes). */
size_t tpx_primsdf_grid_bytes(int64_t cap_entries);
int tpx_primsdf_grid_build(const float* srt_dev, int K, void* grid_ws, size_t grid_bytes, void* stream);
int tpx_primsdf_query_grid(const float* x_dev, const float* srt_dev, const float* feat_dev, const void* grid_ws, size_t grid_bytes, int64_t n, int K, int S,
                           int dim_feat, int inference, float* out_dev, void* stream);
/* Backward of the point query: models/primsdf.py:52-109 under autograd, what PrimSDFLoss (dva/losses.py:102-148: SDF L1 in the
 * shape phase, tex / mat L1 in the texture phase) fits primitives through.  Inputs as tpx_primsdf_query_grid, with grid_ws the
 * workspace the forward used, or NULL for the exhaustive walk (the forward of K > 4096 primitives, tpx_primsdf_query);
 * grad_out device fp32 [n,6], the upstream gradient of (sdf, rgb, roughness, metallic).  ADDS into caller-zeroed grad_x [n,3],
 * grad_srt [K,4] and grad_feat [K,6*S^3]; each may be NULL when that gradient is not needed.  Every point walks the primitives the
 * forward walked, through the same device code (cover test, boundary re-decision, nearest primitive and voxel).  With
 * l = (x - pos)/s, w_j = 1 - |l_j|_inf over the covering j, W = sum w_j + 1e-6, v_jc the trilinear sample, o_c = sum w_j v_jc / W and
 * g_c = 0 for c >= 1 where o_c is outside [0,1]:
 *   dL/dv_jc = g_c w_j / W (scattered to the 8 corners of channel c of feat[j]); dL/dw_j = sum_c g_c (v_jc - o_c) / W;
 *   dL/dl_j = sum_c (g_c w_j / W) dv_jc/dl - dL/dw_j sign(l_jd) [|l_jd| = max] / (tied axes);
 *   dL/dx += dL/dl_j / s_j, dL/dpos_j -= dL/dl_j / s_j, dL/ds_j -= (dL/dl_j . l_j) / s_j.
 * Uncovered points: nothing when inference == 0; at inference (sdf = f + d sign(f), d = |x - c|, c = pos_k + s_k grid_v,
 * u = (x - c)/d, 0 at d = 0): dL/dfeat[k, v] += g_0, dL/dx += g_0 sign(f) u, dL/dpos_k -= g_0 sign(f) u, dL/ds_k -= g_0 sign(f) u . grid_v.
 * grad_srt / grad_feat are fp32 atomic reductions: their last bits vary from run to run. */
int tpx_primsdf_query_backward(const float* x_dev, const float* srt_dev, const float* feat_dev, const void* grid_ws, size_t grid_bytes, int64_t n, int K,
                               int S, int dim_feat, int inference, const float* grad_out_dev, float* grad_x_dev, float* grad_srt_dev, float* grad_feat_dev,
                               void* stream);
/* The sdf column of the same query on the R x R x R lattice (coords[i], coords[j], coords[k]) that extract_texmesh evaluates
 * (inference.py:106-116: linspace / meshgrid(indexing='ij') points in 8192-point chunks, reshape(R,R,R)), without materialising the
 * points: grid_out device fp32 [R,R,R], grid_out[i,j,k] = sdf at (x, y, z) = (coords[i], coords[j], coords[k]); coords device fp32 [R]
 * (the caller's linspace).  Bit-identical to column 0 of tpx_primsdf_query_grid / tpx_primsdf_query on those points.  grid_ws as for
 * tpx_primsdf_query_grid (built from the same srt), or NULL for the exhaustive loop. */
int tpx_primsdf_sdf_grid(const float* coords_dev, int R, const float* srt_dev, const float* feat_dev, const void* grid_ws, size_t grid_bytes, int K, int S,
                         int dim_feat, int inference, float* grid_out_dev, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Ray-march preview — RayMarcher.forward (dva/ray_marcher.py:142-229) = compute_raydirs (dva/mvp/extensions/utils/
 * utils_kernel.cu:15-55) + mvpraymarch(algo 0, usebvh "fixedorder", chlast, maxhitboxes 512, blocksize (8,16))
 * (dva/mvp/extensions/mvpraymarch/mvpraymarch_subset_kernel.h:14-101): called on every 10th denoising step and for the
 * turntable (inference.py:349-350).  One batch element per blockIdx.z; all pointers device fp32, contiguous:
 * template channels-last [N,K,S,S,S,4]; primpos [N,K,3] ALREADY divided by volradius (as the reference passes it),
 * primrot [N,K,3,3], primscale [N,K,3]; camera as convert_camera_parameters returns it (campos [N,3] in world units,
 * camrot [N,3,3], focal [N,2] = diagonal of K[:2,:2], princpt [N,2]); pixel (w,h) -> ray through (w,h); stepsize = dt / volradius.
 * rgba_out [N,H,W,4] (the reference's rayrgba; RayMarcher permutes it to [N,4,H,W]).  Each 8 x 4-pixel warp visits the
 * primitives whose box any of its rays meets, in the "fixedorder" tree's leaf order (ascending index rotated by
 * 2^ceil(log2 K) - K, so ascending when K is a power of two), at most the first 512 of them.
 * ---------------------------------------------------------------------------------------------------------- */
int tpx_raymarch_preview(const float* template_chlast, const float* primpos, const float* primrot, const float* primscale, const float* campos,
                         const float* camrot, const float* focal, const float* princpt, int N, int K, int S, int H, int W, float volradius, float stepsize,
                         float fadescale, float fadeexp, float* rgba_out, void* stream);
/* The same march, saving what the backward needs (MVPRaymarch.forward with gradmode, dva/mvp/extensions/mvpraymarch/mvpraymarch.py:
 * 74-150), with subsampled rays (dva/ray_marcher.py:33-73,174-190).  Arguments as tpx_raymarch_preview, plus:
 *   stride >= 1 (ray_subsample_factor): rgba_out is [N,h,w,4] with h = H / stride, w = W / stride (h, w >= 1), and output pixel (j,i)
 *   traces the ray through image pixel (x0 + stride j, y0 + stride i) -- the pixel_coords that subsample_pixel_coords /
 *   resize_pixel_coords hand to compute_raydirs; the hit list is per warp of 8 x 4 OUTPUT pixels, as the reference's;
 *   offsets: device int32 [N,2] per-image (x0, y0), each in [0, stride) (read by the kernel, not checked here), or NULL for (0, 0);
 *   raysat_out: device fp32 [N,h,w,3] or NULL: PrimAccumAdditive's saturation colour (primaccum.h:63-79), the rgb of the first sample
 *   whose accumulated alpha reaches 1, or (-1,-1,-1) if the ray never saturates.
 * With stride 1, offsets NULL and raysat_out NULL the image is tpx_raymarch_preview's, bit for bit. */
int tpx_raymarch_forward(const float* template_chlast, const float* primpos, const float* primrot, const float* primscale, const float* campos,
                         const float* camrot, const float* focal, const float* princpt, int N, int K, int S, int H, int W, float volradius, float stepsize,
                         float fadescale, float fadeexp, int stride, const int* offsets, float* rgba_out, float* raysat_out, void* stream);
/* Backward of tpx_raymarch_forward (MVPRaymarch.backward, mvpraymarch.py:152-213 -> raymarch_subset_backward_kernel with forwarddir,
 * mvpraymarch_subset_kernel.h:103-217, primaccum.h:81-98, primsampler.h:68-91, primtransf.h:155-179).  Inputs: the forward's, its
 * raysat [N,h,w,3] and grad_rgba [N,h,w,4] (16-B aligned).  ADDS into caller-zeroed grad_template (channels-last [N,K,S,S,S,4], 16-B
 * aligned), grad_primpos [N,K,3] (per unit of primpos / volradius, the units the march sees), grad_primrot [N,K,3,3] and
 * grad_primscale [N,K,3].  The ray's march is repeated from the same first step through the same device code, so every inside test,
 * saturation and step count is the forward's.  Per listed primitive and step, with acc the alpha accumulated before the sample:
 *   sat = acc + a dt >= 1; dL_rgb = (sat ? 1 - acc : a dt) dL.rgb; dL_a = sat ? 0 : dt ((rgb,1) - (raysat valid ? (raysat,1) : 0)) . dL;
 *   dL_y += -fadescale fadeexp |y|^(fadeexp-1) sign(y) a dL_a; the template gets the trilinear scatter of (dL_rgb, fade dL_a) and
 *   dL_y the trilinear weights' derivative x (S-1)/2; grad_scale += (R^T (x - t)) * dL_y; dL_y *= s; grad_rot[r] += (x - t)[r] dL_y;
 *   grad_pos -= R dL_y.
 * Camera gradients are not computed (the reference returns None for them).  Floating-point atomics: the summation order, and so the
 * last bits of the gradients, vary from run to run. */
int tpx_raymarch_backward(const float* template_chlast, const float* primpos, const float* primrot, const float* primscale, const float* campos,
                          const float* camrot, const float* focal, const float* princpt, int N, int K, int S, int H, int W, float volradius, float stepsize,
                          float fadescale, float fadeexp, int stride, const int* offsets, const float* raysat, const float* grad_rgba,
                          float* grad_template, float* grad_primpos, float* grad_primrot, float* grad_primscale, void* stream);
/* tpx_raymarch_preview for N images of N / views primitive sets: image n marches primitive set n / views (template, primpos, primrot,
 * primscale hold N / views sets) through camera n (campos, camrot, focal, princpt hold N cameras).  views >= 1 divides N.  A
 * turntable of V views of one set is one launch over one template, bit-identical to V tpx_raymarch_preview calls; views = 1 is
 * tpx_raymarch_preview. */
int tpx_raymarch_preview_views(const float* template_chlast, const float* primpos, const float* primrot, const float* primscale, const float* campos,
                               const float* camrot, const float* focal, const float* princpt, int N, int views, int K, int S, int H, int W,
                               float volradius, float stepsize, float fadescale, float fadeexp, float* rgba_out, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Preview payloads (dva/visualize.py), forward only.  All pointers device fp32, contiguous.
 * tpx_colored_boxes: the box template of generate_colored_boxes (dva/ray_marcher.py:232-279) for N batch copies of K primitives of S^3
 * (S >= 2): colors [K,3] (the caller's np.random.rand(K, 3) * 255.0 rounded to fp32); per voxel (z, y, x) the dominant-axis sign
 * normal n of meshgrid(linspace(-1,1,S)^3) with its y and z negated, normalised (0 / 0 = NaN at a centre voxel whose coordinates are
 * all 0, as in the reference), mult = max(sum(lightdir * n), 0.2) with lightdir = -3 / ||(-3,-3,-3)|| per axis and NaN kept, and
 * rgb = colors[k] * (1.4f * mult), alpha = alpha, each an fp32 operation in the reference's order.  layout TPX_LAYOUT_NCDHW writes
 * out [N,K,4,S,S,S] (the reference's); TPX_LAYOUT_CHLAST writes [N,K,S,S,S,4] (the march's template, 16-B aligned).
 * tpx_primvolume_payload: recon_param [B,P,4+6 S^3] (LatentCodec.pack's layout: scale, pos[3], sdf S^3, tex 3 S^3, mat 2 S^3) ->
 * out [B,P,S,S,S,4] channels-last (16-B aligned): alpha = exp(-(sdf * (1 / 0.005f))^2) * 255 (visualize.py:217-232, bit for bit
 * with torch's CUDA ops); mode TPX_PAYLOAD_RGB colours tex * 255, TPX_PAYLOAD_MAT colours (0, roughness, metallic) * 255.
 * ---------------------------------------------------------------------------------------------------------- */
enum { TPX_LAYOUT_NCDHW = 0, TPX_LAYOUT_CHLAST = 1 };
enum { TPX_PAYLOAD_RGB = 0, TPX_PAYLOAD_MAT = 1 };
int tpx_colored_boxes(const float* colors, int N, int K, int S, float alpha, int layout, float* out, void* stream);
int tpx_primvolume_payload(const float* recon_param, int B, int P, int S, int mode, float* out, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Marching cubes — the `mcubes.marching_cubes(grid, 0.0)` call of extract_texmesh (inference.py:106-124), which copies the SDF grid
 * to the host for a CPU library.  vol device fp32 [X,Y,Z] C order, X, Y, Z >= 2, X*Y*Z < 2^31.  Output: an indexed triangle mesh with
 * shared vertices, deterministic (no output position depends on scheduling):
 *   inside iff value < iso (strict); one vertex per lattice edge whose ends classify differently; the edge p -> p + e_a is owned by
 *   p; vertex ids ordered by the C-order linear index of p, then by a; position p + t e_a, t = (iso - f(p)) / (f(p+e_a) - f(p)) in
 *   fp32, emitted as origin[d] + spacing[d] * pos[d] (component d = array axis d; origin 0 / spacing 1 = index units);
 *   triangles ordered by the C-order linear index of the cell, then by the case table (csrc/mc_tables.cuh, generated by mc_table.py);
 *   faces int64 [F,3]; (v1-v0) x (v2-v0) points toward increasing value (outward for an SDF that is negative inside).
 * Lifecycle: ws = tpx_mc_workspace_bytes(X,Y,Z) bytes of 256-B aligned device memory (0 = volume too large or too small; about
 * 6 bytes per grid point); tpx_mc_count writes counts_dev[0] = V, counts_dev[1] = F (device int64); the caller reads them back,
 * allocates verts [V,3] fp32 and faces [F,3] int64 (NULL allowed for a zero count), and calls tpx_mc_emit on the same workspace
 * with the same vol, X, Y, Z and iso, on the same stream.  Neither call synchronises.  If V or F is 2^31 or more, emit writes
 * nothing; the caller must treat such counts as an error.
 * ---------------------------------------------------------------------------------------------------------- */
size_t tpx_mc_workspace_bytes(int64_t X, int64_t Y, int64_t Z);
int tpx_mc_count(const float* vol_dev, int64_t X, int64_t Y, int64_t Z, float iso, void* ws, size_t ws_bytes, int64_t* counts_dev, void* stream);
int tpx_mc_emit(const float* vol_dev, int64_t X, int64_t Y, int64_t Z, float iso, float ox, float oy, float oz, float sx, float sy, float sz, void* ws,
                size_t ws_bytes, float* verts_dev, int64_t* faces_dev, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Mesh clean-up and decimation — the host stage extract_texmesh runs between marching cubes and the unwrap (inference.py:126-129:
 * clean_mesh(v, t, min_f=8, min_d=5, ...) then decimate_mesh(v, t, 100000), both pymeshlab, utils/meshutils.py:63-193).
 * Input: verts device fp32 [V,3], faces device int64 [F,3] (as tpx_mc_emit writes them), V and F below 2^31.  An index outside [0, V)
 * or a face that repeats an index is an error; zero-area faces with distinct indices are allowed.  Output: the vertices some kept face
 * uses, in ascending original id, and the kept faces in their original order, remapped, each with its own cyclic vertex order.
 * Deterministic: repeated calls, on any stream, give identical bytes.  Workspaces: 256-B aligned device memory of *_workspace_bytes(V, F)
 * bytes (0 = too large); the emit call takes the same workspace, V and F, on the same stream.  The full contract, with the arithmetic
 * spelled out, is in DESIGN.md §1 f-7.
 * ---------------------------------------------------------------------------------------------------------- */
/* clean_mesh's remove_connected_component_by_face_number(min_f) and ..._by_diameter(PercentageValue(min_d)) (utils/meshutils.py:63-193,
 * called at inference.py:126-127): faces are adjacent iff they share an undirected edge; a component is removed iff it has fewer than
 * min_faces faces or its box diagonal is below min_diameter (a fraction: min_d = 5 is 0.05) times the box diagonal of all referenced
 * vertices.  _count writes counts_dev[0] = V_out, [1] = F_out (device int64; both -1 for malformed faces, which _emit must then not be
 * called for); neither call synchronises.  About 150 bytes of workspace per face. */
size_t tpx_mesh_components_workspace_bytes(int64_t V, int64_t F);
int tpx_mesh_components_count(const float* verts_dev, int64_t V, const int64_t* faces_dev, int64_t F, int64_t min_faces, double min_diameter, void* ws,
                              size_t ws_bytes, int64_t* counts_dev, void* stream);
int tpx_mesh_components_emit(const float* verts_dev, int64_t V, int64_t F, const void* ws, size_t ws_bytes, float* verts_out_dev, int64_t* faces_out_dev,
                             void* stream);
/* decimate_mesh(v, t, target) (utils/meshutils.py:63-193, called at inference.py:129 with 100000): quadric-error edge collapse in rounds of
 * independent collapses (DESIGN.md §1 f-7); boundary and non-manifold vertices stay fixed.  Stops when F <= target (a reachable target
 * ends at F in {target - 1, target}) or when a round accepts nothing (the mesh is then left above target).  tpx_decimate SYNCHRONISES
 * the stream once per round (it reads the accepted count back) and on return; it writes counts_dev[0] = V_out, [1] = F_out,
 * [2] = rounds, and, when trace_host is not NULL, the face count after each of the first trace_cap rounds into that host array.
 * Malformed faces return TPX_ERR_ARG.  About 290 bytes of workspace per face.  tpx_decimate_emit writes the result (it reads the live counts back, so it synchronises too). */
size_t tpx_decimate_workspace_bytes(int64_t V, int64_t F);
int tpx_decimate(const float* verts_dev, int64_t V, const int64_t* faces_dev, int64_t F, int64_t target, void* ws, size_t ws_bytes, int64_t* counts_dev,
                 int64_t* trace_host, int64_t trace_cap, void* stream);
int tpx_decimate_emit(int64_t V, int64_t F, const void* ws, size_t ws_bytes, float* verts_out_dev, int64_t* faces_out_dev, void* stream);
/* clean_mesh(v, t, v_pct, ..., repair=True, remesh=False) (utils/meshutils.py:118-193, called at inference.py:126), the filters before and
 * after the component filter, as this package reads VCG (DESIGN.md §1 "clean-up contract"; pymeshlab itself is not run anywhere here).
 * Weld: meshing_remove_unreferenced_vertices, meshing_merge_close_vertices(PercentageValue(100 merge_distance)),
 * meshing_remove_duplicate_faces, meshing_remove_null_faces.  Faces may repeat an index (such faces are dropped); an index outside [0, V)
 * makes _count write -1, -1.  merge_distance = 0 merges nothing.  Greedy in ascending id: a referenced vertex is a seed iff no earlier
 * seed lies within r = merge_distance x the box diagonal of the referenced vertices (fp64 dx² + dy² + dz² < r²), otherwise it takes
 * the smallest such seed's id; faces onto the seeds, then a face is kept iff its indices are distinct, no lower face id has the same
 * index set and (v1 - v0) x (v2 - v0) is not exactly zero.  _count writes counts_dev[0] = V_out, [1] = F_out, [2] = merge rounds
 * and SYNCHRONISES (it reads the undecided count back every 8 rounds, and once at the end); _emit does not synchronise.
 * About 100 bytes of workspace per face plus 180 per vertex. */
size_t tpx_mesh_weld_workspace_bytes(int64_t V, int64_t F);
int tpx_mesh_weld_count(const float* verts_dev, int64_t V, const int64_t* faces_dev, int64_t F, double merge_distance, void* ws, size_t ws_bytes,
                        int64_t* counts_dev, void* stream);
int tpx_mesh_weld_emit(const float* verts_dev, int64_t V, int64_t F, const void* ws, size_t ws_bytes, float* verts_out_dev, int64_t* faces_out_dev,
                       void* stream);
/* clean_mesh's repair=True (utils/meshutils.py:118-193, inference.py:126): meshing_repair_non_manifold_edges(method=0) then
 * meshing_repair_non_manifold_vertices(vertdispratio=0).  Input as the component filter (no repeated index; F below 2^30).  The faces
 * on an edge with more than two faces are visited in ascending (doubled area, face id); one is deleted iff one of its edges still has
 * more than two faces.  Then every vertex whose faces form more than one fan (edge-connected around it) keeps the fan with the smallest
 * face id; each other fan gets a copy at the same position, appended after the surviving vertices in (vertex id, smallest face id of
 * the fan) order.  _count writes counts_dev[0] = V_out, [1] = F_out (both -1 for malformed faces); neither call synchronises.
 * About 270 bytes of workspace per face. */
size_t tpx_mesh_repair_workspace_bytes(int64_t V, int64_t F);
int tpx_mesh_repair_count(const float* verts_dev, int64_t V, const int64_t* faces_dev, int64_t F, void* ws, size_t ws_bytes, int64_t* counts_dev,
                          void* stream);
int tpx_mesh_repair_emit(const float* verts_dev, int64_t V, int64_t F, const void* ws, size_t ws_bytes, float* verts_out_dev, int64_t* faces_out_dev,
                         void* stream);
/* Isotropic remeshing: meshing_isotropic_explicit_remeshing(iterations, targetlen) as decimate_mesh(..., remesh=True) runs it after the
 * decimation (utils/meshutils.py:101-105, inference.py:128-129; clean_mesh's remesh=True, utils/meshutils.py:179-183, is the same filter),
 * as this package reads VCG's IsotropicRemeshing (DESIGN.md §1 "Isotropic remeshing contract").  The host drives the iterations:
 * _begin once, then per iteration _split_count / _split_emit (the mesh grows) and _relax (in place), then a compaction.
 * Creases are a sorted list of int64 edge keys (min << 32 | max), at most 3F of them.  Every call takes a workspace of
 * tpx_remesh_workspace_bytes(V, F) for the mesh it reads (about 250 bytes per face); the grid over the input mesh
 * (tpx_remesh_grid_bytes(F0), about 40 MB plus 150 bytes per face) lives from _begin to the last _relax, with the input vertices.
 * _begin checks the input faces, writes the creases (cos_feature = cos(feature angle)) and builds the grid; counts_dev[0] = nC, -1 for
 * malformed faces.  _split_count: counts_dev[0..2] = V', F', nC' (-1 for malformed faces); _split_emit (nC_out = nC') writes the split
 * mesh and its creases from the same workspace.  Neither of the three synchronises.  _relax runs the collapse rounds, the flip rounds,
 * the smoothing and the projection in place on verts_dev [V,3] and faces_dev (the live faces end up in its first F' rows) and writes
 * counts_dev[0..2] = F', collapse rounds, flip rounds; it SYNCHRONISES once per round and at its end (malformed faces: TPX_ERR_ARG). */
size_t tpx_remesh_workspace_bytes(int64_t V, int64_t F);
size_t tpx_remesh_grid_bytes(int64_t F);
int tpx_remesh_begin(const float* verts_dev, int64_t V, const int64_t* faces_dev, int64_t F, double cos_feature, void* grid, size_t grid_bytes, void* ws,
                     size_t ws_bytes, int64_t* creases_out_dev, int64_t* counts_dev, void* stream);
/* The projection on its own: for each of the n points pts_dev [n,3], the closest point of the input mesh of _begin (verts0_dev, F0 faces,
 * its grid) into out_dev [n,3] and that face's id into face_out_dev [n] (smallest squared distance, then smallest face id; -1 and the
 * point itself when the input has no face of non-zero area).  Does not synchronise. */
int tpx_remesh_closest(const float* pts_dev, int64_t n, const float* verts0_dev, int64_t V0, int64_t F0, const void* grid, size_t grid_bytes,
                       float* out_dev, int64_t* face_out_dev, void* stream);
int tpx_remesh_split_count(const float* verts_dev, int64_t V, const int64_t* faces_dev, int64_t F, const int64_t* creases_dev, int64_t nC, double target_len,
                           void* ws, size_t ws_bytes, int64_t* counts_dev, void* stream);
int tpx_remesh_split_emit(const float* verts_dev, int64_t V, int64_t F, const int64_t* creases_dev, int64_t nC, int64_t nC_out, const void* ws, size_t ws_bytes,
                          float* verts_out_dev, int64_t* faces_out_dev, int64_t* creases_out_dev, void* stream);
int tpx_remesh_relax(float* verts_dev, int64_t V, int64_t* faces_dev, int64_t F, const int64_t* creases_dev, int64_t nC, const float* verts0_dev, int64_t V0,
                     int64_t F0, const void* grid, size_t grid_bytes, double target_len, double cos_feature, void* ws, size_t ws_bytes, int64_t* counts_dev,
                     void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Box-projection UV unwrap and the primitive noise filter — the fast-unwrap branch of extract_texmesh (inference.py:140-150:
 * compute_vertex_normal + box_projection_uv_unwrap, utils/uv_unwrap.py:65-685) and its first block (inference.py:90-103).
 * verts device fp32 [V,3], faces device int32 [F,3], 1 <= V < 2^31 - 1, 1 <= F < 2^31 / 3; an index outside [0, V) is never read
 * (the face is treated as (0, 0, 0)) and makes tpx_uv_unwrap report U = -1.  Deterministic: repeated calls, on any stream, give
 * identical bytes.  The full contract, quirks included, is in DESIGN.md §1 f-8.  Workspace: tpx_uv_unwrap_workspace_bytes(V, F) bytes
 * of 256-B aligned device memory (0 = too large; about 300 bytes per face), shared by the three unwrap calls.
 * ---------------------------------------------------------------------------------------------------------- */
size_t tpx_uv_unwrap_workspace_bytes(int64_t V, int64_t F);
/* compute_vertex_normal (uv_unwrap.py:65-85): face normals (v1 - v0) x (v2 - v0) summed per vertex in the reference's scatter_add_
 * order (corner 0 of every face by ascending id, then corner 1, then corner 2), (0,0,1) where |n|^2 <= 1e-20, normalised; normals_dev
 * fp32 [V,3].  Does not synchronise. */
int tpx_vertex_normals(const float* verts_dev, int64_t V, const int32_t* faces_dev, int64_t F, void* ws, size_t ws_bytes, float* normals_dev, void* stream);
/* box_projection_uv_unwrap(v, n, f, island_padding) (uv_unwrap.py:644-685) up to the unique rows: writes counts_dev[0] = U (device
 * int64; -1 for malformed faces).  taps_host (NULL allowed) is a host array of 6 device pointers, each NULL or receiving a stage output:
 * [0] slice int32 [F], [1] projected uv fp32 [F,3,2], [2] slice angle fp32 [6], [3] rotated uv fp32 [F,3,2], [4] atlas index int32 [F],
 * [5] placed uv fp32 [F,3,2].  island_padding in [0, 0.5).  Does not synchronise: the caller reads U back once, allocates, and calls
 * tpx_uv_unwrap_emit with the same workspace, V and F on the same stream, which writes uv_dev fp32 [U,2] (rows sorted by (u, v)) and
 * vtex_idx_dev int64 [F,3] (torch.unique(placed.view(-1,2), dim=0, return_inverse=True), uv_unwrap.py:573-580). */
int tpx_uv_unwrap(const float* verts_dev, const float* normals_dev, int64_t V, const int32_t* faces_dev, int64_t F, double island_padding, void* ws,
                  size_t ws_bytes, int64_t* counts_dev, void** taps_host, void* stream);
int tpx_uv_unwrap_emit(int64_t V, int64_t F, const void* ws, size_t ws_bytes, float* uv_dev, int64_t* vtex_idx_dev, void* stream);
/* The noise filter of extract_texmesh (inference.py:90-103) on srt_dev fp32 [K,4] = (scale, x, y, z): d_ij = sqrt(sum_d (p_i - p_j)^2)
 * in fp32 plus 1 on the diagonal, nn_i = first argmin_j d_ij, keep_dev[i] = d_i,nn < s_i + s_nn (uint8 [K]); nn_dev (NULL allowed)
 * int32 [K] receives nn.  Does not synchronise. */
int tpx_prim_noise_filter(const float* srt_dev, int K, uint8_t* keep_dev, int32_t* nn_dev, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Texture bake —the back half of extract_texmesh (inference.py:163-211), device-resident.  All tensors contiguous, row-major;
 * atlas H, W in 1..8192; index tensors int32.
 *
 * tpx_uv_rasterize stands behind dr.rasterize as called at inference.py:163-172 (positions (2 uv - 1, 0, 1), i.e. a UV-space
 * rasterisation; nvdiffrast is a third-party extension that cannot be run here, so the contract is fixed below rather than
 * measured).  vt device fp32 [Nt,2] in [0,1], ft device int32 [F,3] (F < 2^24: rast carries the id as a float), outputs
 * rast device fp32 [H,W,4] = (u, v, 0, triangle_id + 1), zeros where nothing covers, and winner device int32 [H,W] = triangle_id or -1.
 *   texel (row i, col j) is sampled at its centre ((j + 1/2) / W, (i + 1/2) / H) in uv: row 0 is v = 0, nvdiffrast's bottom-up rows;
 *   a triangle covers a texel iff its three edge functions, oriented by the sign of its area, are >= 0 there (edges inclusive, both
 *   windings, zero-area triangles and triangles with an index outside [0, Nt) skipped); an edge is evaluated identically for the
 *   two triangles sharing it, so a shared edge leaves no hole; where several triangles cover a texel the lowest index wins;
 *   (u, v) are the barycentric weights of vertices 0 and 1.  Deterministic: repeated calls give identical bits.
 * tpx_rast_interpolate stands behind dr.interpolate (inference.py:173-174): out device fp32 [H,W,C] =
 * u attr[tri[t,0]] + v attr[tri[t,1]] + (1 - u - v) attr[tri[t,2]] with t = rast[...,3] - 1; zeros where rast[...,3] == 0 or an index
 * is outside [0, Nv).  attr device fp32 [Nv,C], tri device int32 [F,3] (may index a different vertex array than ft did).
 * ---------------------------------------------------------------------------------------------------------- */
int tpx_uv_rasterize(const float* vt_dev, int64_t Nt, const int32_t* ft_dev, int64_t F, int H, int W, float* rast_dev, int32_t* winner_dev, void* stream);
int tpx_rast_interpolate(const float* attr_dev, int64_t Nv, int C, const int32_t* tri_dev, int64_t F, const float* rast_dev, int H, int W, float* out_dev,
                         void* stream);
/* The masked query of inference.py:173-198 in one launch: per texel of rast, the 3-D position interpolated from v device fp32 [Nv,3] /
 * f device int32 [F,3] exactly as tpx_rast_interpolate computes it, the 6-channel grid-binned PrimSDF query (srt, feat, grid_ws, K, S,
 * dim_feat as for tpx_primsdf_sdf_grid; grid_ws NULL = exhaustive loop), feats_dev fp32 [H,W,6] = 255 * (R, G, B, 0, roughness, metallic)
 * and mask_dev uint8 [H,W] = 1 where a triangle covers the texel; uncovered texels get zeros.  feats / 255 is bit-identical to the
 * tex / mat columns of tpx_primsdf_query_grid at those positions. */
int tpx_primsdf_bake(const float* rast_dev, int H, int W, const float* v_dev, int64_t Nv, const int32_t* f_dev, int64_t F, const float* srt_dev,
                     const float* feat_dev, const void* grid_ws, size_t grid_bytes, int K, int S, int dim_feat, float* feats_dev, uint8_t* mask_dev,
                     void* stream);
/* Seam padding (inference.py:200-211: binary_dilation x pad, binary_erosion x 3, kd-tree nearest neighbour, all on the host there):
 * in place on feats_dev fp32 [H,W,C], every texel outside mask_dev (uint8 [H,W], non-zero = inside) whose 4-connected distance to the mask
 * is <= pad (0..8192) takes the value of the Euclidean-nearest mask texel, the smallest (row, col) among equidistant ones; all other
 * texels are untouched.  Exact (integer distances), deterministic.  src_dev (NULL allowed) int32 [H,W] receives the flat index of the
 * source texel, -1 where nothing was written.  ws: tpx_texture_inpaint_bytes(H, W) bytes of device scratch. */
size_t tpx_texture_inpaint_bytes(int H, int W);
int tpx_texture_inpaint(float* feats_dev, const uint8_t* mask_dev, int H, int W, int C, int pad, void* ws, size_t ws_bytes, int32_t* src_dev, void* stream);

/* nn.GELU() (erf form) in place on an fp16 tensor of n elements (n % 8 == 0, 16-B aligned), within one fp16 ulp of the exact GELU
 * of every finite input — the activation of the DINOv2 MLP
 * (models/conditioner/dinov2/layers/mlp.py:33-39); the rest of that encoder (SURVEY.md §8f-2) is built from the entry points above. */
int tpx_gelu_erf(void* x_f16, int64_t n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TPX_B200_H */
