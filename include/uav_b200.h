/* uav_b200.h — C ABI of libuav_b200.so: the sm_90a kernels behind the Upscale-A-Video
 * diffusion sampling hot path (SURVEY.md §8a/§8b).
 *
 * Conventions
 *  - Plain C: raw device pointers + explicit shapes. The library never allocates, frees or
 *    retains caller memory; every call is stream-ordered on `stream` and never synchronises.
 *  - Activations are channels-last: a "b c t h w" tensor of the reference is stored as
 *    [b][t][h][w][c] (c contiguous). `ld_*` arguments are the element distance between two
 *    consecutive pixels (>= channel count), so a tensor may be a channel slice of a wider
 *    buffer (this is how the skip-connection torch.cat of unet_blocks.py:573,645 disappears).
 *  - Weights are K-major fp16: conv weight (Cout,Cin,kh,kw) of the reference is passed as
 *    [Cout][kh][kw][Cin]; Conv3d (Cout,Cin,kt,kh,kw) as [Cout][kt][kh][kw][Cin]; Linear as
 *    [Cout][Cin] (unchanged). Bias is fp32.
 *  - Every function returns uav_status_t; on failure uav_last_error_string() describes it.
 *    No exceptions, no exit(), no CPU fallback.
 *
 * Each entry point cites the reference code (relative to /root/reference/models_video/)
 * whose device work it replaces.
 */
#ifndef UAV_B200_H_
#define UAV_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  UAV_OK = 0,
  UAV_ERR_INVALID = 1,     /* bad argument (shape / alignment / null) */
  UAV_ERR_CUDA = 2,        /* a CUDA runtime / driver call failed */
  UAV_ERR_UNSUPPORTED = 3  /* valid but not implemented for this configuration */
} uav_status_t;

typedef enum { UAV_F16 = 0, UAV_F32 = 1 } uav_dtype_t;
typedef enum {
  UAV_ACT_NONE = 0,
  UAV_ACT_SILU = 1,
  UAV_ACT_GEGLU = 2,
  UAV_ACT_RELU = 3,    /* RAFT encoders / motion encoder / heads */
  UAV_ACT_SIGMOID = 4, /* RAFT SepConvGRU z, r gates */
  UAV_ACT_TANH = 5,    /* RAFT SepConvGRU candidate state */
  UAV_ACT_GELU = 6,    /* CLIP text encoder MLP, hidden_act "gelu" (exact erf form) */
  UAV_ACT_QUICK_GELU = 7 /* CLIP text encoder MLP, hidden_act "quick_gelu": x * sigmoid(1.702 x) */
} uav_act_t;

typedef void* uav_stream_t; /* cudaStream_t */

const char* uav_version(void);
const char* uav_last_error_string(void);
/* number of kernels this library has launched in the calling process (bench: gpu_launches) */
uint64_t uav_launch_count(void);

/* Fused epilogue of every implicit-GEMM entry point:
 *   v = acc + bias[n] + rowvec[row / rows_per_vec][n]
 *   v = act(v)            (GEGLU: out[n] = v[n] * gelu(v[n + N/2]), output has N/2 columns)
 *   v = v * out_scale + residual[row][n]
 *   out[row][n] = (out_dtype) v          (fp16 conversions saturate to +-65504 instead of producing inf)
 *   gn_partial[n / 8][row / 16] = {sum, sum of squares} of the 8 x 16 block of v   (optional, see below)
 * Replaces the separate ATen kernels for "+ temb[:, :, None, None, None]" (resnet.py:272-276),
 * "(input_tensor + hidden_states) / output_scale_factor" (resnet.py:292, scale == 1 in every
 * shipped config), "attn(...) + hidden_states" (attention.py:531,537,549,559,563),
 * "hidden_states + residual" (attention.py:405), "input_tensor + hidden_states * w"
 * (temporal_module.py:192, w == 1) and GEGLU (diffusers_attention.py:802-823). */
typedef struct {
  const float* bias;     /* [N] or NULL */
  const void* rowvec;    /* fp16 [num_vec][ld_rowvec] or NULL */
  int64_t rows_per_vec;  /* output rows sharing one rowvec row (t*h*w of one batch item) */
  int64_t ld_rowvec;
  const void* residual;  /* fp16 [M][ld_res] or NULL */
  int64_t ld_res;
  int act;               /* uav_act_t */
  int out_dtype;         /* uav_dtype_t */
  int64_t ld_out;        /* element distance between output rows */
  /* -- optional extensions; an all-zero tail means "off" ------------------------------------------------ */
  float out_scale;       /* 0 = 1.  Scale applied before the residual add: lets the VAE decoder keep its residual
                            stream at 2^-k of the reference's values (fp16 range; every consumer is linear or a
                            GroupNorm, which is scale invariant once eps is scaled by 2^-2k) */
  /* GroupNorm statistics of the OUTPUT, produced on the way out so that the consumer's nn.GroupNorm
   * (resnet.py:267,278) needs no separate read pass: fp32 [n_out / 8][gn_blocks][2] = {sum, sum of squares} over
   * 8 channels x 16 consecutive rows of an M-tile (block = m_tile * 8 + row / 16 inside the tile; rows outside the
   * tensor contribute 0).  gn_blocks must equal uav_gn_partial_blocks() of the launch; requires the fp16 TMA-store
   * epilogue (n_out >= 33, aligned) and no GEGLU.  Deterministic (no atomics). */
  void* gn_partial;
  int64_t gn_blocks;
} uav_epilogue_t;

/* number of 16-row statistics blocks the implicit-GEMM launch over `images` images of `w` x `h` output pixels
 * produces (8 per M-tile; an M-tile is a tw x th = 128 pixel rectangle of one image, or 128 rows when h == 1) */
int64_t uav_gn_partial_blocks(int64_t w, int64_t h, int64_t images);

/* out[M][N] = epilogue(a[M][K] @ w[N][K]^T).  a: fp16, row stride lda (K % 8 == 0).
 * Replaces nn.Linear call sites: attention.py:97-106,156,177-178,202,327,355,382,400;
 * diffusers FeedForward (attention.py:493); time_emb_proj (resnet.py:243,273);
 * TimestepEmbedding (unet_video.py:176,478); AttentionBlock q/k/v/proj
 * (diffusers_attention.py:296-301). */
uav_status_t uav_linear(const void* a, int64_t M, int64_t K, int64_t lda, const void* w,
                        int64_t N, void* out, const uav_epilogue_t* epi, uav_stream_t stream);

/* 2-D convolution over NB = b*t images, channels-last, ksize 1 or 3, stride 1 or 2.
 * pad_mode 0: symmetric zero padding ksize/2 (InflatedConv3d resnet.py:94-101,
 *             Downsample3D padding=1 resnet.py:172);
 * pad_mode 1: stride 2, F.pad (0,1,0,1) then no padding (Downsample3D padding=0,
 *             resnet.py:188-192, VAE encoder).
 * x: fp16 [NB][H][W][ld_in] (first Cin channels used, Cin % 8 == 0); w: fp16
 * [Cout][ksize][ksize][Cin]; out: [NB][Ho][Wo][ld_out].  Stride 2 needs even H and W. */
uav_status_t uav_conv2d(const void* x, int64_t NB, int64_t H, int64_t W, int64_t Cin,
                        int64_t ld_in, const void* w, int64_t Cout, int ksize, int stride,
                        int pad_mode, void* out, const uav_epilogue_t* epi,
                        uav_stream_t stream);

/* stride-1 "same"-size convolution with an arbitrary kh x kw tap window (kh * kw <= 49) and asymmetric zero padding
 * (pad_top rows above / pad_left columns left; the rest below / right): output [NB][H][W][ld_out].
 * Used by the RAFT path: 7x7 convf1 (update.py:84), the 1x5 / 5x1 SepConvGRU convs (update.py:36-41) and, on
 * space-to-depth inputs, the stride-2 convs of the encoders (extractor.py:10,44,136: a k x k stride-2 conv is a
 * ceil(k/2) x ceil(k/2) stride-1 conv over the 2x2-phase-stacked input).  w: fp16 [Cout][kh][kw][Cin]. */
uav_status_t uav_conv2d_taps(const void* x, int64_t NB, int64_t H, int64_t W, int64_t Cin, int64_t ld_in,
                             const void* w, int64_t Cout, int kh, int kw, int pad_top, int pad_left, void* out,
                             const uav_epilogue_t* epi, uav_stream_t stream);

/* Temporal (k,1,1) convolution with zero padding (k-1)/2 in t (nn.Conv3d in
 * ResnetBlock3DCNN, resnet.py:332,348,361).  x: fp16 [B][T][HW][ld_in];
 * w: fp16 [Cout][k][Cin]; out: [B][T][HW][ld_out]. */
uav_status_t uav_conv_temporal(const void* x, int64_t B, int64_t T, int64_t HW, int64_t Cin,
                               int64_t ld_in, const void* w, int64_t Cout, int k, void* out,
                               const uav_epilogue_t* epi, uav_stream_t stream);

/* 3x3x3 convolution, zero padding 1 in t,h,w (ResnetBlock3D_plus.conv_3d, resnet.py:461).
 * x: fp16 [B][T][H][W][ld_in]; w: fp16 [Cout][3][3][3][Cin]. */
uav_status_t uav_conv3d(const void* x, int64_t B, int64_t T, int64_t H, int64_t W, int64_t Cin,
                        int64_t ld_in, const void* w, int64_t Cout, void* out,
                        const uav_epilogue_t* epi, uav_stream_t stream);

/* Upsample3D (resnet.py:143-156): F.interpolate(scale 2, nearest) followed by the 3x3 conv, computed WITHOUT
 * materialising the upsampled tensor: output pixel (2y+a, 2x+b) only sees 2x2 source pixels, so the 3x3 filter
 * collapses into four 2x2 phase filters (rows {W0, W1+W2} for a=0, {W0+W1, W2} for a=1; same for columns) —
 * 4/9 of the MACs and no 4x-sized intermediate.  w4: fp16 [4 phases (a*2+b)][Cout][2][2][Cin] (summed in fp32 by the
 * caller, then rounded once).  x: [NB][H][W][ld_in]; out: [NB][2H][2W][ld_out]; bias-only fp16 epilogue. */
uav_status_t uav_upsample2x_conv3x3(const void* x, int64_t NB, int64_t H, int64_t W, int64_t Cin,
                                    int64_t ld_in, const void* w4, int64_t Cout, void* out,
                                    const uav_epilogue_t* epi, uav_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * normalisation
 * ------------------------------------------------------------------------------------------- */
/* bytes of caller-owned scratch (`workspace`) needed by uav_groupnorm_silu, uav_groupnorm_silu_from_partials and
 * uav_groupnorm_affine: fp64 {sum, sumsq} per (n, group) and split, plus the read pass's per-block partials */
size_t uav_groupnorm_workspace_bytes(int64_t n_outer, int groups);

/* GroupNorm (+ optional SiLU) over channels-last data: x [n_outer][pixels][ld_in] fp16, statistics
 * per (n_outer, group) over pixels * C/groups elements, fp32 affine, fp16 output.
 * 5-D nn.GroupNorm of the reference ("b c t h w", resnet.py:231,247,267,278; unet_video.py:331,567):
 * n_outer = b, pixels = t*h*w (statistics span the frames of the chunk).  Per-frame 4-D GroupNorm
 * (attention.py:325,374; AttentionBlock diffusers_attention.py:269): n_outer = b*t, pixels = h*w.
 * SiLU = the `nonlinearity` that always follows (resnet.py:268,284; unet_video.py:568). */
uav_status_t uav_groupnorm_silu(const void* x, int64_t n_outer, int64_t pixels, int64_t C,
                                int64_t ld_in, int groups, const float* gamma, const float* beta,
                                float eps, int silu, void* y, int64_t ld_out, void* workspace,
                                size_t workspace_bytes, uav_stream_t stream);

/* One producer of the tensor a GroupNorm consumes: the statistics blocks an implicit-GEMM launch wrote through
 * uav_epilogue_t.gn_partial.  `slabs`: how many statistics slabs (batch items, or frames for the per-frame norm) the
 * launch's blocks divide into evenly, in order — equal to the consumer's n_outer, or 1 when the same rows serve
 * every n (a skip tensor computed once for both classifier-free-guidance halves). */
typedef struct {
  const void* partial; /* fp32 [C / 8][blocks][2] */
  int64_t blocks;
  int64_t C;           /* channels of this source, % 8 == 0 */
  int64_t slabs;
  /* the source tensor itself, for a concatenation that is never materialised (all sources then carry one; x of the call
   * is ignored): fp16 [slab][pixels][ld]; slab_stride = elements between slabs, 0 when every n reads the same rows */
  const void* x;
  int64_t ld;
  int64_t slab_stride;
} uav_gn_source_t;

/* uav_groupnorm_silu without the statistics read pass: x is the channel concatenation (in order) of up to 4 tensors
 * whose producers emitted their statistics blocks (the torch.cat of unet_blocks.py:573,645 followed by resnet.py:267).
 * (C / groups) % 8 == 0.  Two launches (fp64 fixed-order reduction of the blocks, apply) instead of three, and
 * 2 instead of 3 element passes over x.  When the sources carry their own tensors (source.x), the concatenation is
 * never built: the apply pass runs once per source and writes the normalised, DENSE [.., C] tensor y that the following
 * convolution reads (x / ld_in of the call are then unused).  workspace: uav_groupnorm_workspace_bytes. */
uav_status_t uav_groupnorm_silu_from_partials(const void* x, int64_t n_outer, int64_t pixels, int64_t C,
                                              int64_t ld_in, int groups, const float* gamma, const float* beta,
                                              float eps, int silu, void* y, int64_t ld_out,
                                              const uav_gn_source_t* sources, int n_sources, void* workspace,
                                              size_t workspace_bytes, uav_stream_t stream);

/* Only the per-(slab, channel) affine of a GroupNorm, for a consumer that applies it itself (uav_conv_out_fused):
 * affine fp32 [n_outer][C][2] = {gamma * rstd, beta - mean * gamma * rstd}.  Statistics from the producers' blocks
 * (n_sources > 0; x may be NULL) or from a read pass over x (n_sources == 0). */
uav_status_t uav_groupnorm_affine(const void* x, int64_t n_outer, int64_t pixels, int64_t C, int64_t ld_in, int groups,
                                  const float* gamma, const float* beta, float eps, const uav_gn_source_t* sources,
                                  int n_sources, float* affine, void* workspace, size_t workspace_bytes,
                                  uav_stream_t stream);

/* The tail of UNetVideoModel.forward in one HBM-bound kernel (unet_video.py:567-569):
 *   out = conv_out(SiLU(GroupNorm(x)))    3x3, zero padding 1, C = 256 -> Cout <= 5 channels,
 * x: fp16 [B][T][H][W][ld] (raw, before conv_norm_out), affine: the GroupNorm's fp32 [B][C][2] table from
 * uav_groupnorm_affine, w: fp16 [Cout][3][3][C], out: the reference's planar "b c t h w" tensor [B][Cout][T][H][W] in
 * out_dtype.  Reads x once (no normalised copy of the 256-channel tensor is ever written), replaces GroupNorm apply +
 * InflatedConv3d (resnet.py:94-101) + the rearrange back to b c t h w. */
uav_status_t uav_conv_out_fused(const void* x, int64_t B, int64_t T, int64_t H, int64_t W, int64_t C, int64_t ld,
                                const float* affine, const void* w, const float* bias, int64_t Cout, void* out,
                                int out_dtype, uav_stream_t stream);

/* ... and the same kernel with the sampler arithmetic of the step in its epilogue (BASELINE north_star: "DDIM step +
 * classifier-free-guidance add fused into the UNet epilogue"): the two batch items of x are the unconditional / text halves
 * of ONE clip; per output element, with torch's per-op fp16 rounding (bit-identical to uav_cfg_combine followed by
 * uav_ddim_step_v0 on the fp16 output of uav_conv_out_fused):
 *   noise_pred = u + g * (c - u)                                   (pipeline_upscale_a_video.py:644-645)
 *   pred_original_sample = DDIMScheduler.step_v0(noise_pred, sample) (scheduling_ddim.py:383-433)
 * All three tensors are fp16 (1, Cout, T, H, W) in the reference layout.  x: fp16 [2][T][H][W][ld]. */
typedef struct {
  float guidance_scale;
  int pred_type;             /* 0 epsilon, 1 sample, 2 v_prediction */
  float sqrt_alpha, sqrt_beta;
  int clip;
  float clip_range;
  const void* sample;        /* x_t */
  void* noise_pred;
  void* pred_original_sample;
} uav_cfg_step_t;
uav_status_t uav_conv_out_cfg_step(const void* x, int64_t T, int64_t H, int64_t W, int64_t C, int64_t ld,
                                   const float* affine, const void* w, const float* bias, int64_t Cout,
                                   const uav_cfg_step_t* step, uav_stream_t stream);

/* nn.LayerNorm over the last dim of fp16 tokens (attention.py:457,474,491,494). C % 8 == 0. */
uav_status_t uav_layernorm(const void* x, int64_t rows, int64_t C, int64_t ld_in,
                           const float* gamma, const float* beta, float eps, void* y,
                           int64_t ld_out, uav_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * attention
 * ------------------------------------------------------------------------------------------- */
/* out = softmax(q k^T * scale) v per (batch, head), never materialising the scores
 * (CrossAttention._attention attention.py:209-238; AttentionBlock diffusers_attention.py:330-381).
 * q [batch][nq][ldq], k/v [batch / kv_batch_div][nk][ld], out [batch][nq][ldo]; head h occupies
 * columns [h*head_dim, (h+1)*head_dim).  kv_batch_div = frames when the text K/V are shared by all
 * frames of a batch item (the reference repeats them: attention.py:364).  head_dim 64, 128, or
 * 512 (single head).  q, k, v and out must be 16-byte aligned. */
uav_status_t uav_attention(const void* q, const void* k, const void* v, void* out, int64_t batch,
                           int heads, int head_dim, int64_t nq, int64_t nk, int64_t ldq,
                           int64_t ldk, int64_t ldv, int64_t ldo, int64_t kv_batch_div,
                           float scale, uav_stream_t stream);

/* TemporalAttention._attention (attention.py:699-733): per pixel, sequence = frames (any F >= 1);
 * q is scaled, q and k get the rotary embedding on dims [0,32) (cos/sin table rot[F][16][2]),
 * scores += rel_bias[heads][F][F], row-max subtract, softmax, PV.  Tokens are ordered
 * (b, f, hw) — the channels-last video layout — so no rearrange copies are needed.  head_dim 64
 * or 128.  q, k, v, out and rot_cos_sin must be 16-byte aligned.  F <= 8 with an even head count
 * runs on the windowed-pipeline kernel; everything else on an online-softmax kernel that streams
 * 16-frame key tiles. */
uav_status_t uav_temporal_attention(const void* q, const void* k, const void* v, void* out,
                                    int64_t B, int64_t F, int64_t HW, int heads, int head_dim,
                                    int64_t ldq, int64_t ldk, int64_t ldv, int64_t ldo,
                                    float scale, const float* rot_cos_sin, const float* rel_bias,
                                    uav_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * data movement
 * ------------------------------------------------------------------------------------------- */
/* dst[p][0:C] = src[p][0:C] for `pixels` rows (torch.cat of skip connections, unet_blocks.py:573,645) */
uav_status_t uav_copy_channels(const void* src, int64_t ld_src, void* dst, int64_t ld_dst,
                               int64_t C, int64_t pixels, uav_stream_t stream);
/* F.interpolate(mode="nearest") of NB channels-last images to (Ho, Wo) (Upsample3D resnet.py:143-146) */
uav_status_t uav_upsample_nearest(const void* src, int64_t ld_src, int64_t NB, int64_t Hi,
                                  int64_t Wi, int64_t C, void* dst, int64_t ld_dst, int64_t Ho,
                                  int64_t Wo, uav_stream_t stream);
/* API edge: reference layout (B, C, T*H*W) fp16/fp32 -> channels-last fp16 at channel offset c_off
 * (also performs torch.cat([sample, low_res], dim=1), unet_video.py:440), times `scale`. */
uav_status_t uav_planar_to_channels_last(const void* src, int src_dtype, int64_t B, int64_t C,
                                         int64_t thw, void* dst, int64_t ld_dst, int64_t c_off,
                                         float scale, uav_stream_t stream);
/* API edge: channels-last -> (B, C, T*H*W); clamp != 0 applies .clamp(-1, 1) (pipeline...:353) */
uav_status_t uav_channels_last_to_planar(const void* src, int src_dtype, int64_t ld_src, int64_t B,
                                         int64_t C, int64_t thw, void* dst, int dst_dtype,
                                         int clamp, uav_stream_t stream);
uav_status_t uav_silu(const void* x, void* y, int64_t n, uav_stream_t stream);
/* Fuse_sft_block tail (resnet.py:77-78): out = (dec + w * (dec * scale + shift)) * out_scale (0 = 1; the VAE decoder's
 * residual-stream scale, see uav_epilogue_t.out_scale); dense fp16, n % 8 == 0 */
uav_status_t uav_sft_fuse(const void* dec, const void* scale, const void* shift, float w, float out_scale, void* out,
                          int64_t n, uav_stream_t stream);
/* diffusers Timesteps(dim, flip_sin_to_cos, freq_shift) (unet_video.py:173,472): fp32 math, fp16 out */
uav_status_t uav_timestep_embedding(const float* t, int64_t B, int64_t dim, int flip_sin_to_cos,
                                    float freq_shift, void* out, uav_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * sampler: run on the reference's own "b c t h w" latents; dtype = UAV_F16 replays torch's
 * per-op fp16 rounding exactly (SURVEY.md Appendix B), UAV_F32 is plain fp32.
 * ------------------------------------------------------------------------------------------- */
/* out = uncond + g * (text - uncond); pred2 = [uncond | text], n = elements of one half
 * (pipeline_upscale_a_video.py:644-645) */
uav_status_t uav_cfg_combine(const void* pred2, void* out, int64_t n, float guidance_scale,
                             int dtype, uav_stream_t stream);
/* dst[:, :, t0+k] = covered(k) ? dst*0.5 + src[:, :, k]*0.5 : src[:, :, k]
 * (pipeline_upscale_a_video.py:630-634); tensors (outer, T, hw) / (outer, Tw, hw) */
uav_status_t uav_window_blend(void* dst, int64_t T, const void* src, int64_t Tw, int64_t t0,
                              uint32_t covered_mask, int64_t outer, int64_t hw, int dtype,
                              uav_stream_t stream);
/* DDIMScheduler.step_v0 (scheduling_ddim.py:383-433); pred_type 0 epsilon, 1 sample, 2 v_prediction */
uav_status_t uav_ddim_step_v0(const void* model_output, const void* sample, void* x0, int64_t n,
                              int pred_type, float sqrt_alpha, float sqrt_beta, int clip,
                              float clip_range, int dtype, uav_stream_t stream);
/* DDIMScheduler.step_vt (scheduling_ddim.py:436-520); dir_coef = (1 - a_prev - std^2)^0.5 */
uav_status_t uav_ddim_step_vt(const void* x0, const void* model_output, const void* sample,
                              void* prev, int64_t n, int pred_type, float sqrt_alpha,
                              float sqrt_beta, float sqrt_alpha_prev, float dir_coef, int clip,
                              float clip_range, float std_dev, const void* noise, int dtype,
                              uav_stream_t stream);
/* add_noise (scheduling_ddim.py:524-545 / diffusers DDPMScheduler.add_noise) */
uav_status_t uav_add_noise(const void* x, const void* noise, void* out, int64_t n,
                           float sqrt_alpha, float sqrt_one_minus_alpha, int dtype,
                           uav_stream_t stream);
/* one frame update of Propagation.forward, learnable=False (propagation_module.py:234-254):
 * fbConsistencyCheck mask + flow_warp(nearest|bilinear) + fuse + select, for C planes of H x W.
 * cs_* = channel (plane) strides in elements. */
uav_status_t uav_propagate_step(const void* feat_prop, const void* feat_cur, const void* flow_prop,
                                const void* flow_check, void* out, int64_t C, int64_t H, int64_t W,
                                int64_t cs_prop, int64_t cs_cur, int64_t cs_out,
                                int64_t cs_flow_prop, int64_t cs_flow_check, int nearest, int fuse,
                                float fuse_scale, float alpha1, float alpha2, int dtype, uav_stream_t stream);
/* the flow resize of Propagation.forward (propagation_module.py:206-209):
 * out = F.interpolate(in, (t_out, h_out, w_out), mode='area') * scale, bit-identical to torch's CUDA
 * kernel (fp32 window sum, one divide, rounded to dtype, then * scale in fp32 and rounded again).
 * in: [planes][t_in][h_in][w_in], out: [planes][t_out][h_out][w_out], both contiguous. */
uav_status_t uav_flow_resize_area(const void* in, void* out, int64_t planes, int64_t t_in, int64_t h_in,
                                  int64_t w_in, int64_t t_out, int64_t h_out, int64_t w_out, float scale,
                                  int dtype, uav_stream_t stream);

/* ---- after the decode: colour fix + output packing (SURVEY.md §8f rank 4) ---------------------------------
 * All tensors are the reference's planar fp32 "t c h w" frames (planes = t * c). */

/* F.interpolate(vframes, scale_factor=scale, mode='bicubic') of the low-resolution frames before the colour fix
 * (inference_upscale_a_video.py:327): align_corners=False, A=-0.75, border-clamped taps. out: [planes][h*scale][w*scale] */
uav_status_t uav_bicubic_upsample(const float* in, int64_t planes, int64_t h, int64_t w, int scale, float* out,
                                  uav_stream_t stream);
/* calc_mean_std (color_correction.py:45-58): per plane mean and sqrt(unbiased var + eps) over hw elements.
 * Deterministic (no atomics). workspace: uav_plane_stats_workspace_bytes(planes) bytes, 16-byte aligned. */
size_t uav_plane_stats_workspace_bytes(int64_t planes);
uav_status_t uav_plane_stats(const float* x, int64_t planes, int64_t hw, float eps, void* workspace, float* mean,
                             float* stdv, uav_stream_t stream);
/* adaptive_instance_normalization (color_correction.py:60-73):
 * out = (content - c_mean[plane]) / c_std[plane] * s_std[plane] + s_mean[plane], one rounding per reference op */
uav_status_t uav_adain_apply(const float* content, int64_t planes, int64_t hw, const float* c_mean, const float* c_std,
                             const float* s_mean, const float* s_std, float* out, uav_stream_t stream);
/* one level of wavelet_decomposition (color_correction.py:75-103): low = wavelet_blur(image, radius) (depthwise
 * [1 2 1; 2 4 2; 1 2 1]/16, dilation = radius, replicate padding); if high != NULL: high = image - low
 * (high_first != 0) or high += image - low; if add != NULL the value written to `low` is add + low (the final
 * content_high_freq + style_low_freq of wavelet_reconstruction, :105-118). low may be NULL. Outputs must not alias image. */
uav_status_t uav_wavelet_level(const float* image, int64_t planes, int64_t H, int64_t W, int radius, float* low,
                               float* high, int high_first, const float* add, uav_stream_t stream);
/* (frames / 2 + 0.5).clamp(0, 1) * 255 -> "t h w c" -> uint8 by truncation (inference_upscale_a_video.py:354-356).
 * frames: [T][C][H][W] fp32, out: [T][H][W][C] uint8, C <= 4. Bit-exact. */
uav_status_t uav_pack_video_uint8(const float* frames, int64_t T, int64_t C, int64_t H, int64_t W, uint8_t* out,
                                  uav_stream_t stream);
/* the PNG rounding of torchvision save_image(normalize=True, value_range=(-1, 1)) (inference_upscale_a_video.py:350):
 * clamp(-1, 1), (x + 1) / 2, * 255, + 0.5, clamp(0, 255), truncate. Same layout as uav_pack_video_uint8. Bit-exact. */
uav_status_t uav_pack_frames_png(const float* frames, int64_t T, int64_t C, int64_t H, int64_t W, uint8_t* out,
                                 uav_stream_t stream);

/* ---- before sampling: frame ingest (inference_upscale_a_video.py:180-188) ------------------------------------
 * frames: [T][H][W][3] uint8 in BGR order (OpenCV's decode); out: [3][T][h_out][w_out] fp32 RGB in [-1, 1]:
 * (v / 255. - 0.5) * 2 with one IEEE fp32 rounding per op, then, when (h_out, w_out) != (H, W),
 * F.interpolate(x, (h_out, w_out), mode='area') bit-identical to torch's CUDA kernel for NCHW fp32 frames (nhwc = 0:
 * the reference's image folders, made contiguous by utils.read_frame_from_videos) or for channels-last ones (nhwc = 1:
 * its video files, which torchvision.io.read_video returns as a permuted view). The two kernels round the average
 * differently. 1 <= h_out <= H, 1 <= w_out <= W, not a 1x1 output of a larger frame. */
uav_status_t uav_unpack_video_uint8(const uint8_t* frames, int64_t T, int64_t H, int64_t W, int64_t h_out, int64_t w_out,
                                    int nhwc, float* out, uav_stream_t stream);

/* ---- RAFT bidirectional optical flow (SURVEY.md §8f rank 1; models_video/RAFT) -----------------------------
 * Non-GEMM kernels; activations channels-last fp16 [pixel][C], correlation volume / coordinates / flows fp32. */

/* nn.InstanceNorm2d defaults (no affine, biased variance) + optional ReLU (extractor.py:27-31,49-50,129-130,176-178).
 * x, y: [n][hw][C] fp16, C % 8 == 0.  Deterministic.  workspace: uav_instnorm_workspace_bytes(n, C) bytes. */
size_t uav_instnorm_workspace_bytes(int64_t n, int64_t C);
uav_status_t uav_instnorm_relu(const void* x, int64_t n, int64_t hw, int64_t C, float eps, int relu, void* y, void* workspace,
                               uav_stream_t stream);
/* y = relu(a + b) over n fp16 elements (ResidualBlock tail, extractor.py:57) */
uav_status_t uav_add_relu(const void* a, const void* b, void* y, int64_t n, uav_stream_t stream);
/* net = tanh(cnet[:, :C]) -> net[rows][ld_net]; inp = relu(cnet[:, C:2C]) -> inp_a (and inp_b if not NULL) (raft.py:117-120) */
uav_status_t uav_raft_split_tanh_relu(const void* cnet, int64_t rows, int64_t C, void* net, int64_t ld_net, void* inp_a,
                                      int64_t ld_a, void* inp_b, int64_t ld_b, uav_stream_t stream);
/* F.avg_pool2d(x, 2, stride=2) on [planes][h][w] fp32 (corr.py:24-27) */
uav_status_t uav_avgpool2x2_f32(const float* in, int64_t planes, int64_t h, int64_t w, float* out, uav_stream_t stream);
/* CorrBlock.__call__ (corr.py:30-50), radius 4, 4 levels: levels[i] = [pixels][hs[i]][ws[i]] fp32 (one plane per query
 * pixel), coords = [pixels][2] (x, y) at level 0; out fp16 [pixels][ld_out], channel = level * 81 + a * 9 + b where a
 * offsets x and b offsets y (the reference's meshgrid order); channels [324, ld_out) are zeroed. */
uav_status_t uav_raft_corr_lookup(const float* const* levels, const int32_t* hs, const int32_t* ws, const float* coords,
                                  int64_t pixels, void* out, int64_t ld_out, uav_stream_t stream);
/* SepConvGRU gate arithmetic (update.py:47-60), zr = [sigmoid(convz) | sigmoid(convr)] fp16 [rows][ld_zr]:
 *   uav_raft_gru_rh:     out[:, :C] = r * h
 *   uav_raft_gru_update: h = (1 - z) * h + z * q   (in place) */
uav_status_t uav_raft_gru_rh(const void* zr, int64_t ld_zr, const void* h, int64_t ld_h, void* out, int64_t ld_out, int64_t rows,
                             int64_t C, uav_stream_t stream);
uav_status_t uav_raft_gru_update(const void* zr, int64_t ld_zr, const void* q, int64_t ld_q, void* h, int64_t ld_h, int64_t rows,
                                 int64_t C, uav_stream_t stream);
/* coords1 += delta (delta may be NULL), flow = coords1 - coords0 (raft.py:128-134) written as fp16 into channels [0, 2)
 * of up to three [rows][ld] buffers (NULL = skip); rows = images * h8 * w8 */
uav_status_t uav_raft_flow_update(float* coords1, const float* delta, int64_t ld_delta, int64_t rows, int64_t h8, int64_t w8,
                                  void* flow16, int64_t ld16, void* dst_a, int64_t ld_a, void* dst_b, int64_t ld_b,
                                  uav_stream_t stream);
/* RAFT.upsample_flow (raft.py:73-84): mask fp16 [images*h8*w8][ld_mask] (576 channels = 9 x 8 x 8), out fp32 planar
 * [images][2][8*h8][8*w8] */
uav_status_t uav_raft_convex_upsample(const float* coords1, const void* mask, int64_t ld_mask, int64_t nimg, int64_t h8,
                                      int64_t w8, float* out, uav_stream_t stream);

/* ---- CLIP text encoder (SURVEY.md §8f rank 3) ---------------------------------------------------------------
 * causal self-attention over a short sequence (transformers CLIPAttention under CLIPTextTransformer's causal mask):
 * q, k, v, out fp16 [batch][n][ld] with `heads * head_dim` used columns (column slices of a fused qkv buffer allowed),
 * n <= 128, head_dim <= 128 and even; out[i] = softmax_j<=i(scale * q_i . k_j) v_j.  head_dim 128 also takes n > 128 (the
 * LLaVA decoder's prefill) on the causal wgmma kernel: then token strides are multiples of 8, pointers 16-byte
 * aligned and scale finite and > 0 */
uav_status_t uav_attention_causal(const void* q, const void* k, const void* v, void* out, int64_t batch, int heads, int head_dim,
                                  int64_t n, int64_t ldq, int64_t ldk, int64_t ldv, int64_t ldo, float scale,
                                  uav_stream_t stream);

/* ---- LLaVA-1.5 captioner (llava.py): Llama decoder and sampler --------------------------------------------------
 * uav_rmsnorm: transformers LlamaRMSNorm on fp16 [rows][ld] rows of C % 8 == 0 columns: fp32 mean of squares,
 *   x * rsqrt(var + eps) rounded to fp16, then times the fp16 weight in fp16 */
uav_status_t uav_rmsnorm(const void* x, int64_t rows, int64_t C, int64_t ldx, const void* weight, float eps, void* out,
                         int64_t ldo, uav_stream_t stream);
/* rotate-half rotary embedding of head_dim 128 on the q and k columns of n fused q|k|v fp16 rows ([n][ld_qkv]: q at
 * columns [0, C), k at [C, 2C), v at [2C, 3C), C = heads * 128) at positions [p0, p0 + n): q is rotated in place, the
 * rotated k and v go to rows [p0, p0 + n) of k_cache / v_cache ([cache_rows][ld_kv] fp16).  cos_sin: fp32
 * [positions][64][2] = cos, sin of position * inv_freq[i] */
uav_status_t uav_rope_kv_append(void* qkv, int64_t ld_qkv, int64_t n, int heads, int head_dim, int64_t p0,
                                const float* cos_sin, int64_t positions, void* k_cache, void* v_cache, int64_t ld_kv,
                                int64_t cache_rows, uav_stream_t stream);
/* uav_rope_kv_append on `batch` sequences at once (n rows each, positions [p0, p0 + n) in every sequence): sequence b's
 * rows start at qkv + b * qkv_batch_stride and its caches at k_cache / v_cache + b * kv_batch_stride (elements), each
 * [cache_rows][ld_kv].  Serves the prefill (n = prompt length) and every decode step (n = 1); each sequence's result
 * is bit-identical to a uav_rope_kv_append call on it alone.  batch > 1 needs qkv_batch_stride >= n * ld_qkv and
 * kv_batch_stride >= cache_rows * ld_kv. */
uav_status_t uav_rope_kv_append_batched(void* qkv, int64_t ld_qkv, int64_t qkv_batch_stride, int64_t batch, int64_t n,
                                        int heads, int head_dim, int64_t p0, const float* cos_sin, int64_t positions,
                                        void* k_cache, void* v_cache, int64_t ld_kv, int64_t kv_batch_stride,
                                        int64_t cache_rows, uav_stream_t stream);
/* out[r][c] = silu(gate_up[r][c]) * gate_up[r][inter + c] (transformers LlamaMLP on the fused gate|up output), fp16 */
uav_status_t uav_swiglu(const void* gate_up, int64_t ld_gu, int64_t rows, int64_t inter, void* out, int64_t ldo,
                        uav_stream_t stream);
/* one-row GEMV, the decode step's weight stream: out[n] = sum_k w[n][k] x[k] (+ residual[n]), w fp16 [N][K] dense,
 * x fp16 [K], fp32 accumulation; out_dtype UAV_F16 (residual fp16 or NULL) or UAV_F32 (no residual).  K % 8 == 0,
 * K <= 16384.  Split-K over the warps of a row with a fixed-order combine: deterministic. */
uav_status_t uav_gemv(const void* w, int64_t N, int64_t K, const void* x, const void* residual, void* out, int out_dtype,
                      uav_stream_t stream);
/* uav_gemv on 1 <= rows <= 8 input rows with w streamed once for all of them: out[r][n] = sum_k w[n][k] x[r][k]
 * (+ residual[r][n]); x fp16 [rows][K], residual fp16 [rows][N] and out [rows][N] dense.  rows * K <= 110592 when
 * rows > 1 (x is held in shared memory).  Each row's result is bit-identical to uav_gemv on that row. */
uav_status_t uav_gemv_rows(const void* w, int64_t N, int64_t K, const void* x, int64_t rows, const void* residual,
                           void* out, int out_dtype, uav_stream_t stream);
/* attention of one query row per head (q fp16 [heads * 128]) against the first L rows of a KV cache ([L][ld_kv] fp16),
 * out fp16 [heads * 128]; key chunks are combined in a fixed order (flash-decoding).  workspace: fp32 scratch of
 * uav_attention_decode_workspace_bytes(heads, L) bytes */
size_t uav_attention_decode_workspace_bytes(int heads, int64_t L);
uav_status_t uav_attention_decode(const void* q, const void* k_cache, const void* v_cache, int64_t ld_kv, int64_t L,
                                  int heads, int head_dim, float scale, void* out, void* workspace, size_t ws_bytes,
                                  uav_stream_t stream);
/* uav_attention_decode for `batch` sequences that share the cache length L: sequence b's query row is q + b * ldq,
 * its caches k_cache / v_cache + b * kv_batch_stride (elements) and its output out + b * ldo.  Each sequence's result
 * is bit-identical to uav_attention_decode on it alone.  batch > 1 needs ldq, ldo >= heads * 128, ldq % 4 == 0 and
 * kv_batch_stride >= L * ld_kv, % 4 == 0.  workspace: uav_attention_decode_batched_workspace_bytes(batch, heads, L) */
size_t uav_attention_decode_batched_workspace_bytes(int64_t batch, int heads, int64_t L);
uav_status_t uav_attention_decode_batched(const void* q, int64_t ldq, const void* k_cache, const void* v_cache,
                                          int64_t ld_kv, int64_t kv_batch_stride, int64_t batch, int64_t L, int heads,
                                          int head_dim, float scale, void* out, int64_t ldo, void* workspace,
                                          size_t ws_bytes, uav_stream_t stream);
/* next token from fp32 logits [V] (V <= 49152): temperature, then transformers TopPLogitsWarper's keep rule, then the
 * inverse CDF of the kept set in vocabulary order at u * (kept mass), u in [0, 1).  temperature == 0: argmax, first
 * index on ties.  The token id is written to *token (device int64). */
uav_status_t uav_sample_top_p(const float* logits, int64_t V, float temperature, float top_p, float u, int64_t* token,
                              uav_stream_t stream);
/* uav_sample_top_p on 1 <= rows <= 8 rows of fp32 logits ([rows][ld_logits]), one CTA per row: row r is sampled
 * with the host uniform u[r] (read before the call returns: no device copy) into tokens[r].  Each row's token is the
 * one uav_sample_top_p picks for that row. */
uav_status_t uav_sample_top_p_batched(const float* logits, int64_t ld_logits, int64_t rows, int64_t V,
                                      float temperature, float top_p, const float* u, int64_t* tokens,
                                      uav_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* UAV_B200_H_ */
