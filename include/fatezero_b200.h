/* fatezero_b200.h — C ABI of libfatezero_b200.so (sm_90a kernels of the FateZero hot path).
 *
 * The reference (ChenyangQiQi/FateZero) has NO native boundary: its seam is Python duck-typing
 * (SURVEY.md §8(b)).  This header therefore defines the boundary the drop-in Python package
 * (fatezero_b200/, re-exported as video_diffusion/) binds with ctypes; every entry point cites the
 * reference Python call site whose GPU work it replaces (paths relative to /root/reference/video_diffusion).
 *
 * Conventions: plain pointers and sizes, no torch types.  All tensor pointers are DEVICE pointers owned by
 * the caller (borrowed for the duration of the call's stream work); fp16 unless stated; `stream` is a
 * cudaStream_t (0 = legacy default stream).  Every function returns 0 on success, non-zero on error, with a
 * human-readable message available from fz_last_error() (thread-local).  No hidden synchronisation.
 */
#ifndef FATEZERO_B200_H
#define FATEZERO_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* fz_stream_t; /* == cudaStream_t */

const char* fz_last_error(void);
int fz_version(void);
/* Runtime probe: returns 0 when the current device is sm_90 and the kernels can run. */
int fz_device_check(void);
/* One-time device-side initialisation (constant tables; synchronises `stream` the first time).  Idempotent.  Must have run before the
 * library is first used under CUDA-graph stream capture (fatezero_b200.engine.UNetEngine calls it at construction). */
int fz_init(fz_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * Tap-GEMM family (wgmma / TMA).  D[M,N] = sum_tap A_tap[M,K] W_tap[N,K]^T  (+ fused epilogue)
 * --------------------------------------------------------------------------------------------------------- */
enum { FZ_EPI_ROWMAJOR = 0, FZ_EPI_GEGLU = 1 };

typedef struct fz_epilogue {
  const float* bias;       /* [gemm columns] fp32 or NULL                                                        */
  const float* group_bias; /* [M / rows_per_group, N] fp32 or NULL: time_emb_proj row per batch element           */
  int rows_per_group;      /*   (resnet.py:355-366 `hidden_states + temb`)                                        */
  const void* residual;    /* [M, ldr] fp16 or NULL: `+ hidden_states` skip connections                           */
  long long ldr;
  const void* residual2;   /* second skip tensor (resnet shortcut next to the LoRA identity skip) or NULL           */
  long long ldr2;
  int mode;                /* FZ_EPI_GEGLU: columns [0,BN/2) x, [BN/2,BN) gate per tile -> x*gelu(gate)           */
                           /*   (GEGLU takes the bias only: residuals, group_bias or out_vt are refused)         */
  int vt_col_start;        /* columns >= vt_col_start are stored transposed into out_vt (V^T for the PV GEMM)     */
  void* out_vt;            /* [M / vt_S, vt_heads, vt_d, vt_S] fp16 or NULL                                       */
  int vt_S, vt_d, vt_heads; /* row m = bf*vt_S + s  ->  out_vt[((bf*heads + h)*d + dd)*vt_ld + s]                  */
  int vt_ld;               /* 0 = vt_S                                                                            */
} fz_epilogue_t;

/* nn.Linear / 1x1 conv: attention_register.py:81,99-100,124,156-160,214; models/attention.py:114,132,320; resnet.py:331 */
int fz_gemm_f16(const void* A, long long lda, const void* W, long long ldw, int M, int N, int K,
                const fz_epilogue_t* epi, void* out, long long ldo, int force_block_n, fz_stream_t stream);
/* per-frame 3x3 conv of PseudoConv3d.forward (resnet.py:57-64), stride 1 or 2, NHWC */
int fz_conv3x3_nhwc_f16(const void* x, long long ldx, int NB, int H, int W, int Cin, const void* w, int Cout, int stride,
                        const fz_epilogue_t* epi, void* out, long long ldo, int force_block_n, fz_stream_t stream);
/* the VAE encoder's downsample (diffusers Downsample2D, padding 0: F.pad(x, (0, 1, 0, 1)) then a 3x3 stride-2 conv without padding) */
int fz_conv3x3_down_asym_nhwc_f16(const void* x, long long ldx, int NB, int H, int W, int Cin, const void* w, int Cout,
                                  const fz_epilogue_t* epi, void* out, long long ldo, int force_block_n, fz_stream_t stream);
/* temporal Conv1d(k=3) of LoRALinearLayer / conv_temporal (resnet.py:72-78, lora.py:46-54) */
int fz_tconv3_f16(const void* x, long long ldx, int B, int F, int HW, int Cin, const void* w, int Cout,
                  const fz_epilogue_t* epi, void* out, long long ldo, int force_block_n, fz_stream_t stream);
/* same conv when the frames of the clip are sharded over GPUs: x_ext is [B, F+2, HW, Cin], frames 0 and F+1 are the neighbour ranks'
 * boundary frames (zeros at the clip ends = the conv's zero padding), the F output frames are the interior ones */
int fz_tconv3_halo_f16(const void* x_ext, long long ldx, int B, int F, int HW, int Cin, const void* w, int Cout,
                       const fz_epilogue_t* epi, void* out, long long ldo, int force_block_n, fz_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * Fused attention with the inline controller (replaces the monkeypatched closures of
 * prompt_attention/attention_register.py:23-59,71-128,131-218 and the controller calls they make into
 * attention_store.py:38-49,81-93 / attention_util.py:80-92,102-158,213-253,282-286).
 * --------------------------------------------------------------------------------------------------------- */
enum {
  FZ_ATTN_NONE = 0,      /* plain attention                                                                    */
  FZ_ATTN_STORE = 1,     /* inversion: write fp16 probabilities to `store` (+ optional running sum `acc`)      */
  FZ_ATTN_REPLACE = 2,   /* edit / self: probabilities come from `base`                                        */
  FZ_ATTN_BLEND = 3,     /* edit / self: rows with mask==0 come from `base`                                    */
  FZ_ATTN_CROSSEDIT = 4  /* edit / cross: refine|replace, reweight, alpha-lerp against `base` (+ `acc`)        */
};

/* device table consumed by FZ_ATTN_CROSSEDIT (floats):
 *   [0] mode (0 refine, 1 replace)  [1..7] reserved
 *   [8 .. 88)   alpha[80]   cross_replace_alpha of this step (ptp_utils.py:179-199)
 *   [88 .. 168) eq[80]      equalizer row, 1.0 when no Reweight (attention_util.py:307-316)
 *   [168 .. 248) a[80]      refinement alphas (seq_aligner.py:113-114)
 *   [248 .. 328) mapper[80] refinement mapper as float (seq_aligner.py:115-117)
 *   [328 .. 328+6400) M[80][80] replacement matrix M[w][n] (seq_aligner.py:152-185)                             */
#define FZ_XEDIT_FLOATS (8 + 4 * 80 + 80 * 80)

typedef struct fz_attn_args {
  const void* q;   long long ldq;   /* Q rows  [BF*S_q, ldq], head h at columns [h*d, h*d+d)                        */
  const void* k;   long long ldk;   /* K rows  [n_src*keys_per_slot, ldk], same column convention                   */
  const void* vt;  long long vt_ld; /* V^T     [n_src, heads, d, vt_ld]                                             */
  void* out;       long long ldo;   /* O rows  [BF*S_q, ldo]                                                        */
  int S_q, keys_per_slot, n_slots, n_src;
  int d, heads, F, BF;
  float scale;
  const int* src_index;             /* HOST array [n_slots][BF]: K/V source row of each query frame                 */
  int edit_bf_start;                /* query frames >= this use row_mode (0 in inversion, F under CFG)             */
  int row_mode;
  void* store;                      /* cache slab written  [BF-edit_bf_start, heads, S_q, cache_ld] fp16             */
  const void* base;                 /* cache slab read     (same geometry)                                           */
  long long cache_ld;               /* n_slots*S_q for self maps; 80 for cross maps (77 keys padded to 16 bytes)     */
                                    /*   must split into n_slots runs of cache_ld/n_slots >= keys_per_slot keys      */
  void* acc;       long long acc_ld;/* fp16 running sum slab or NULL (attention_store.py:95-101)                    */
  const float* xedit;               /* device table, see above                                                       */
  const float* mask;                /* device [BF-edit_bf_start, S_q], 1 = keep current row                          */
  void* dbg;                        /* reserved, ignored (may be NULL)                                                   */
  int causal;                       /* 1: key n is visible to query s only if n <= s (CLIP text encoder; needs n_slots == 1, row_mode NONE) */
} fz_attn_args_t;

int fz_attention_f16(const fz_attn_args_t* args, fz_stream_t stream);

/* Several edited row groups in one launch: one inverted clip edited with n_groups target prompts under one CFG batch
 * [uncond_1..K ; cond_1..K].  Rows bf >= args->edit_bf_start belong to group g = (bf - edit_bf_start) / F and read cache frame
 * fc = (bf - edit_bf_start) % F of the SAME `base` slab [F, heads, S_q, cache_ld] (the inversion map of the step); BF - edit_bf_start
 * must equal n_groups * F.  The per-row hook fields of `args` (row_mode, xedit, mask, acc) are ignored: each group brings its own.
 * Modes NONE / REPLACE / BLEND / CROSSEDIT / STORE may be mixed in one launch (STORE groups all write args->store: use
 * fz_attention_grouped_slabs_f16 below to give each its own slab).  BF <= 128 (fz_attention_f16: BF <= 64).
 * Every row computes exactly what fz_attention_f16 computes for it with its group's hook, so each group's rows and `acc` are bitwise
 * equal to a launch over that group alone. */
#define FZ_ATTN_MAX_GROUPS 8
typedef struct fz_attn_group {
  int row_mode;                     /* FZ_ATTN_NONE / REPLACE / BLEND / CROSSEDIT                                       */
  const float* xedit;               /* CROSSEDIT: device table (layout above)                                           */
  const float* mask;                /* BLEND: device [F, S_q], 1 = keep current row                                     */
  void* acc;                        /* fp16 running sum slab [F, heads, S_q, args->acc_ld] or NULL                       */
} fz_attn_group_t;
typedef struct fz_attn_groups {
  int n_groups;                     /* 1 .. FZ_ATTN_MAX_GROUPS                                                          */
  fz_attn_group_t g[FZ_ATTN_MAX_GROUPS];
} fz_attn_groups_t;
int fz_attention_grouped_f16(const fz_attn_args_t* args, const fz_attn_groups_t* groups, fz_stream_t stream);

/* The grouped launch with a cache slab per group, so that groups of different clips share one launch: the batched inversion of
 * several clips (p2p_ddim_spatial_temporal.py:68-129 once per clip in test_fatezero_dataset.py; one STORE group of F rows per clip,
 * edit_bf_start = 0) and the batched edit of several clips (:172-222; each group reads the inversion map of its own clip).  Group g
 * writes (STORE) cache frame fc = (bf - edit_bf_start) % F of store[g] and adds to its own running sum groups->g[g].acc; REPLACE /
 * BLEND / CROSSEDIT read base[g].  A NULL entry means the slab of `args` (store / base), so `slabs` == NULL or all-NULL is exactly
 * fz_attention_grouped_f16.  Every slab has the geometry [F, heads, S_q, args->cache_ld].  STORE may be mixed with the other modes. */
typedef struct fz_attn_slabs {
  void* store[FZ_ATTN_MAX_GROUPS];       /* STORE: cache slab written by group g, or NULL                                    */
  const void* base[FZ_ATTN_MAX_GROUPS];  /* REPLACE / BLEND / CROSSEDIT: cached source map read by group g, or NULL             */
} fz_attn_slabs_t;
int fz_attention_grouped_slabs_f16(const fz_attn_args_t* args, const fz_attn_groups_t* groups, const fz_attn_slabs_t* slabs,
                                   fz_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * HBM-bound kernels of the step
 * --------------------------------------------------------------------------------------------------------- */
/* GroupNorm (+SiLU) on NHWC fp16. frames_per_stat = F reproduces nn.GroupNorm on the 5-D tensor (resnet.py:338,369;
 * unet_3d_condition.py:439); 1 = per-frame (models/attention.py:112). workspace_f64: 1 MiB scratch (per-chunk partial sums, per-set statistics, arrival counters); it must be
 * zero-filled once before the first call and is left consistent by every call (calls sharing it must be stream-ordered). */
int fz_groupnorm_nhwc_f16(const void* x, void* y, int NB, int HW, int C, int groups, int frames_per_stat, const float* gamma,
                          const float* beta, float eps, int silu, void* workspace_f64, fz_stream_t stream);
/* Same normalisation of a batch made of NB / images_per_item items (prompts of a batched edit): the partial-sum chunking of the
 * statistics pass is planned for images_per_item images, so every image's statistics are bitwise those of a call over its item alone
 * (fz_groupnorm_nhwc_f16 plans it for NB images).  images_per_item must divide NB and be a multiple of frames_per_stat. */
int fz_groupnorm_batched_nhwc_f16(const void* x, void* y, int NB, int HW, int C, int groups, int frames_per_stat, int images_per_item,
                                  const float* gamma, const float* beta, float eps, int silu, void* workspace_f64, fz_stream_t stream);

/* Frame-sharded GroupNorm (one clip's frames over several GPUs, SURVEY.md 8(e); resnet.py:338,369 normalise over ALL frames):
 * fz_groupnorm_stats_f16 leaves float2 (sum, sumsq) [NB][groups] at workspace_f64 + 768 KiB; the caller adds the per-set sums over
 * the ranks and passes them to fz_groupnorm_apply_f16 as image_sums, float2 (sum, sumsq) [NB][groups], or to
 * fz_groupnorm_apply_sums64_f16 as double2 [NB][groups] (fz_gn_combine's fp64 set totals).  The apply kernel adds frames_per_stat
 * consecutive images of a set in fp64 and divides by C/groups * HW * count_frames, count_frames = frames of the set on ALL ranks. */
int fz_groupnorm_stats_f16(const void* x, int NB, int HW, int C, int groups, void* workspace_f64, fz_stream_t stream);
int fz_groupnorm_apply_f16(const void* x, void* y, int NB, int HW, int C, int groups, int frames_per_stat, int count_frames,
                           const float* gamma, const float* beta, float eps, int silu, const void* image_sums, fz_stream_t stream);
int fz_groupnorm_apply_sums64_f16(const void* x, void* y, int NB, int HW, int C, int groups, int frames_per_stat, int count_frames,
                                  const float* gamma, const float* beta, float eps, int silu, const void* image_sums, fz_stream_t stream);
/* nn.LayerNorm over channels of token rows (models/attention.py:281,303,320,331) */
int fz_layernorm_f16(const void* x, void* y, long long M, int C, const float* gamma, const float* beta, float eps, fz_stream_t stream);
/* F.interpolate(scale_factor=2, mode="nearest") (resnet.py:145) */
int fz_upsample2x_nhwc_f16(const void* x, void* y, int NB, int H, int W, int C, fz_stream_t stream);
/* torch.cat([hidden, skip], dim=1) (unet_3d_blocks.py:522,611) */
int fz_concat_channels_f16(const void* a, int Ca, const void* b, int Cb, void* y, long long rows, fz_stream_t stream);
/* latents [B,Cl,F,H,W] fp32 -> im2col rows [B*F*H*W, 64] fp16 for conv_in (unet_3d_condition.py:375) */
int fz_im2col_latents_f16(const float* x, void* out, int B, int Cl, int F, int H, int W, fz_stream_t stream);
/* conv_out tail: temporal conv over frames + scatter to eps [B,Co,F,H,W] fp32 (unet_3d_condition.py:441) */
int fz_out_temporal_f32(const void* y, int ldy, float* eps, int B, int Co, int F, int HW, const float* down, const float* up, int rank,
                        const float* w_full, const float* b_full, fz_stream_t stream);
/* y[n] = bias[n] + sum_k act(x[k]) W[n,k]; W fp16 (time embedding MLP and the 22 time_emb_proj rows, resnet.py:355) */
int fz_rowvec_linear(const float* x, const void* W_f16, const float* bias, float* y, int N, int K, int silu_in, fz_stream_t stream);
int fz_timestep_sinusoid(float t, float* out, int C0, int flip_sin_to_cos, float freq_shift, fz_stream_t stream);
/* temporal attention over frames (models/attention.py:327-337): qkv [B*F*HW, 3C] -> out [B*F*HW, C], 1 <= F <= 32 */
int fz_temporal_attn_f16(const void* qkv, void* out, int B, int F, int HW, int heads, int d, float scale, fz_stream_t stream);
/* x <- inversion step (p2p_ddim_spatial_temporal.py:150-161) */
int fz_ddim_invert_step(float* x, const float* eps, long long n, float alpha_prev, float alpha_next, fz_stream_t stream);
/* x <- CFG + DDIM eta=0 step (+ latent blend x_inv + m (x - x_inv)) (p2p_ddim_spatial_temporal.py:400-407; spatial_blend.py:116-122) */
int fz_cfg_ddim_step(float* x, const float* eps2, long long n, float guidance, float alpha_t, float alpha_prev, const float* x_inv,
                     const float* mask_a, const float* mask_b, long long fhw, int apply_blend, fz_stream_t stream);
/* The same step for K <= 8 items (prompts of a batched edit): x [K, n_item], eps2 [uncond_1..K ; cond_1..K] x n_item, x_inv [n_item]
 * shared by every item; mask_a / mask_b / apply_blend: HOST arrays [K] (device mask pointers, NULL where an item does not blend).
 * Item k gets exactly the arithmetic of fz_cfg_ddim_step on its slice (which is this call with K = 1). */
int fz_cfg_ddim_step_batched(float* x, const float* eps2, int K, long long n_item, float guidance, float alpha_t, float alpha_prev,
                             const float* x_inv, const float* const* mask_a, const float* const* mask_b, const int* apply_blend,
                             long long fhw, fz_stream_t stream);
/* The same step for K <= 8 items of possibly different clips (the edit jobs of p2preplace_edit_clips: :400-407 once per clip): x_inv is a
 * HOST array [K] of device pointers, one inverted latent [n_item] per item (two items may share one; NULL where an item does not blend).
 * Item k gets exactly the arithmetic of fz_cfg_ddim_step on its slice with x_inv[k]. */
int fz_cfg_ddim_step_multi(float* x, const float* eps2, int K, long long n_item, float guidance, float alpha_t, float alpha_prev,
                           const float* const* x_inv, const float* const* mask_a, const float* const* mask_b, const int* apply_blend,
                           long long fhw, fz_stream_t stream);
/* x <- one DDIM sampling step (stable_diffusion.py:533-541 + diffusers-0.11.1 DDIMScheduler.step with eta) on K items of n_item fp32
 * elements: e = eu + guidance (ec - eu) with eps = [uncond_1..K ; cond_1..K] (cfg = 1) or e = eps [K, n_item] (cfg = 0);
 * x0 = (x - sqrt(1 - alpha_t) e) / sqrt(alpha_t); x <- sqrt(alpha_prev) x0 + sqrt(1 - alpha_prev - sigma^2) e + sigma noise.
 * sigma = eta sqrt((1 - alpha_prev) / (1 - alpha_t)) sqrt(1 - alpha_t / alpha_prev) >= 0; noise [K, n_item] fp32 (NULL allowed when
 * sigma = 0).  cfg = 1, sigma = 0 is bitwise fz_cfg_ddim_step without blend. */
int fz_ddim_sample_step(float* x, const float* eps, int K, long long n_item, int cfg, float guidance, float alpha_t, float alpha_prev,
                        float sigma, const float* noise, fz_stream_t stream);
/* blend mask from cached cross maps (spatial_blend.py:24-39,78-111); maps: HOST array of device pointers [F, heads, rh*rw, ldm],
 * word_w: HOST [ntok].  The rh x rw grid (rh * rw <= 1024) is max-pooled and resized to h x w with F.interpolate's nearest index per axis.
 * fz_blend_mask is the square grid rh = rw = r. */
int fz_blend_mask_hw(const void* const* maps, int num_maps, int maps_f32, int F, int heads, int rh, int rw, int ldm, int ntok,
                     const float* word_w, float th, int h, int w, float* out, fz_stream_t stream);
int fz_blend_mask(const void* const* maps, int num_maps, int maps_f32, int F, int heads, int r, int ldm, int ntok, const float* word_w,
                  float th, int h, int w, float* out, fz_stream_t stream);

/* CLIP text encoder pieces (pipelines/stable_diffusion.py:230,279 call transformers' CLIPTextModel): token + position embedding rows
 * out[r, :] = fp16(tok[ids[r], :] + pos[r % L, :]) and the quick_gelu activation x * sigmoid(1.702 x) in place. */
int fz_embed_tokens_f16(const float* tok, const float* pos, const long long* ids, void* out, int rows, int L, int C, fz_stream_t stream);
int fz_quick_gelu_f16(void* x, long long n, fz_stream_t stream);
/* exact GELU 0.5 x (1 + erf(x / sqrt 2)) in place, fp32 math with erff: the MLP activation of the SD-2 text encoders (hidden_act "gelu",
 * transformers' CLIPMLP.forward -> ACT2FN["gelu"] = torch.nn.functional.gelu without the tanh approximation) */
int fz_gelu_f16(void* x, long long n, fz_stream_t stream);

/* in-place row softmax x[r, :n] <- softmax(scale * x[r, :n]), fp32 math: the VAE's 512-wide single-head attention runs GEMM -> this -> GEMM */
int fz_softmax_rows_f16(void* x, long long rows, int n, long long ld, float scale, fz_stream_t stream);

/* show_cross_attention on the device (prompt_attention/visualization.py:14-72): out[f, tok, rh*rw] = 255 * a / max(a) with a = sum over the
 * given cross-attention maps ([F, heads, rh*rw, ldm] fp16 or fp32 running sums, rh * rw <= 1024) and heads of the probability of text token
 * tok (the means' constant factors cancel).  The reference averages every stored map and copies the r16 cross maps to the host first.
 * fz_cross_heatmaps is the square grid rh = rw = res. */
int fz_cross_heatmaps_hw(const void* const* maps, int num_maps, int maps_f32, int F, int heads, int rh, int rw, int ldm, int ntok,
                         unsigned char* out, fz_stream_t stream);
int fz_cross_heatmaps(const void* const* maps, int num_maps, int maps_f32, int F, int heads, int res, int ldm, int ntok, unsigned char* out,
                      fz_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * CLIP evaluation of edited clips (paths relative to the reference's CLIP/ directory): frame accuracy and temporal consistency of
 * frame_acc_tem_con.py:11-54 with a CLIP ViT (clip/model.py:206-238 image tower, :343-372 text tower and logits).  The transformer
 * blocks run on fz_gemm_f16 / fz_attention_f16 / fz_layernorm_f16 / fz_quick_gelu_f16; these are the pieces around them.
 * --------------------------------------------------------------------------------------------------------- */
#define FZ_CLIP_MAX_SIDE 8192 /* largest input or resized side, in pixels                                          */
#define FZ_CLIP_MAX_CLIPS 256 /* clips per fz_clip_scores launch                                                    */
/* decode_latents + numpy_to_pil (pipelines/stable_diffusion.py:297-319,566-576) on the device: x [N,3,H,W] fp32 (x_f16 = 0) or fp16 in
 * [-1,1] -> out [N,H,W,3] uint8 = round_half_even(clamp(x / 2 + 0.5, 0, 1) * 255), the fp16 case evaluated in fp16 as torch does. */
int fz_frames_to_u8(const void* x, int x_f16, unsigned char* out, int N, int H, int W, fz_stream_t stream);
/* PIL Image.resize(BICUBIC) as torchvision's Resize calls it (clip/clip.py:79-86; Pillow libImaging/Resample.c, 8 bits per channel):
 * in [N,H,W,3] uint8 (crop_bottom_square: a frame with H > W is first cropped to its bottom W x W square, frame_acc_tem_con.py:11-16)
 * -> out [N,Ho,Wo,3].  kx [Wo, kw_x] / ky [Ho, kw_y]: device int32 weights with 22 fractional bits; bx [Wo][2] / by [Ho][2]: device int32
 * (first input pixel, tap count) per output pixel (host tables: fatezero_b200.clip_eval.resize_coeffs).  tmp: [N, H', Wo, 3] uint8 scratch
 * for the horizontal pass (H' = the cropped height). */
int fz_resize_bicubic_u8(const unsigned char* in, int N, int H, int W, int crop_bottom_square, const int* kx, const int* bx, int kw_x, int Wo,
                         const int* ky, const int* by, int kw_y, int Ho, unsigned char* tmp, unsigned char* out, fz_stream_t stream);
/* CenterCrop(res) + ToTensor + Normalize(mean3, std3) (clip/clip.py:79-86), rounded to fp16 (model.py:340 `image.type(self.dtype)`), written
 * as the im2col rows of conv1 (model.py:222): img [N,Hr,Wr,3] uint8 -> out [N*(res/patch)^2, 3*patch*patch] fp16, column c*patch^2 + ky*patch
 * + kx.  mean3 / std3: HOST arrays. */
int fz_clip_patchify_f16(const unsigned char* img, int N, int Hr, int Wr, int res, int patch, const float* mean3, const float* std3, void* out,
                         fz_stream_t stream);
/* model.py:223-227: out[n*T + t] = ln_pre((t == 0 ? class_emb : patches[n*(T-1) + t-1]) + pos_emb[t]) with fp32 statistics, fp16 out.
 * patches [N*(T-1), C] fp16 (the conv1 GEMM), class_emb [C], pos_emb [T, C], gamma / beta [C] fp32; C % 8 == 0, C <= 1024. */
int fz_clip_embed_f16(const void* patches, const float* class_emb, const float* pos_emb, const float* gamma, const float* beta, float eps,
                      int N, int T, int C, void* out, fz_stream_t stream);
/* Scoring head, fp32, one launch (frame_acc_tem_con.py:19-54, model.py:358-372): img [N,D] image features of K clips stored clip after clip
 * (clip_frames: HOST [K] frame counts summing to N), txt [P,D] text features, pairs: HOST [K][2] (source, target) text rows per clip.
 * Writes img_norm [N], txt_norm [P] (L2 norms); logits [N][2] = scale * cos(frame, source|target), probs [N][2] their two-way softmax;
 * success [N] int32 = logit_target >= logit_source; margin [N] = logit_target - logit_source; cosine [N] = cos(frame i, frame i+1) within
 * the clip (NaN on a clip's last frame); clip_mean [K] = the mean of a clip's cosines (NaN for a one-frame clip). */
int fz_clip_scores(const float* img, const float* txt, int N, int P, int D, const int* clip_frames, const int* pairs, int K, float scale,
                   float* img_norm, float* txt_norm, float* logits, float* probs, int* success, float* margin, float* cosine, float* clip_mean,
                   fz_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * Frame-sharded execution over the GPUs of one NVSwitch box (one process per GPU): peer-memory exchange.
 * Replaces, for the frames-of-one-clip split of SURVEY.md §8(e), what the reference gets for free from holding every frame on one
 * device: K / V of other frames (prompt_attention/attention_register.py:162-193), joint-frame GroupNorm statistics
 * (models/resnet.py:338,369), the frame halo of the temporal Conv1d (models/resnet.py:72-78) and the frames<->pixels exchange of the
 * temporal attention (models/attention.py:327-337).  A symmetric arena (fz_p2p_alloc on every rank, exported / imported with CUDA IPC)
 * gives every rank a pointer into every peer; fz_p2p_push copies 2-D segments into peers with 16-byte NVLink stores and raises a flag in
 * the destination's arena when all of its segments have landed; fz_p2p_wait / fz_gn_combine spin on the LOCAL flags and clear them.
 * --------------------------------------------------------------------------------------------------------- */
typedef struct {
  const void* src;      /* local source (16-byte aligned) */
  long long src_pitch;  /* bytes between source rows */
  void* dst;            /* destination: pointer into the peer's (or the own) arena */
  long long dst_pitch;
  int rows;
  int row_bytes;        /* multiple of 16 */
  int dst_slot;         /* which flag / counter the segment reports to; -1 = local copy, no flag */
} fz_p2p_seg_t;
int fz_p2p_alloc(long long nbytes, void** ptr);              /* cudaMalloc + zero fill (flags start cleared) */
int fz_p2p_free(void* ptr);
int fz_p2p_export(void* ptr, void* handle64);                /* cudaIpcMemHandle_t, 64 bytes */
int fz_p2p_import(const void* handle64, void** ptr);         /* peer pointer valid in this process */
int fz_p2p_unimport(void* ptr);
/* Exchange in one launch: copy the segments, raise flags[d] (flag word in destination d's arena, peer pointer) once everything has been
 * written, then — if wait_flags is not null — wait for (and clear) this rank's own incoming flags selected by wait_mask (bit r = source
 * rank r; wait_flags = the site's 32 local flag words).  counter: local zero-initialised arrival counter.  dst_slot of a segment is
 * informational (-1 = local copy). */
int fz_p2p_push(const fz_p2p_seg_t* segs, int n_segs, void* const* flags, void* counter, int n_dst, void* wait_flags, unsigned wait_mask,
                fz_stream_t stream);
/* flags: local array of up to 32 flag words; waits for (and clears) those selected by mask */
int fz_p2p_wait(void* flags, unsigned mask, fz_stream_t stream);
/* GroupNorm statistics exchange in one single-CTA launch, low-latency protocol: every (sum, sumsq) of sums [NB*G] float2 is written into
 * peer_inbox[r] (rank r's inbox slot for this rank, [NB*G][2] 8-byte words {value, epoch}); the kernel then polls the local inbox
 * ([world][NB*G][2] words) until every peer's words carry this use's epoch (`epoch`: local per-site counter, advanced by the kernel), adds
 * them to sums in fp64 and leaves each statistics set's total in the slot of its first local image of totals [NB*G] double2, 0 in the
 * other slots (input layout of fz_groupnorm_apply_sums64_f16). */
int fz_gn_combine(void* epoch, void* const* peer_inbox, const void* inbox, const void* sums, void* totals, int NB, int F_loc, int G, int world,
                  int me, fz_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* FATEZERO_B200_H */
