// fz_clip.cu — CLIP ViT evaluation of edited frames (CLIP/frame_acc_tem_con.py of the reference): decoded-frame quantisation, Pillow's
// two-pass fixed-point bicubic resize, the CLIP preprocess + patch im2col, the image tower's token embedding + ln_pre, and the scoring head
// (frame accuracy and temporal consistency).  The transformer blocks themselves run on fz_gemm / fz_attention / fz_layernorm.
#include "fz_common.cuh"

#include <cmath>

#include "../../include/fatezero_b200.h"

namespace fz {

// ---------------------------------------------------------------------------------------------------------------
// decoded VAE frames [N,3,H,W] in [-1,1] -> uint8 [N,H,W,3]: numpy_to_pil((x / 2 + 0.5).clamp(0, 1) * 255).round())
// ---------------------------------------------------------------------------------------------------------------
template <bool F16>
__global__ void frames_to_u8_kernel(const void* __restrict__ x, unsigned char* __restrict__ out, int N, long long HW) {
  const long long total = static_cast<long long>(N) * HW;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long n = i / HW, p = i - n * HW;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const long long src = (n * 3 + c) * HW + p;
      float v;
      if (F16) {
        // torch evaluates `image / 2 + 0.5` and the clamp in fp16 for an fp16 tensor (each op rounded to fp16), then .float()
        const __half h = static_cast<const __half*>(x)[src];
        __half t = __float2half_rn(__fmul_rn(__half2float(h), 0.5f));
        t = __float2half_rn(__fadd_rn(__half2float(t), 0.5f));
        v = __half2float(t);
      } else {
        v = __fadd_rn(__fmul_rn(static_cast<const float*>(x)[src], 0.5f), 0.5f);
      }
      v = fminf(fmaxf(v, 0.f), 1.f);
      // numpy: float32 * 255 then np.round (half to even) then astype(uint8)
      out[i * 3 + c] = static_cast<unsigned char>(rintf(__fmul_rn(v, 255.f)));
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Pillow ImagingResample (libImaging/Resample.c), 8 bits per channel: per output pixel a run of `cnt` taps starting at `start`, int32 weights
// with 22 fractional bits; accumulate from 2^21, >> 22, clamp to 0..255.  The horizontal pass runs first into a uint8 image.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kPrecisionBits = 22;

__device__ __forceinline__ unsigned char clip8(int ss) {
  ss >>= kPrecisionBits;
  return static_cast<unsigned char>(ss < 0 ? 0 : ss > 255 ? 255 : ss);
}

// in [N, H, W, 3] (rows [row0, row0 + Hc) are used: the bottom-square crop) -> tmp [N, Hc, Wo, 3]
__global__ void resize_h_kernel(const unsigned char* __restrict__ in, int H, int W, int row0, int Hc, const int* __restrict__ kx,
                                const int* __restrict__ bx, int kw, int Wo, unsigned char* __restrict__ tmp, long long total) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int xo = static_cast<int>(i % Wo);
    const long long ny = i / Wo;
    const int y = static_cast<int>(ny % Hc);
    const long long n = ny / Hc;
    const unsigned char* row = in + ((n * H + row0 + y) * W) * 3;
    const int s = bx[2 * xo], cnt = min(bx[2 * xo + 1], kw);
    const int* k = kx + static_cast<long long>(xo) * kw;
    int s0 = 1 << (kPrecisionBits - 1), s1 = s0, s2 = s0;
    for (int t = 0; t < cnt; ++t) {
      const int xi = min(max(s + t, 0), W - 1);
      const int w = k[t];
      s0 += row[xi * 3 + 0] * w;
      s1 += row[xi * 3 + 1] * w;
      s2 += row[xi * 3 + 2] * w;
    }
    unsigned char* o = tmp + i * 3;
    o[0] = clip8(s0);
    o[1] = clip8(s1);
    o[2] = clip8(s2);
  }
}

// tmp [N, Hc, Wo, 3] -> out [N, Ho, Wo, 3]
__global__ void resize_v_kernel(const unsigned char* __restrict__ tmp, int Hc, int Wo, const int* __restrict__ ky, const int* __restrict__ by,
                                int kw, int Ho, unsigned char* __restrict__ out, long long total) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int xo = static_cast<int>(i % Wo);
    const long long ny = i / Wo;
    const int yo = static_cast<int>(ny % Ho);
    const long long n = ny / Ho;
    const int s = by[2 * yo], cnt = min(by[2 * yo + 1], kw);
    const int* k = ky + static_cast<long long>(yo) * kw;
    int s0 = 1 << (kPrecisionBits - 1), s1 = s0, s2 = s0;
    for (int t = 0; t < cnt; ++t) {
      const int yi = min(max(s + t, 0), Hc - 1);
      const unsigned char* p = tmp + ((n * Hc + yi) * Wo + xo) * 3;
      const int w = k[t];
      s0 += p[0] * w;
      s1 += p[1] * w;
      s2 += p[2] * w;
    }
    unsigned char* o = out + i * 3;
    o[0] = clip8(s0);
    o[1] = clip8(s1);
    o[2] = clip8(s2);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// CenterCrop(res) + ToTensor + Normalize, rounded to fp16, written as conv1 im2col rows: row n*g*g + py*g + px, column c*P*P + ky*P + kx
// (the K order of conv1.weight.reshape(width, -1)).
// ---------------------------------------------------------------------------------------------------------------
struct ClipNorm {
  float mean[3], std[3];
};

__global__ void __launch_bounds__(256) patchify_kernel(const unsigned char* __restrict__ img, int Hr, int Wr, int top, int left, int res, int P,
                                                       const ClipNorm nrm, __half* __restrict__ out) {
  const int g = res / P;
  const int r = blockIdx.x;  // patch row
  const int n = r / (g * g), pp = r % (g * g), py = pp / g, px = pp % g;
  const int K = 3 * P * P;
  __half* o = out + static_cast<long long>(r) * K;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const int c = k / (P * P), kk = k % (P * P), ky = kk / P, kx = kk % P;
    const int y = top + py * P + ky, x = left + px * P + kx;
    const unsigned char u = img[((static_cast<long long>(n) * Hr + y) * Wr + x) * 3 + c];
    // torchvision: img.float().div(255), then tensor.sub_(mean).div_(std), all fp32 and correctly rounded
    const float t = __fdiv_rn(static_cast<float>(u), 255.f);
    o[k] = __float2half_rn(__fdiv_rn(__fsub_rn(t, nrm.mean[c]), nrm.std[c]));
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Image-tower token embedding: token 0 = class_embedding, tokens 1..T-1 = the patch-GEMM rows; + positional_embedding; then ln_pre
// (centred two-pass statistics in fp32, mean = sum / C and var = sum (x - mean)^2 / C as divisions).  One warp per token row.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kEmbedMaxPerLane = 32;  // C <= 1024

__global__ void __launch_bounds__(256) clip_embed_kernel(const __half* __restrict__ patches, const float* __restrict__ cls,
                                                         const float* __restrict__ pos, const float* __restrict__ gamma,
                                                         const float* __restrict__ beta, float eps, int N, int T, int C,
                                                         __half* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long row = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (row >= static_cast<long long>(N) * T) return;
  const long long n = row / T;
  const int t = static_cast<int>(row % T);
  const float* pr = pos + static_cast<long long>(t) * C;
  const __half* src = patches + (n * (T - 1) + (t - 1)) * C;
  float v[kEmbedMaxPerLane];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < kEmbedMaxPerLane; ++i) {
    const int c = lane + 32 * i;
    v[i] = 0.f;
    if (c < C) {
      const float base = t == 0 ? cls[c] : __half2float(src[c]);
      v[i] = __fadd_rn(base, pr[c]);
      sum += v[i];
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = __fdiv_rn(sum, static_cast<float>(C));
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < kEmbedMaxPerLane; ++i) {
    if (lane + 32 * i < C) {
      const float d = v[i] - mean;
      sq = fmaf(d, d, sq);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = __fdiv_rn(1.f, __fsqrt_rn(__fadd_rn(__fdiv_rn(sq, static_cast<float>(C)), eps)));
  __half* o = out + row * C;
#pragma unroll
  for (int i = 0; i < kEmbedMaxPerLane; ++i) {
    const int c = lane + 32 * i;
    if (c < C) o[c] = __float2half_rn(fmaf((v[i] - mean) * rstd, gamma[c], beta[c]));
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Scoring head (frame_acc_tem_con.py:19-54 and model.py:358-372), one CTA: L2 norms of every feature row; per frame the logits
// scale * <f/|f|, t/|t|> against its clip's source and target prompt, their two-way softmax, success = logit_t >= logit_s and the margin
// logit_t - logit_s; the cosine of each frame with the next frame of its clip and the per-clip mean of those cosines (summed in frame
// order).  Reductions run over the D features in a fixed order, so a frame's results do not depend on the other clips in the launch.
// ---------------------------------------------------------------------------------------------------------------
struct ScoreParams {
  int frames[FZ_CLIP_MAX_CLIPS];
  int src[FZ_CLIP_MAX_CLIPS];
  int tgt[FZ_CLIP_MAX_CLIPS];
  int K, N, P, D;
  float scale;
};
static_assert(sizeof(ScoreParams) <= 4000, "kernel parameter block limit");

__device__ __forceinline__ float warp_dot_normed(const float* a, float na, const float* b, float nb, int D, int lane) {
  float s = 0.f;
  for (int c = lane; c < D; c += 32) s = fmaf(__fdiv_rn(a[c], na), __fdiv_rn(b[c], nb), s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}

__global__ void __launch_bounds__(1024) clip_scores_kernel(const float* __restrict__ img, const float* __restrict__ txt, const __grid_constant__ ScoreParams p,
                                                           float* __restrict__ img_norm, float* __restrict__ txt_norm, float* __restrict__ logits,
                                                           float* __restrict__ probs, int* __restrict__ success, float* __restrict__ margin,
                                                           float* __restrict__ cosine, float* __restrict__ clip_mean) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int r = warp; r < p.N + p.P; r += nw) {
    const float* f = r < p.N ? img + static_cast<long long>(r) * p.D : txt + static_cast<long long>(r - p.N) * p.D;
    float s = 0.f;
    for (int c = lane; c < p.D; c += 32) s = fmaf(f[c], f[c], s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) (r < p.N ? img_norm[r] : txt_norm[r - p.N]) = __fsqrt_rn(s);
  }
  __syncthreads();
  for (int i = warp; i < p.N; i += nw) {
    int k = 0, first = 0;
    while (k < p.K && i >= first + p.frames[k]) first += p.frames[k++];
    const float* f = img + static_cast<long long>(i) * p.D;
    const float nf = img_norm[i];
    const int ts = p.src[k], tt = p.tgt[k];
    const float ls = p.scale * warp_dot_normed(f, nf, txt + static_cast<long long>(ts) * p.D, txt_norm[ts], p.D, lane);
    const float lt = p.scale * warp_dot_normed(f, nf, txt + static_cast<long long>(tt) * p.D, txt_norm[tt], p.D, lane);
    float cs = nanf("");
    if (i + 1 < first + p.frames[k]) cs = warp_dot_normed(f, nf, f + p.D, img_norm[i + 1], p.D, lane);
    if (lane == 0) {
      // softmax over the two prompts, max-subtracted like torch's softmax
      const float m = fmaxf(ls, lt);
      const float es = expf(ls - m), et = expf(lt - m);
      const float den = es + et;
      logits[2 * i] = ls;
      logits[2 * i + 1] = lt;
      probs[2 * i] = __fdiv_rn(es, den);
      probs[2 * i + 1] = __fdiv_rn(et, den);
      success[i] = lt >= ls;
      margin[i] = lt - ls;
      cosine[i] = cs;
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < p.K; k += blockDim.x) {
    int first = 0;
    for (int j = 0; j < k; ++j) first += p.frames[j];
    float s = 0.f;
    for (int i = first; i + 1 < first + p.frames[k]; ++i) s += cosine[i];
    clip_mean[k] = p.frames[k] > 1 ? __fdiv_rn(s, static_cast<float>(p.frames[k] - 1)) : nanf("");
  }
}

static int grid_for(long long total) {
  return static_cast<int>(std::min<long long>((total + 255) / 256, 132 * 16));
}

}  // namespace fz

extern "C" int fz_frames_to_u8(const void* x, int x_f16, unsigned char* out, int N, int H, int W, cudaStream_t stream) {
  FZ_CHECK_ARG(x && out, "fz_frames_to_u8: null pointer");
  FZ_CHECK_ARG(N > 0 && H > 0 && W > 0, "fz_frames_to_u8: bad shape N=%d H=%d W=%d", N, H, W);
  const long long HW = static_cast<long long>(H) * W;
  const int grid = fz::grid_for(N * HW);
  if (x_f16)
    fz::frames_to_u8_kernel<true><<<grid, 256, 0, stream>>>(x, out, N, HW);
  else
    fz::frames_to_u8_kernel<false><<<grid, 256, 0, stream>>>(x, out, N, HW);
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}

extern "C" int fz_resize_bicubic_u8(const unsigned char* in, int N, int H, int W, int crop_bottom_square, const int* kx, const int* bx, int kw_x,
                                    int Wo, const int* ky, const int* by, int kw_y, int Ho, unsigned char* tmp, unsigned char* out,
                                    cudaStream_t stream) {
  FZ_CHECK_ARG(in && kx && bx && ky && by && tmp && out, "fz_resize_bicubic_u8: null pointer");
  FZ_CHECK_ARG(N > 0 && H > 0 && W > 0 && H <= FZ_CLIP_MAX_SIDE && W <= FZ_CLIP_MAX_SIDE, "fz_resize_bicubic_u8: input %dx%d out of range (1..%d)",
               W, H, FZ_CLIP_MAX_SIDE);
  FZ_CHECK_ARG(Wo > 0 && Ho > 0 && Wo <= FZ_CLIP_MAX_SIDE && Ho <= FZ_CLIP_MAX_SIDE, "fz_resize_bicubic_u8: output %dx%d out of range (1..%d)",
               Wo, Ho, FZ_CLIP_MAX_SIDE);
  FZ_CHECK_ARG(kw_x > 0 && kw_y > 0 && kw_x <= 2 * FZ_CLIP_MAX_SIDE + 5 && kw_y <= 2 * FZ_CLIP_MAX_SIDE + 5, "fz_resize_bicubic_u8: tap count out of range");
  // frame_acc_tem_con.py:11-16: a portrait frame (h > w) is cropped to its bottom w x w square before the preprocess
  const int Hc = crop_bottom_square && H > W ? W : H;
  const int row0 = H - Hc;
  const long long th = static_cast<long long>(N) * Hc * Wo, tv = static_cast<long long>(N) * Ho * Wo;
  fz::resize_h_kernel<<<fz::grid_for(th), 256, 0, stream>>>(in, H, W, row0, Hc, kx, bx, kw_x, Wo, tmp, th);
  FZ_CUDA(cudaGetLastError());
  fz::resize_v_kernel<<<fz::grid_for(tv), 256, 0, stream>>>(tmp, Hc, Wo, ky, by, kw_y, Ho, out, tv);
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}

extern "C" int fz_clip_patchify_f16(const unsigned char* img, int N, int Hr, int Wr, int res, int patch, const float* mean3, const float* std3,
                                    void* out, cudaStream_t stream) {
  FZ_CHECK_ARG(img && mean3 && std3 && out, "fz_clip_patchify_f16: null pointer");
  FZ_CHECK_ARG(patch > 0 && patch % 8 == 0 && res > 0 && res % patch == 0, "fz_clip_patchify_f16: resolution %d must be a multiple of the patch "
               "size %d, itself a multiple of 8", res, patch);
  FZ_CHECK_ARG(N > 0 && Hr >= res && Wr >= res, "fz_clip_patchify_f16: %dx%d image smaller than the %d crop", Wr, Hr, res);
  fz::ClipNorm nrm;
  for (int c = 0; c < 3; ++c) {
    FZ_CHECK_ARG(std3[c] > 0.f, "fz_clip_patchify_f16: std[%d] must be positive", c);
    nrm.mean[c] = mean3[c];
    nrm.std[c] = std3[c];
  }
  // torchvision CenterCrop: offsets int(round((size - res) / 2.0)), Python's round (half to even)
  const int top = static_cast<int>(std::nearbyint((Hr - res) / 2.0)), left = static_cast<int>(std::nearbyint((Wr - res) / 2.0));
  const int g = res / patch;
  fz::patchify_kernel<<<N * g * g, 256, 0, stream>>>(img, Hr, Wr, top, left, res, patch, nrm, static_cast<__half*>(out));
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}

extern "C" int fz_clip_embed_f16(const void* patches, const float* class_emb, const float* pos_emb, const float* gamma, const float* beta,
                                 float eps, int N, int T, int C, void* out, cudaStream_t stream) {
  FZ_CHECK_ARG(patches && class_emb && pos_emb && gamma && beta && out, "fz_clip_embed_f16: null pointer");
  FZ_CHECK_ARG(N > 0 && T >= 2 && C % 8 == 0 && C > 0 && C <= 32 * fz::kEmbedMaxPerLane, "fz_clip_embed_f16: N=%d T=%d C=%d unsupported "
               "(C %% 8 == 0, C <= %d)", N, T, C, 32 * fz::kEmbedMaxPerLane);
  const long long rows = static_cast<long long>(N) * T;
  fz::clip_embed_kernel<<<static_cast<unsigned>((rows + 7) / 8), 256, 0, stream>>>(static_cast<const __half*>(patches), class_emb, pos_emb,
                                                                                  gamma, beta, eps, N, T, C, static_cast<__half*>(out));
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}

extern "C" int fz_clip_scores(const float* img, const float* txt, int N, int P, int D, const int* clip_frames, const int* pairs, int K,
                              float scale, float* img_norm, float* txt_norm, float* logits, float* probs, int* success, float* margin,
                              float* cosine, float* clip_mean, cudaStream_t stream) {
  FZ_CHECK_ARG(img && txt && clip_frames && pairs && img_norm && txt_norm && logits && probs && success && margin && cosine && clip_mean,
               "fz_clip_scores: null pointer");
  FZ_CHECK_ARG(N > 0 && P > 0 && D > 0, "fz_clip_scores: bad shape N=%d P=%d D=%d", N, P, D);
  FZ_CHECK_ARG(K >= 1 && K <= FZ_CLIP_MAX_CLIPS, "fz_clip_scores: %d clips (1..%d)", K, FZ_CLIP_MAX_CLIPS);
  fz::ScoreParams p;
  long long total = 0;
  for (int k = 0; k < K; ++k) {
    FZ_CHECK_ARG(clip_frames[k] >= 1, "fz_clip_scores: clip %d has %d frames", k, clip_frames[k]);
    FZ_CHECK_ARG(pairs[2 * k] >= 0 && pairs[2 * k] < P && pairs[2 * k + 1] >= 0 && pairs[2 * k + 1] < P,
                 "fz_clip_scores: clip %d: prompt rows (%d, %d) outside 0..%d", k, pairs[2 * k], pairs[2 * k + 1], P - 1);
    p.frames[k] = clip_frames[k];
    p.src[k] = pairs[2 * k];
    p.tgt[k] = pairs[2 * k + 1];
    total += clip_frames[k];
  }
  FZ_CHECK_ARG(total == N, "fz_clip_scores: the clips hold %lld frames, the features %d", total, N);
  p.K = K;
  p.N = N;
  p.P = P;
  p.D = D;
  p.scale = scale;
  fz::clip_scores_kernel<<<1, 1024, 0, stream>>>(img, txt, p, img_norm, txt_norm, logits, probs, success, margin, cosine, clip_mean);
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}
