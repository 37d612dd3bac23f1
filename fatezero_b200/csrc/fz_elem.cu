// fz_elem.cu — HBM-bound kernels of the UNet step: GroupNorm (joint-frame statistics), LayerNorm, nearest upsample,
// channel concat, input im2col / output temporal conv, time embedding, temporal attention, CFG + DDIM + latent blend,
// and the cross-attention blend mask.  All activations are fp16 NHWC ([B*F, H*W, C] == token-major), statistics fp32/fp64,
// 16-byte vector loads/stores, grids sized to cover the 132 SMs.
#include "fz_common.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>

#include "../../include/fatezero_b200.h"

namespace fz {

static inline int sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

struct alignas(16) Half8 {
  __half v[8];
};

// ---------------------------------------------------------------------------------------------------------------
// GroupNorm.  x: [NB, HW, C]; statistics group sidx = (nb / frames_per_stat) * G + g.
// resnet.py:338,369 and unet_3d_condition.py:439 call nn.GroupNorm on the 5-D tensor => frames_per_stat = F (joint);
// models/attention.py:112 normalises "(b f) c h w" => frames_per_stat = 1.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kGnThreads = 256;
constexpr int kGnMaxSlots = 4;
// 1 MiB workspace: [0, 768 KiB) per-CTA partial sums, then (sum, sumsq) per (image, group), then one arrival counter per image.
// The counters must be zero before the first call (the Python layer allocates the workspace zeroed); every call leaves them zero.
constexpr size_t kGnStatsOffset = 768 * 1024;
constexpr size_t kGnCounterOffset = 960 * 1024;

// Statistics pass: every CTA reduces its pixel chunk of one image to per-group partial (sum, sumsq) WITHOUT atomics
// (v0 used ~4k contended shared-memory atomics per CTA): registers -> smem [TY][C] -> per channel -> per group -> partial[nb][chunk][g].
// The chunks are large (about two CTAs per SM for the whole tensor) so that this reduction tail is amortised, and each thread keeps
// kGnBatch independent 16-byte loads in flight.  The LAST CTA of an image folds the image's chunks into image_sums[nb][g]; the apply
// kernel adds the frames_per_stat images of its statistics set (v2 had every apply CTA re-reduce all partials: ~150 KB of L2 reads).
constexpr int kGnBatch = 8;

template <int SLOTS>
__global__ void __launch_bounds__(kGnThreads) gn_stats_kernel(const __half* __restrict__ x, int HW, int C, int G, int TX,
                                                             int px_per_cta, float2* __restrict__ partial,
                                                             float2* __restrict__ image_sums, unsigned* __restrict__ counters) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float gn_smem[];  // [TY][C] sums, [TY][C] sumsq
  const int nb = blockIdx.y;
  const int cpg = C / G;
  const int tx = threadIdx.x % TX, ty = threadIdx.x / TX;
  const int TY = kGnThreads / TX;
  float* s_sum = gn_smem;
  float* s_sq = gn_smem + TY * C;
  float acc[SLOTS][8], acc2[SLOTS][8];
#pragma unroll
  for (int s = 0; s < SLOTS; ++s)
#pragma unroll
    for (int e = 0; e < 8; ++e) { acc[s][e] = 0.f; acc2[s][e] = 0.f; }
  const int p0 = blockIdx.x * px_per_cta;
  const int p1 = min(HW, p0 + px_per_cta);
  if (ty < TY) {
    const __half* xb = x + (static_cast<long long>(nb) * HW) * C;
    constexpr int U = kGnBatch / SLOTS;
    for (int p = p0 + ty; p < p1; p += TY * U) {
      Half8 h[U][SLOTS];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int pp = p + u * TY;
        if (pp < p1) {
#pragma unroll
          for (int s = 0; s < SLOTS; ++s) h[u][s] = *reinterpret_cast<const Half8*>(xb + static_cast<long long>(pp) * C + (tx + s * TX) * 8);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (p + u * TY < p1) {
#pragma unroll
          for (int s = 0; s < SLOTS; ++s) {
#pragma unroll
            for (int e = 0; e < 8; ++e) {
              const float f = __half2float(h[u][s].v[e]);
              acc[s][e] += f;
              acc2[s][e] = fmaf(f, f, acc2[s][e]);
            }
          }
        }
      }
    }
#pragma unroll
    for (int s = 0; s < SLOTS; ++s) {
      const int cv = tx + s * TX;
      float4* d0 = reinterpret_cast<float4*>(s_sum + ty * C + cv * 8);
      float4* d1 = reinterpret_cast<float4*>(s_sq + ty * C + cv * 8);
      d0[0] = make_float4(acc[s][0], acc[s][1], acc[s][2], acc[s][3]);
      d0[1] = make_float4(acc[s][4], acc[s][5], acc[s][6], acc[s][7]);
      d1[0] = make_float4(acc2[s][0], acc2[s][1], acc2[s][2], acc2[s][3]);
      d1[1] = make_float4(acc2[s][4], acc2[s][5], acc2[s][6], acc2[s][7]);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += kGnThreads) {
    float a = 0.f, b = 0.f;
    for (int t = 0; t < TY; ++t) { a += s_sum[t * C + c]; b += s_sq[t * C + c]; }
    s_sum[c] = a;
    s_sq[c] = b;
  }
  __syncthreads();
  if (threadIdx.x < G) {
    float a = 0.f, b = 0.f;
    for (int c = threadIdx.x * cpg; c < (threadIdx.x + 1) * cpg; ++c) { a += s_sum[c]; b += s_sq[c]; }
    partial[(static_cast<long long>(nb) * gridDim.x + blockIdx.x) * G + threadIdx.x] = make_float2(a, b);
    __threadfence();
  }
  __shared__ bool s_last;
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(&counters[nb], 1u) == gridDim.x - 1u;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (threadIdx.x < G) {
    double a = 0.0, b = 0.0;
    const float2* pp = partial + static_cast<long long>(nb) * gridDim.x * G + threadIdx.x;
    for (unsigned i = 0; i < gridDim.x; ++i) {
      const float2 v = __ldcg(pp + static_cast<size_t>(i) * G);
      a += v.x;
      b += v.y;
    }
    image_sums[nb * G + threadIdx.x] = make_float2(static_cast<float>(a), static_cast<float>(b));
  }
  if (threadIdx.x == 0) counters[nb] = 0;  // ready for the next call (stream order)
}

template <int SLOTS>
__global__ void __launch_bounds__(kGnThreads) gn_apply_kernel(const __half* __restrict__ x, __half* __restrict__ y, int HW, int C, int G,
                                                             int frames_per_stat, int count_frames, int TX, int px_per_cta,
                                                             const float2* __restrict__ image_sums, const double2* __restrict__ image_sums64,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                                             int silu) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float s_mean[64], s_rstd[64];
  const int nb = blockIdx.y;
  const int cpg = C / G;
  if (threadIdx.x < G) {
    const int first = (nb / frames_per_stat) * frames_per_stat;
    double sa = 0.0, sb = 0.0;
    for (int i = 0; i < frames_per_stat; ++i) {
      if (image_sums64) {  // fz_groupnorm_apply_sums64_f16: fp64 sums (the set totals of the frame-sharded exchange)
        const double2 v = image_sums64[(first + i) * G + threadIdx.x];
        sa += v.x;
        sb += v.y;
      } else {
        const float2 v = image_sums[(first + i) * G + threadIdx.x];
        sa += v.x;
        sb += v.y;
      }
    }
    const double cnt = static_cast<double>(cpg) * HW * count_frames;  // count_frames > frames_per_stat: frames held by other GPUs
    const double mean = sa / cnt;
    double var = sb / cnt - mean * mean;
    if (var < 0) var = 0;
    s_mean[threadIdx.x] = static_cast<float>(mean);
    s_rstd[threadIdx.x] = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
  }
  __syncthreads();
  const int tx = threadIdx.x % TX, ty = threadIdx.x / TX;
  const int TY = kGnThreads / TX;
  if (ty >= TY) return;
  // y = (x - mean) * (rstd * gamma) + beta: centring first keeps a (near-)constant group exact; a fused shift beta - mean * rstd * gamma
  // would carry a rounding error of 2^-24 |mean| rstd |gamma| into every output
  float sc[SLOTS][8], mn[SLOTS][8], sh[SLOTS][8];
#pragma unroll
  for (int s = 0; s < SLOTS; ++s) {
    const int cv = tx + s * TX;
    const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + cv * 8)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + cv * 8 + 4));
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + cv * 8)), b1 = __ldg(reinterpret_cast<const float4*>(beta + cv * 8 + 4));
    const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
    const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int g = (cv * 8 + e) / cpg;
      sc[s][e] = s_rstd[g] * gg[e];
      mn[s][e] = s_mean[g];
      sh[s][e] = bb[e];
    }
  }
  const int p0 = blockIdx.x * px_per_cta;
  const int p1 = min(HW, p0 + px_per_cta);
  const long long base = (static_cast<long long>(nb) * HW) * C;
  constexpr int U = (SLOTS == 1) ? 4 : (SLOTS == 2 ? 2 : 1);
  for (int p = p0 + ty; p < p1; p += TY * U) {
    Half8 h[U][SLOTS];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int pp = p + u * TY;
      if (pp < p1) {
#pragma unroll
        for (int s = 0; s < SLOTS; ++s) h[u][s] = *reinterpret_cast<const Half8*>(x + base + static_cast<long long>(pp) * C + (tx + s * TX) * 8);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int pp = p + u * TY;
      if (pp < p1) {
#pragma unroll
        for (int s = 0; s < SLOTS; ++s) {
          Half8 o;
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            float v = fmaf(__half2float(h[u][s].v[e]) - mn[s][e], sc[s][e], sh[s][e]);
            if (silu) v = __fdividef(v, 1.0f + __expf(-v));  // fast reciprocal: the IEEE division made this kernel MUFU/issue-bound
            o.v[e] = __float2half_rn(v);
          }
          *reinterpret_cast<Half8*>(y + base + static_cast<long long>(pp) * C + (tx + s * TX) * 8) = o;
        }
      }
    }
  }
}

// TX * slots == C / 8 exactly, slots in {1, 2, 4}; px_per_cta so that the whole tensor is covered by about `ctas_per_sm` CTAs per SM.
static void gn_geometry(int C, int HW, int NB, int ctas_per_sm, int* TX, int* slots, int* px_per_cta, int* chunks) {
  const int CV = C / 8;
  int s = (CV + kGnThreads - 1) / kGnThreads;
  while (CV % s || s == 3) ++s;
  *slots = s;
  *TX = CV / s;
  const int TY = kGnThreads / *TX;
  const int want = std::max(1, (ctas_per_sm * sm_count()) / std::max(1, NB));
  const int ppc = std::max(TY, (HW + want - 1) / want);
  *px_per_cta = ppc;
  *chunks = (HW + ppc - 1) / ppc;
}

// ---------------------------------------------------------------------------------------------------------------
// LayerNorm over the channel axis of token rows (models/attention.py:281,303,320,331), one warp per row.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kLnMaxVec = 8;  // C <= 8*32*8 = 2048

// NV = 16-byte vectors per lane (ceil(C/256)), ROWS = rows per warp in flight (memory-level parallelism); both compile-time so the
// row buffer stays in registers and occupancy follows the real channel count.
template <int NV, int ROWS>
__global__ void __launch_bounds__(256) layernorm_kernel(const __half* __restrict__ x, __half* __restrict__ y, long long M, int C,
                                                       const float* __restrict__ gamma, const float* __restrict__ beta, float eps) {
  const int lane = threadIdx.x & 31;
  pdl_launch_dependents();
  pdl_wait();
  const long long row0 = (static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5)) * ROWS;
  if (row0 >= M) return;
  const int CV = C / 8;
  // the rows are converted to fp32 ONCE and stay in registers for the mean, the centred second moment and the output
  // (the kernel was issue-bound: 65 % issue slots busy, three half->float conversions per element)
  Half8 raw[ROWS][NV];
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
    const long long row = min(row0 + r, M - 1);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int cv = lane + i * 32;
      if (cv < CV) raw[r][i] = *reinterpret_cast<const Half8*>(x + row * C + cv * 8);
    }
  }
  float v[ROWS][NV][8];
  float sum[ROWS], mean[ROWS], sq[ROWS];
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
    sum[r] = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const bool ok = lane + i * 32 < CV;
      const __half2* h2 = reinterpret_cast<const __half2*>(&raw[r][i]);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = ok ? __half22float2(h2[e]) : make_float2(0.f, 0.f);
        v[r][i][2 * e] = f.x;
        v[r][i][2 * e + 1] = f.y;
        sum[r] += f.x + f.y;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], o);
  }
  const float inv_c = 1.0f / C;
  // the mean sum / C, rounded as a division rounds it (one fma correction of sum * (1/C); a division's slow path would cost this kernel a
  // stack frame): exact for a constant row, whose sum of fp16 values is exact in fp32
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
    const float q = sum[r] * inv_c;
    mean[r] = fmaf(fmaf(-q, static_cast<float>(C), sum[r]), inv_c, q);
  }
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
    sq[r] = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      if (lane + i * 32 < CV) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float d = v[r][i][e] - mean[r];
          sq[r] = fmaf(d, d, sq[r]);
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sq[r] += __shfl_xor_sync(0xffffffffu, sq[r], o);
  }
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int cv = lane + i * 32;
    if (cv < CV) {
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + cv * 8)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + cv * 8 + 4));
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + cv * 8)), b1 = __ldg(reinterpret_cast<const float4*>(beta + cv * 8 + 4));
      const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int r = 0; r < ROWS; ++r) {
        const long long row = row0 + r;
        if (row < M) {
          const float rstd = rsqrtf(sq[r] * inv_c + eps);
          // from the centred value: a fused x * rstd + (-mean * rstd) rounds the shift, an absolute error of 2^-24 |mean| rstd that
          // swamps beta on a (near-)constant row, where rstd approaches eps^-1/2
          Half8 o;
          __half2* o2 = reinterpret_cast<__half2*>(&o);
#pragma unroll
          for (int e = 0; e < 4; ++e)
            o2[e] = __floats2half2_rn(fmaf((v[r][i][2 * e] - mean[r]) * rstd, gg[2 * e], bb[2 * e]),
                                      fmaf((v[r][i][2 * e + 1] - mean[r]) * rstd, gg[2 * e + 1], bb[2 * e + 1]));
          *reinterpret_cast<Half8*>(y + row * C + cv * 8) = o;
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// nearest 2x upsample (resnet.py:145) and channel concat (unet_3d_blocks.py:522,611), NHWC
// ---------------------------------------------------------------------------------------------------------------
__global__ void upsample2x_kernel(const Half8* __restrict__ x, Half8* __restrict__ y, int NB, int H, int W, int CV) {
  pdl_launch_dependents();
  pdl_wait();
  const long long total = static_cast<long long>(NB) * (2 * H) * (2 * W) * CV;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cv = i % CV;
    long long r = i / CV;
    const int ox = r % (2 * W);
    r /= (2 * W);
    const int oy = r % (2 * H);
    const int nb = r / (2 * H);
    y[i] = x[((static_cast<long long>(nb) * H + oy / 2) * W + ox / 2) * CV + cv];
  }
}

__global__ void concat2_kernel(const Half8* __restrict__ a, int CVa, const Half8* __restrict__ b, int CVb, Half8* __restrict__ y, long long rows) {
  pdl_launch_dependents();
  pdl_wait();
  const int CV = CVa + CVb;
  const long long total = rows * CV;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cv = i % CV;
    const long long r = i / CV;
    y[i] = (cv < CVa) ? a[r * CVa + cv] : b[r * CVb + (cv - CVa)];
  }
}

// ---------------------------------------------------------------------------------------------------------------
// UNet input: latents [B, Cl, F, H, W] fp32 -> im2col rows [B*F*H*W, 64] fp16 (col = tap*Cl + c, tap = ky*3+kx, zero padded)
// so conv_in (unet_3d_condition.py:375) runs as a K=64 GEMM.
// ---------------------------------------------------------------------------------------------------------------
__global__ void im2col_in_kernel(const float* __restrict__ x, __half* __restrict__ out, int B, int Cl, int F, int H, int W) {
  const long long rows = static_cast<long long>(B) * F * H * W;
  const long long total = rows * 8;  // 8 vectors of 8 halfs per row
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int v = i % 8;
    long long r = i / 8;
    const int xx = r % W;
    long long t = r / W;
    const int yy = t % H;
    t /= H;
    const int f = t % F;
    const int b = t / F;
    Half8 o;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int col = v * 8 + e;
      float val = 0.f;
      if (col < 9 * Cl) {
        const int tap = col / Cl, c = col % Cl;
        const int sy = yy + tap / 3 - 1, sx = xx + tap % 3 - 1;
        if (sy >= 0 && sy < H && sx >= 0 && sx < W) val = x[(((static_cast<long long>(b) * Cl + c) * F + f) * H + sy) * W + sx];
      }
      o.v[e] = __float2half_rn(val);
    }
    *reinterpret_cast<Half8*>(out + r * 64 + v * 8) = o;
  }
}

// conv_out tail: y [B*F*HW, ldy] fp16 (Co valid channels, conv bias already added) -> temporal conv over frames
//   lora : out = y + up(down(y))   (down [R, Co, 3], up [Co, R, 3], lora.py:46-54)       (w_full == null)
//   full : out = bias + W * y      (W [Co, Co, 3], resnet.py:42-55)                        (w_full != null)
// and scatter to eps [B, Co, F, H, W] fp32 (the layout the DDIM step consumes).
__global__ void out_temporal_kernel(const __half* __restrict__ y, int ldy, float* __restrict__ eps, int B, int Co, int F, int HW,
                                    const float* __restrict__ down, const float* __restrict__ up, int R, const float* __restrict__ w_full,
                                    const float* __restrict__ b_full) {
  const long long total = static_cast<long long>(B) * F * HW;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int p = i % HW;
    const int f = (i / HW) % F;
    const int b = i / (static_cast<long long>(HW) * F);
    auto ld = [&](int ff, int c) -> float {
      if (ff < 0 || ff >= F) return 0.f;
      return __half2float(y[((static_cast<long long>(b) * F + ff) * HW + p) * ldy + c]);
    };
    float outv[8];
    if (w_full) {
      for (int c = 0; c < Co; ++c) {
        float a = b_full ? b_full[c] : 0.f;
        for (int ci = 0; ci < Co; ++ci)
          for (int t = 0; t < 3; ++t) a += w_full[(c * Co + ci) * 3 + t] * ld(f + t - 1, ci);
        outv[c] = a;
      }
    } else if (down) {
      // mid[r][g] for frames g = f-1, f, f+1 (zero outside), as the fp16-rounded intermediate of the reference autocast path
      float mid[4][3];
      for (int r = 0; r < R; ++r)
        for (int dg = 0; dg < 3; ++dg) {
          const int g = f + dg - 1;
          float a = 0.f;
          if (g >= 0 && g < F)
            for (int ci = 0; ci < Co; ++ci)
              for (int t = 0; t < 3; ++t) a += down[(r * Co + ci) * 3 + t] * ld(g + t - 1, ci);
          mid[r][dg] = (g >= 0 && g < F) ? __half2float(__float2half_rn(a)) : 0.f;
        }
      for (int c = 0; c < Co; ++c) {
        float a = ld(f, c);
        for (int r = 0; r < R; ++r)
          for (int t = 0; t < 3; ++t) a += up[(c * R + r) * 3 + t] * mid[r][t];
        outv[c] = a;
      }
    } else {
      for (int c = 0; c < Co; ++c) outv[c] = ld(f, c);
    }
    for (int c = 0; c < Co; ++c) eps[((static_cast<long long>(b) * Co + c) * F + f) * HW + p] = outv[c];
  }
}

// ---------------------------------------------------------------------------------------------------------------
// small dense layers on a single row (time embedding path, unet_3d_condition.py:356-362; resnet.py:355):
//   y[n] = bias[n] + sum_k act(x[k]) * W[n,k]     act = identity | SiLU ;  one warp per output
// ---------------------------------------------------------------------------------------------------------------
__global__ void rowvec_linear_kernel(const float* __restrict__ x, const __half* __restrict__ W, const float* __restrict__ bias,
                                     float* __restrict__ y, int N, int K, int silu_in) {
  const int lane = threadIdx.x & 31;
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= N) return;
  float a = 0.f;
  for (int k = lane * 2; k < K; k += 64) {
    float x0 = x[k], x1 = (k + 1 < K) ? x[k + 1] : 0.f;
    if (silu_in) { x0 = x0 / (1.f + __expf(-x0)); x1 = x1 / (1.f + __expf(-x1)); }
    const __half2 w = *reinterpret_cast<const __half2*>(W + static_cast<long long>(n) * K + k);
    a += x0 * __low2float(w) + x1 * __high2float(w);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if (lane == 0) y[n] = a + (bias ? bias[n] : 0.f);
}

// Timesteps(C0, flip_sin_to_cos, freq_shift) — diffusers embeddings.get_timestep_embedding
__global__ void timestep_sinusoid_kernel(float t, float* __restrict__ out, int C0, int flip, float freq_shift) {
  const int half = C0 / 2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= half) return;
  const float e = expf(-logf(10000.f) * static_cast<float>(i) / (static_cast<float>(half) - freq_shift));
  const float a = t * e;
  const float s = sinf(a), c = cosf(a);
  if (flip) { out[i] = c; out[half + i] = s; }
  else { out[i] = s; out[half + i] = c; }
}

// ---------------------------------------------------------------------------------------------------------------
// temporal attention over the frame axis (models/attention.py:327-337): qkv [B*F*HW, 3C] fp16 -> out [B*F*HW, C] fp16
// one warp per (b, pixel, head); probabilities are rounded to fp16 before PV like the reference's `.to(value.dtype)`.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kTaMaxF = 32;
__global__ void __launch_bounds__(256) temporal_attn_kernel(const __half* __restrict__ qkv, __half* __restrict__ out, int B, int F, int HW,
                                                           int heads, int d, float scale) {
  extern __shared__ __half ta_smem[];
  pdl_launch_dependents();
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const int C = heads * d;
  __half* sq = ta_smem + static_cast<size_t>(warp) * (3 * F * d + F * F * 2);
  __half* sk = sq + F * d;
  __half* sv = sk + F * d;
  float* sp = reinterpret_cast<float*>(sv + F * d);
  const long long items = static_cast<long long>(B) * HW * heads;
  for (long long it = static_cast<long long>(blockIdx.x) * wpb + warp; it < items; it += static_cast<long long>(gridDim.x) * wpb) {
    const int h = it % heads;
    const int p = (it / heads) % HW;
    const int b = it / (static_cast<long long>(heads) * HW);
    const int d2 = d / 2;
    for (int i = lane; i < F * d2; i += 32) {
      const int f = i / d2, j = i % d2;
      const long long row = (static_cast<long long>(b) * F + f) * HW + p;
      const __half2* src = reinterpret_cast<const __half2*>(qkv + row * 3 * C + h * d) + j;
      reinterpret_cast<__half2*>(sq)[i] = src[0];
      reinterpret_cast<__half2*>(sk)[i] = src[C / 2];
      reinterpret_cast<__half2*>(sv)[i] = src[C];
    }
    __syncwarp();
    for (int i = lane; i < F * F; i += 32) {
      const int f = i / F, g = i % F;
      float a = 0.f;
      for (int j = 0; j < d2; ++j) {
        const float2 qa = __half22float2(reinterpret_cast<const __half2*>(sq)[f * d2 + j]);
        const float2 ka = __half22float2(reinterpret_cast<const __half2*>(sk)[g * d2 + j]);
        a += qa.x * ka.x + qa.y * ka.y;
      }
      sp[i] = a * scale;
    }
    __syncwarp();
    if (lane < F) {
      float mx = -INFINITY;
      for (int g = 0; g < F; ++g) mx = fmaxf(mx, sp[lane * F + g]);
      float sum = 0.f;
      for (int g = 0; g < F; ++g) { const float e = __expf(sp[lane * F + g] - mx); sp[lane * F + g] = e; sum += e; }
      const float inv = 1.f / sum;
      for (int g = 0; g < F; ++g) sp[lane * F + g] = __half2float(__float2half_rn(sp[lane * F + g] * inv));
    }
    __syncwarp();
    for (int i = lane; i < F * d; i += 32) {
      const int f = i / d, dd = i % d;
      float a = 0.f;
      for (int g = 0; g < F; ++g) a += sp[f * F + g] * __half2float(sv[g * d + dd]);
      const long long row = (static_cast<long long>(b) * F + f) * HW + p;
      out[row * C + h * d + dd] = __float2half_rn(a);
    }
    __syncwarp();
  }
}

// Pixel-major variant (the one the step uses: F <= 8): one warp owns (pixel, head group) with all F frames, where a head group is
// hg consecutive heads (hg * d = 320 channels for the SD head sizes 40 / 80 / 160, so the warp's working set is always 15 KB).
// The F q|k|v segments (3 x 640 contiguous bytes per frame) are fetched with coalesced 16-byte loads into shared memory (row
// stride 3*gd + 8 halves, so the 8 lanes of a quarter-warp, one frame each, hit 8 distinct 16-byte bank groups); lane r handles the
// query rows (head, frame) = (r / F, r % F), r + 32, ...: scores against the F keys of its head (shared-memory broadcast reads),
// fp32 softmax, probabilities rounded to fp16 like the reference, PV, and the result replaces its own q slice; the warp then writes
// the F output segments with coalesced 16-byte stores.  v1 (warp per (pixel, head), 4-byte loads, 80-byte segments) ran at 0.9 TB/s.
template <int F>
__global__ void __launch_bounds__(256) temporal_attn_px_kernel(const __half* __restrict__ qkv, __half* __restrict__ out, int B, int HW, int heads,
                                                              int d, int hg, float scale) {
  extern __shared__ uint4 tap_smem[];
  pdl_launch_dependents();
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const int C = heads * d;
  const int gd = hg * d;          // channels of one head group
  const int gv = gd / 8;          // 16-byte vectors per q / k / v segment
  const int RS8 = 3 * gv + 1;     // shared-memory row stride in 16-byte units
  const int groups = heads / hg;
  uint4* sm = tap_smem + static_cast<size_t>(warp) * F * RS8;
  const int rows = hg * F;
  const long long items = static_cast<long long>(B) * HW * groups;
  for (long long it = static_cast<long long>(blockIdx.x) * wpb + warp; it < items; it += static_cast<long long>(gridDim.x) * wpb) {
    const int grp = it % groups;
    const int p = (it / groups) % HW;
    const int b = it / (static_cast<long long>(groups) * HW);
    // ---- gather: F rows x 3 segments x gv vectors, 8 loads in flight per lane ----
    const int total = F * 3 * gv;
    for (int base = 0; base < total; base += 8 * 32) {
      uint4 v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int idx = base + u * 32 + lane;
        if (idx < total) {
          const int f = idx / (3 * gv), c = idx - f * 3 * gv, part = c / gv, cc = c - part * gv;
          v[u] = __ldg(reinterpret_cast<const uint4*>(qkv + ((static_cast<long long>(b) * F + f) * HW + p) * 3 * C + part * C + grp * gd) + cc);
        }
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int idx = base + u * 32 + lane;
        if (idx < total) {
          const int f = idx / (3 * gv), c = idx - f * 3 * gv;
          sm[f * RS8 + c] = v[u];
        }
      }
    }
    __syncwarp();
    // ---- per query row ----
    for (int r = lane; r < rows; r += 32) {
      const int h = r / F, f = r - h * F;
      const uint4* qp = sm + f * RS8 + (h * d) / 8;
      float sc[F];
#pragma unroll
      for (int g = 0; g < F; ++g) sc[g] = 0.f;
      for (int j = 0; j < d / 8; ++j) {
        const uint4 q8 = qp[j];
        const __half2* qh = reinterpret_cast<const __half2*>(&q8);
        const float2 q0 = __half22float2(qh[0]), q1 = __half22float2(qh[1]), q2 = __half22float2(qh[2]), q3 = __half22float2(qh[3]);
#pragma unroll
        for (int g = 0; g < F; ++g) {
          const uint4 k8 = sm[g * RS8 + gv + (h * d) / 8 + j];
          const __half2* kh = reinterpret_cast<const __half2*>(&k8);
          const float2 k0 = __half22float2(kh[0]), k1 = __half22float2(kh[1]), k2 = __half22float2(kh[2]), k3 = __half22float2(kh[3]);
          sc[g] += q0.x * k0.x + q0.y * k0.y + q1.x * k1.x + q1.y * k1.y + q2.x * k2.x + q2.y * k2.y + q3.x * k3.x + q3.y * k3.y;
        }
      }
      float mx = -INFINITY;
#pragma unroll
      for (int g = 0; g < F; ++g) { sc[g] *= scale; mx = fmaxf(mx, sc[g]); }
      float sum = 0.f;
#pragma unroll
      for (int g = 0; g < F; ++g) { sc[g] = __expf(sc[g] - mx); sum += sc[g]; }
      const float inv = 1.f / sum;
#pragma unroll
      for (int g = 0; g < F; ++g) sc[g] = __half2float(__float2half_rn(sc[g] * inv));
      uint4* op = sm + f * RS8 + (h * d) / 8;  // own q slice: nobody else reads it
      for (int j = 0; j < d / 8; ++j) {
        float o[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int g = 0; g < F; ++g) {
          const uint4 v8 = sm[g * RS8 + 2 * gv + (h * d) / 8 + j];
          const __half2* vh = reinterpret_cast<const __half2*>(&v8);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float2 vv = __half22float2(vh[e]);
            o[2 * e] = fmaf(sc[g], vv.x, o[2 * e]);
            o[2 * e + 1] = fmaf(sc[g], vv.y, o[2 * e + 1]);
          }
        }
        uint4 w;
        __half2* wh = reinterpret_cast<__half2*>(&w);
#pragma unroll
        for (int e = 0; e < 4; ++e) wh[e] = __floats2half2_rn(o[2 * e], o[2 * e + 1]);
        op[j] = w;
      }
    }
    __syncwarp();
    // ---- scatter: F rows x gv vectors ----
    for (int idx = lane; idx < F * gv; idx += 32) {
      const int f = idx / gv, c = idx - f * gv;
      reinterpret_cast<uint4*>(out + ((static_cast<long long>(b) * F + f) * HW + p) * C + grp * gd)[c] = sm[f * RS8 + c];
    }
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------------------------------
// DDIM steps on fp32 latents [*, 4, F, H, W] (p2p_ddim_spatial_temporal.py:150-161 and :400-407 + diffusers DDIMScheduler.step
// eta=0) with the latent blend of spatial_blend.py:116-122 fused in.
// ---------------------------------------------------------------------------------------------------------------
__global__ void ddim_invert_kernel(float* __restrict__ x, const float* __restrict__ eps, long long n, float sqrt_a_prev, float sqrt_1m_a_prev,
                                   float sqrt_a_next, float sqrt_1m_a_next) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float e = eps[i];
    const float x0 = (x[i] - sqrt_1m_a_prev * e) / sqrt_a_prev;
    x[i] = sqrt_a_next * x0 + sqrt_1m_a_next * e;
  }
}

// K items of n_item elements: x [K, n_item], eps2 = [uncond_1..K | cond_1..K]. mask (optional, per item): [F*H*W] floats per frame pixel,
// broadcast over channels; x_inv (per item, [n_item]): the inverted latent the item blends towards (items of one clip share it).
constexpr int kCfgMaxItems = 8;
struct CfgItems {
  const float* x_inv[kCfgMaxItems];
  const float* mask_a[kCfgMaxItems];
  const float* mask_b[kCfgMaxItems];
  int apply_blend[kCfgMaxItems];
};

__global__ void cfg_ddim_kernel(float* __restrict__ x, const float* __restrict__ eps2, int K, long long n_item, float guidance, float sqrt_a_t,
                                float sqrt_1m_a_t, float sqrt_a_prev, float sqrt_1m_a_prev, const __grid_constant__ CfgItems items,
                                long long fhw) {
  const long long n = static_cast<long long>(K) * n_item;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float eu = eps2[i], ec = eps2[n + i];
    const float e = eu + guidance * (ec - eu);
    const float x0 = (x[i] - sqrt_1m_a_t * e) / sqrt_a_t;
    float xn = sqrt_a_prev * x0 + sqrt_1m_a_prev * e;
    const int k = K == 1 ? 0 : static_cast<int>(i / n_item);
    if (items.apply_blend[k]) {
      const long long j = i - k * n_item;
      const long long q = j % fhw;
      float m = items.mask_a[k][q];
      if (items.mask_b[k]) m = fmaxf(m, items.mask_b[k][q]);
      const float xi = items.x_inv[k][j];
      xn = xi + m * (xn - xi);
    }
    x[i] = xn;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Blend mask (spatial_blend.py:24-39, 78-111): mean over (layers, heads) of sum_n map[f,hd,p,n]*w[n] on the r x r grid,
// 3x3 max-pool (stride 1, pad 1), nearest resize to (h, w), divide by the per-frame max, compare with th.
// maps: up to 8 pointers to [F, heads, r*r, ldm] fp16 (or fp32 running sums when maps_f32 != 0). One CTA per frame.
// ---------------------------------------------------------------------------------------------------------------
struct MaskParams {
  const void* maps[8];
  int num_maps;
  int maps_f32;
  int F, heads, r, ldm, ntok;
  float w[80];
  float th;
  int h, w_out;
  float* out;  // [F, h, w] 0/1
};

__global__ void __launch_bounds__(256) blend_mask_kernel(const __grid_constant__ MaskParams p) {
  extern __shared__ float mk_smem[];
  float* agg = mk_smem;              // [r*r]
  float* pooled = mk_smem + p.r * p.r;  // [r*r]
  __shared__ float s_max;
  const int f = blockIdx.x;
  const int rr = p.r * p.r;
  for (int px = threadIdx.x; px < rr; px += blockDim.x) {
    float a = 0.f;
    for (int l = 0; l < p.num_maps; ++l)
      for (int hd = 0; hd < p.heads; ++hd) {
        const long long off = ((static_cast<long long>(f) * p.heads + hd) * rr + px) * p.ldm;
        float s = 0.f;
        if (p.maps_f32) {
          const float* m = static_cast<const float*>(p.maps[l]) + off;
          for (int n = 0; n < p.ntok; ++n) s += m[n] * p.w[n];
        } else {
          const __half* m = static_cast<const __half*>(p.maps[l]) + off;
          for (int n = 0; n < p.ntok; ++n) s += __half2float(m[n]) * p.w[n];
        }
        a += s;
      }
    agg[px] = a / static_cast<float>(p.num_maps * p.heads);
  }
  if (threadIdx.x == 0) s_max = 0.f;
  __syncthreads();
  for (int px = threadIdx.x; px < rr; px += blockDim.x) {
    const int y = px / p.r, x = px % p.r;
    float m = -INFINITY;
    for (int dy = -1; dy <= 1; ++dy)
      for (int dx = -1; dx <= 1; ++dx) {
        const int yy = y + dy, xx = x + dx;
        if (yy >= 0 && yy < p.r && xx >= 0 && xx < p.r) m = fmaxf(m, agg[yy * p.r + xx]);
      }
    pooled[px] = m;
  }
  __syncthreads();
  // F.interpolate(mode="nearest") source index: min(floor(dst * (float)in / out), in - 1) in fp32 (the exact integer quotient
  // (dst * in) / out differs for some sizes, e.g. in = 16, out = 82)
  const float sy_scale = static_cast<float>(p.r) / p.h, sx_scale = static_cast<float>(p.r) / p.w_out;
  // max over the RESIZED grid == max over the source pixels that the nearest resize actually samples
  float lm = 0.f;
  for (int i = threadIdx.x; i < p.h * p.w_out; i += blockDim.x) {
    const int y = i / p.w_out, x = i % p.w_out;
    const int sy = min(p.r - 1, static_cast<int>(floorf(y * sy_scale))), sx = min(p.r - 1, static_cast<int>(floorf(x * sx_scale)));
    lm = fmaxf(lm, pooled[sy * p.r + sx]);
  }
  atomicMax(reinterpret_cast<int*>(&s_max), __float_as_int(fmaxf(lm, 0.f)));
  __syncthreads();
  const float mx = s_max;
  for (int i = threadIdx.x; i < p.h * p.w_out; i += blockDim.x) {
    const int y = i / p.w_out, x = i % p.w_out;
    const int sy = min(p.r - 1, static_cast<int>(floorf(y * sy_scale))), sx = min(p.r - 1, static_cast<int>(floorf(x * sx_scale)));
    const float v = pooled[sy * p.r + sx];
    // reference: (v / mx) > th, with 0/0 = NaN -> False
    p.out[(static_cast<long long>(f) * p.h + y) * p.w_out + x] = (mx > 0.f && (v / mx) > p.th) ? 1.f : 0.f;
  }
}

static inline int grid_for(long long total, int threads) {
  long long g = (total + threads - 1) / threads;
  const long long cap = static_cast<long long>(sm_count()) * 16;
  return static_cast<int>(std::max<long long>(1, std::min(g, cap)));
}

}  // namespace fz

using namespace fz;

// which = 1: statistics only, 2: apply only (image_sums supplied by the caller: float2, or double2 when sums_f64), 3: both
// geometry_images: the number of images the chunking is planned for (NB, or the images of one item of a batched edit)
static int groupnorm_impl(int which, const void* x, void* y, int NB, int HW, int C, int groups, int frames_per_stat, int count_frames,
                          const float* gamma, const float* beta, float eps, int silu, void* workspace_f64, const void* sums_in,
                          cudaStream_t stream, int geometry_images, bool sums_f64 = false) {
  if (int rc = check_single_device()) return rc;
  FZ_CHECK_ARG(C % 8 == 0 && C % groups == 0 && groups <= 64, "fz_groupnorm: C=%d groups=%d unsupported", C, groups);
  FZ_CHECK_ARG(frames_per_stat >= 1 && NB % frames_per_stat == 0, "fz_groupnorm: NB %% frames_per_stat != 0");
  int TX, slots, ppc, chunks, ppc_apply, chunks_apply;
  gn_geometry(C, HW, geometry_images, 2, &TX, &slots, &ppc, &chunks);              // statistics: few fat CTAs (amortise the reduction tail)
  gn_geometry(C, HW, geometry_images, 4, &TX, &slots, &ppc_apply, &chunks_apply);  // apply: one full wave of 4 CTAs per SM
  FZ_CHECK_ARG(slots <= kGnMaxSlots, "fz_groupnorm: C=%d too large", C);
  FZ_CHECK_ARG(static_cast<size_t>(NB) * chunks * groups * sizeof(float2) <= kGnStatsOffset && NB <= 256, "fz_groupnorm: workspace (1 MiB) too small");
  const int TY = kGnThreads / TX;
  const size_t smem = static_cast<size_t>(2) * TY * C * sizeof(float);
  static size_t configured = 0;
  if (smem > 48 * 1024 && smem > configured) {
    FZ_CUDA(cudaFuncSetAttribute(gn_stats_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    FZ_CUDA(cudaFuncSetAttribute(gn_stats_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    FZ_CUDA(cudaFuncSetAttribute(gn_stats_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    configured = smem;
  }
  float2* partial = static_cast<float2*>(workspace_f64);
  float2* image_sums = workspace_f64 ? reinterpret_cast<float2*>(static_cast<uint8_t*>(workspace_f64) + kGnStatsOffset) : nullptr;
  unsigned* counters = workspace_f64 ? reinterpret_cast<unsigned*>(static_cast<uint8_t*>(workspace_f64) + kGnCounterOffset) : nullptr;
  const float2* sums = sums_in && !sums_f64 ? static_cast<const float2*>(sums_in) : image_sums;
  const double2* sums64 = sums_f64 ? static_cast<const double2*>(sums_in) : nullptr;
  const __half* xh = static_cast<const __half*>(x);
  __half* yh = static_cast<__half*>(y);
#define FZ_GN_LAUNCH(SL)                                                                                                             \
  do {                                                                                                                                \
    if (which & 1)                                                                                                                    \
      FZ_CUDA(launch_pdl(gn_stats_kernel<SL>, dim3(chunks, NB), dim3(kGnThreads), smem, stream, xh, HW, C, groups, TX, ppc, partial,    \
                         image_sums, counters));                                                                                     \
    if (which & 2)                                                                                                                    \
      FZ_CUDA(launch_pdl(gn_apply_kernel<SL>, dim3(chunks_apply, NB), dim3(kGnThreads), 0, stream, xh, yh, HW, C, groups,               \
                         frames_per_stat, count_frames, TX, ppc_apply, sums, sums64, gamma, beta, eps, silu));                      \
  } while (0)
  if (slots == 1) FZ_GN_LAUNCH(1);
  else if (slots == 2) FZ_GN_LAUNCH(2);
  else FZ_GN_LAUNCH(4);
#undef FZ_GN_LAUNCH
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}

extern "C" int fz_groupnorm_nhwc_f16(const void* x, void* y, int NB, int HW, int C, int groups, int frames_per_stat, const float* gamma,
                                     const float* beta, float eps, int silu, void* workspace_f64, cudaStream_t stream) {
  FZ_CHECK_ARG(x && y && gamma && beta && workspace_f64, "fz_groupnorm: null pointer");
  return groupnorm_impl(3, x, y, NB, HW, C, groups, frames_per_stat, frames_per_stat, gamma, beta, eps, silu, workspace_f64, nullptr, stream,
                        NB);
}

extern "C" int fz_groupnorm_batched_nhwc_f16(const void* x, void* y, int NB, int HW, int C, int groups, int frames_per_stat,
                                             int images_per_item, const float* gamma, const float* beta, float eps, int silu,
                                             void* workspace_f64, cudaStream_t stream) {
  FZ_CHECK_ARG(x && y && gamma && beta && workspace_f64, "fz_groupnorm: null pointer");
  FZ_CHECK_ARG(images_per_item >= 1 && NB % images_per_item == 0 && images_per_item % frames_per_stat == 0,
               "fz_groupnorm_batched: images_per_item=%d must divide NB=%d and be a multiple of frames_per_stat=%d", images_per_item, NB,
               frames_per_stat);
  return groupnorm_impl(3, x, y, NB, HW, C, groups, frames_per_stat, frames_per_stat, gamma, beta, eps, silu, workspace_f64, nullptr, stream,
                        images_per_item);
}

// Frame-sharded GroupNorm (SURVEY.md 8(e)): statistics and apply as separate calls so that the (sum, sumsq) of the frames held by other
// GPUs can be all-reduced in between.  fz_groupnorm_stats_f16 leaves float2 sums[NB][groups] at workspace + 768 KiB; the apply reads
// float2 sums (fz_groupnorm_apply_f16) or double2 sums (fz_groupnorm_apply_sums64_f16: fz_gn_combine's fp64 set totals).
extern "C" int fz_groupnorm_stats_f16(const void* x, int NB, int HW, int C, int groups, void* workspace_f64, cudaStream_t stream) {
  FZ_CHECK_ARG(x && workspace_f64, "fz_groupnorm_stats: null pointer");
  return groupnorm_impl(1, x, nullptr, NB, HW, C, groups, 1, 1, nullptr, nullptr, 0.f, 0, workspace_f64, nullptr, stream, NB);
}

extern "C" int fz_groupnorm_apply_f16(const void* x, void* y, int NB, int HW, int C, int groups, int frames_per_stat, int count_frames,
                                      const float* gamma, const float* beta, float eps, int silu, const void* image_sums,
                                      cudaStream_t stream) {
  FZ_CHECK_ARG(x && y && gamma && beta && image_sums && count_frames >= frames_per_stat, "fz_groupnorm_apply: bad arguments");
  return groupnorm_impl(2, x, y, NB, HW, C, groups, frames_per_stat, count_frames, gamma, beta, eps, silu, nullptr, image_sums, stream, NB);
}

extern "C" int fz_groupnorm_apply_sums64_f16(const void* x, void* y, int NB, int HW, int C, int groups, int frames_per_stat, int count_frames,
                                             const float* gamma, const float* beta, float eps, int silu, const void* image_sums,
                                             cudaStream_t stream) {
  FZ_CHECK_ARG(x && y && gamma && beta && image_sums && count_frames >= frames_per_stat, "fz_groupnorm_apply: bad arguments");
  return groupnorm_impl(2, x, y, NB, HW, C, groups, frames_per_stat, count_frames, gamma, beta, eps, silu, nullptr, image_sums, stream, NB,
                        true);
}

extern "C" int fz_layernorm_f16(const void* x, void* y, long long M, int C, const float* gamma, const float* beta, float eps,
                                cudaStream_t stream) {
  FZ_CHECK_ARG(x && y && gamma && beta, "fz_layernorm: null pointer");
  FZ_CHECK_ARG(C % 8 == 0 && C <= 8 * 32 * kLnMaxVec, "fz_layernorm: C=%d unsupported", C);
  const int nv = (C / 8 + 31) / 32;
  const __half* xh = static_cast<const __half*>(x);
  __half* yh = static_cast<__half*>(y);
#define FZ_LN_LAUNCH(NV, ROWS) \
  FZ_CUDA(launch_pdl(layernorm_kernel<NV, ROWS>, dim3(static_cast<unsigned>((M + 8 * ROWS - 1) / (8 * ROWS))), dim3(256), 0, stream, xh, yh, M, C, \
                     gamma, beta, eps))
  switch (nv) {
    case 1: FZ_LN_LAUNCH(1, 4); break;
    case 2: FZ_LN_LAUNCH(2, 2); break;
    case 3: FZ_LN_LAUNCH(3, 2); break;
    case 4: FZ_LN_LAUNCH(4, 1); break;
    case 5: FZ_LN_LAUNCH(5, 1); break;
    case 6: FZ_LN_LAUNCH(6, 1); break;
    case 7: FZ_LN_LAUNCH(7, 1); break;
    default: FZ_LN_LAUNCH(8, 1); break;
  }
#undef FZ_LN_LAUNCH
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}

extern "C" int fz_upsample2x_nhwc_f16(const void* x, void* y, int NB, int H, int W, int C, cudaStream_t stream) {
  FZ_CHECK_ARG(x && y && C % 8 == 0, "fz_upsample2x: bad args");
  const long long total = static_cast<long long>(NB) * 4 * H * W * (C / 8);
  FZ_CUDA(launch_pdl(upsample2x_kernel, dim3(grid_for(total, 256)), dim3(256), 0, stream, static_cast<const Half8*>(x), static_cast<Half8*>(y), NB, H, W,
                     C / 8));
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}

extern "C" int fz_concat_channels_f16(const void* a, int Ca, const void* b, int Cb, void* y, long long rows, cudaStream_t stream) {
  FZ_CHECK_ARG(a && b && y && Ca % 8 == 0 && Cb % 8 == 0, "fz_concat_channels: bad args");
  const long long total = rows * ((Ca + Cb) / 8);
  FZ_CUDA(launch_pdl(concat2_kernel, dim3(grid_for(total, 256)), dim3(256), 0, stream, static_cast<const Half8*>(a), Ca / 8,
                     static_cast<const Half8*>(b), Cb / 8, static_cast<Half8*>(y), rows));
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}

extern "C" int fz_im2col_latents_f16(const float* x, void* out, int B, int Cl, int F, int H, int W, cudaStream_t stream) {
  FZ_CHECK_ARG(x && out && Cl * 9 <= 64, "fz_im2col_latents: bad args");
  const long long total = static_cast<long long>(B) * F * H * W * 8;
  im2col_in_kernel<<<grid_for(total, 256), 256, 0, stream>>>(x, static_cast<__half*>(out), B, Cl, F, H, W);
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}

extern "C" int fz_out_temporal_f32(const void* y, int ldy, float* eps, int B, int Co, int F, int HW, const float* down, const float* up, int rank,
                                   const float* w_full, const float* b_full, cudaStream_t stream) {
  FZ_CHECK_ARG(y && eps && Co <= 8 && rank <= 4, "fz_out_temporal: bad args");
  const long long total = static_cast<long long>(B) * F * HW;
  out_temporal_kernel<<<grid_for(total, 256), 256, 0, stream>>>(static_cast<const __half*>(y), ldy, eps, B, Co, F, HW, down, up, rank, w_full,
                                                                b_full);
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}

extern "C" int fz_rowvec_linear(const float* x, const void* W_f16, const float* bias, float* y, int N, int K, int silu_in, cudaStream_t stream) {
  FZ_CHECK_ARG(x && W_f16 && y && K % 2 == 0, "fz_rowvec_linear: bad args");
  rowvec_linear_kernel<<<(N + 7) / 8, 256, 0, stream>>>(x, static_cast<const __half*>(W_f16), bias, y, N, K, silu_in);
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}

extern "C" int fz_timestep_sinusoid(float t, float* out, int C0, int flip_sin_to_cos, float freq_shift, cudaStream_t stream) {
  FZ_CHECK_ARG(out && C0 % 2 == 0, "fz_timestep_sinusoid: bad args");
  timestep_sinusoid_kernel<<<(C0 / 2 + 127) / 128, 128, 0, stream>>>(t, out, C0, flip_sin_to_cos, freq_shift);
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}

template <int F>
static int launch_temporal_px(const void* qkv, void* out, int B, int HW, int heads, int d, int hg, float scale, cudaStream_t stream) {
  const int wpb = 4;
  const size_t per_warp = static_cast<size_t>(F) * (3 * hg * d / 8 + 1) * 16;
  const size_t smem = per_warp * wpb;
  static size_t configured = 0;
  if (smem > 48 * 1024 && smem > configured) {
    FZ_CUDA(cudaFuncSetAttribute(temporal_attn_px_kernel<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    configured = smem;
  }
  const int ctas_per_sm = std::max(1, std::min(8, static_cast<int>((220 * 1024) / (smem + 1024))));
  const long long items = static_cast<long long>(B) * HW * (heads / hg);
  const int grid = static_cast<int>(std::min<long long>((items + wpb - 1) / wpb, static_cast<long long>(sm_count()) * ctas_per_sm));
  FZ_CUDA(launch_pdl(temporal_attn_px_kernel<F>, dim3(grid), dim3(wpb * 32), smem, stream, static_cast<const __half*>(qkv), static_cast<__half*>(out), B, HW,
                     heads, d, hg, scale));
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}

extern "C" int fz_temporal_attn_f16(const void* qkv, void* out, int B, int F, int HW, int heads, int d, float scale, cudaStream_t stream) {
  FZ_CHECK_ARG(qkv && out && F >= 1 && F <= kTaMaxF && d % 2 == 0, "fz_temporal_attn: F=%d d=%d unsupported", F, d);
  if (d % 8 == 0 && d <= 320) {
    int hg = std::max(1, std::min(heads, 320 / d));  // heads per warp: 15 KB of q|k|v per (pixel, head group)
    while (heads % hg) --hg;
    switch (F) {
      case 8: return launch_temporal_px<8>(qkv, out, B, HW, heads, d, hg, scale, stream);
      case 4: return launch_temporal_px<4>(qkv, out, B, HW, heads, d, hg, scale, stream);
      case 2: return launch_temporal_px<2>(qkv, out, B, HW, heads, d, hg, scale, stream);
      default: break;
    }
  }
  // up to 8 warps per block, as many as the per-block shared-memory limit holds (a 32-frame clip at d = 160 takes 34 KB per warp)
  constexpr size_t kSmemBudget = 227 * 1024;
  const size_t per_warp = static_cast<size_t>(3 * F * d + F * F * 2) * sizeof(__half);
  FZ_CHECK_ARG(per_warp <= kSmemBudget, "fz_temporal_attn: F=%d d=%d needs %zu B of shared memory per warp", F, d, per_warp);
  const int wpb = static_cast<int>(std::min<size_t>(8, kSmemBudget / per_warp));
  const size_t smem = per_warp * wpb;
  static size_t configured = 0;
  if (smem > 48 * 1024 && smem > configured) {
    FZ_CUDA(cudaFuncSetAttribute(temporal_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    configured = smem;
  }
  const long long items = static_cast<long long>(B) * HW * heads;
  const int grid = static_cast<int>(std::min<long long>((items + wpb - 1) / wpb, static_cast<long long>(sm_count()) * 4));
  FZ_CUDA(launch_pdl(temporal_attn_kernel, dim3(grid), dim3(wpb * 32), smem, stream, static_cast<const __half*>(qkv), static_cast<__half*>(out), B, F, HW,
                     heads, d, scale));
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}

extern "C" int fz_ddim_invert_step(float* x, const float* eps, long long n, float a_prev, float a_next, cudaStream_t stream) {
  FZ_CHECK_ARG(x && eps, "fz_ddim_invert_step: null pointer");
  ddim_invert_kernel<<<grid_for(n, 256), 256, 0, stream>>>(x, eps, n, sqrtf(a_prev), sqrtf(1.f - a_prev), sqrtf(a_next), sqrtf(1.f - a_next));
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}

static int cfg_ddim_launch(float* x, const float* eps2, int K, long long n_item, float guidance, float a_t, float a_prev, const CfgItems& items,
                           long long fhw, cudaStream_t stream) {
  cfg_ddim_kernel<<<grid_for(static_cast<long long>(K) * n_item, 256), 256, 0, stream>>>(
      x, eps2, K, n_item, guidance, sqrtf(a_t), sqrtf(1.f - a_t), sqrtf(a_prev), sqrtf(1.f - a_prev), items, fhw);
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}

extern "C" int fz_cfg_ddim_step(float* x, const float* eps2, long long n, float guidance, float a_t, float a_prev, const float* x_inv,
                                const float* mask_a, const float* mask_b, long long fhw, int apply_blend, cudaStream_t stream) {
  FZ_CHECK_ARG(x && eps2, "fz_cfg_ddim_step: null pointer");
  FZ_CHECK_ARG(!apply_blend || (x_inv && mask_a && fhw > 0), "fz_cfg_ddim_step: blend needs x_inv and mask");
  CfgItems items;
  memset(&items, 0, sizeof(items));
  items.mask_a[0] = mask_a;
  items.mask_b[0] = mask_b;
  items.apply_blend[0] = apply_blend;
  items.x_inv[0] = x_inv;
  return cfg_ddim_launch(x, eps2, 1, n, guidance, a_t, a_prev, items, fhw, stream);
}

extern "C" int fz_cfg_ddim_step_batched(float* x, const float* eps2, int K, long long n_item, float guidance, float a_t, float a_prev,
                                        const float* x_inv, const float* const* mask_a, const float* const* mask_b, const int* apply_blend,
                                        long long fhw, cudaStream_t stream) {
  FZ_CHECK_ARG(x && eps2 && n_item > 0, "fz_cfg_ddim_step_batched: null pointer");
  FZ_CHECK_ARG(K >= 1 && K <= kCfgMaxItems, "fz_cfg_ddim_step_batched: K=%d unsupported (1..%d)", K, kCfgMaxItems);
  CfgItems items;
  memset(&items, 0, sizeof(items));
  for (int k = 0; k < K; ++k) {
    items.mask_a[k] = mask_a ? mask_a[k] : nullptr;
    items.mask_b[k] = mask_b ? mask_b[k] : nullptr;
    items.apply_blend[k] = apply_blend ? apply_blend[k] : 0;
    items.x_inv[k] = x_inv;
    FZ_CHECK_ARG(!items.apply_blend[k] || (x_inv && items.mask_a[k] && fhw > 0), "fz_cfg_ddim_step_batched: item %d: blend needs x_inv and mask", k);
  }
  return cfg_ddim_launch(x, eps2, K, n_item, guidance, a_t, a_prev, items, fhw, stream);
}

extern "C" int fz_cfg_ddim_step_multi(float* x, const float* eps2, int K, long long n_item, float guidance, float a_t, float a_prev,
                                      const float* const* x_inv, const float* const* mask_a, const float* const* mask_b, const int* apply_blend,
                                      long long fhw, cudaStream_t stream) {
  FZ_CHECK_ARG(x && eps2 && n_item > 0, "fz_cfg_ddim_step_multi: null pointer");
  FZ_CHECK_ARG(K >= 1 && K <= kCfgMaxItems, "fz_cfg_ddim_step_multi: K=%d unsupported (1..%d)", K, kCfgMaxItems);
  CfgItems items;
  memset(&items, 0, sizeof(items));
  for (int k = 0; k < K; ++k) {
    items.x_inv[k] = x_inv ? x_inv[k] : nullptr;
    items.mask_a[k] = mask_a ? mask_a[k] : nullptr;
    items.mask_b[k] = mask_b ? mask_b[k] : nullptr;
    items.apply_blend[k] = apply_blend ? apply_blend[k] : 0;
    FZ_CHECK_ARG(!items.apply_blend[k] || (items.x_inv[k] && items.mask_a[k] && fhw > 0), "fz_cfg_ddim_step_multi: item %d: blend needs x_inv and mask",
                 k);
  }
  return cfg_ddim_launch(x, eps2, K, n_item, guidance, a_t, a_prev, items, fhw, stream);
}

extern "C" int fz_blend_mask(const void* const* maps, int num_maps, int maps_f32, int F, int heads, int r, int ldm, int ntok, const float* word_w,
                             float th, int h, int w, float* out, cudaStream_t stream) {
  FZ_CHECK_ARG(maps && word_w && out && num_maps >= 1 && num_maps <= 8 && ntok <= 80, "fz_blend_mask: bad args");
  MaskParams p;
  for (int i = 0; i < 8; ++i) p.maps[i] = i < num_maps ? maps[i] : nullptr;
  p.num_maps = num_maps; p.maps_f32 = maps_f32; p.F = F; p.heads = heads; p.r = r; p.ldm = ldm; p.ntok = ntok;
  for (int i = 0; i < 80; ++i) p.w[i] = i < ntok ? word_w[i] : 0.f;  // word_w is a HOST array (77 floats, built once per edit)
  p.th = th; p.h = h; p.w_out = w; p.out = out;
  const size_t smem = static_cast<size_t>(2 * r * r) * sizeof(float);
  blend_mask_kernel<<<F, 256, smem, stream>>>(p);
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}


namespace fz {
// ---------------------------------------------------------------------------------------------------------------
// show_cross_attention on the device (prompt_attention/visualization.py:14-72): the heat map of text token `tok` in frame f is the mean
// over the selected cross-attention maps (layers) and heads of the time-averaged probabilities, scaled to 0..255 by its own maximum.
// The reference averages EVERY stored map (get_average_attention: self maps included) and moves the r16 cross maps to the host; here
// one CTA per (frame, token) reads the running-sum slabs in place and emits res*res bytes — the means' constant factors cancel in v / max.
// ---------------------------------------------------------------------------------------------------------------
struct HeatParams {
  const void* maps[8];
  int num_maps, maps_f32, heads, rr, ldm, ntok;
  unsigned char* out;  // [F, ntok, rr]
};
__global__ void __launch_bounds__(256) cross_heatmap_kernel(const __grid_constant__ HeatParams p) {
  const int tok = blockIdx.x, f = blockIdx.y;
  __shared__ float s_max[8];
  float vmax = 0.f;
  float vals[4];  // rr <= 1024 pixels, 256 threads
  int nv = 0;
  for (int px = threadIdx.x; px < p.rr; px += blockDim.x, ++nv) {
    float a = 0.f;
    for (int m = 0; m < p.num_maps; ++m) {
      for (int h = 0; h < p.heads; ++h) {
        const long long idx = ((static_cast<long long>(f) * p.heads + h) * p.rr + px) * p.ldm + tok;
        a += p.maps_f32 ? static_cast<const float*>(p.maps[m])[idx] : __half2float(static_cast<const __half*>(p.maps[m])[idx]);
      }
    }
    vals[nv] = a;
    vmax = fmaxf(vmax, a);
  }
  for (int o = 16; o > 0; o >>= 1) vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
  if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = vmax;
  __syncthreads();
  vmax = s_max[0];
  for (int w = 1; w < (blockDim.x >> 5); ++w) vmax = fmaxf(vmax, s_max[w]);
  nv = 0;
  for (int px = threadIdx.x; px < p.rr; px += blockDim.x, ++nv)
    p.out[(static_cast<long long>(f) * p.ntok + tok) * p.rr + px] =
        vmax > 0.f ? static_cast<unsigned char>(fminf(255.f, 255.f * vals[nv] / vmax)) : 0;  // all-zero column: 0, not 0/0
}

}  // namespace fz

extern "C" int fz_cross_heatmaps(const void* const* maps, int num_maps, int maps_f32, int F, int heads, int res, int ldm, int ntok, unsigned char* out,
                                 cudaStream_t stream) {
  FZ_CHECK_ARG(maps && out && num_maps >= 1 && num_maps <= 8 && res * res <= 1024 && ntok >= 1 && ntok <= ldm, "fz_cross_heatmaps: bad args");
  fz::HeatParams p;
  for (int i = 0; i < 8; ++i) p.maps[i] = i < num_maps ? maps[i] : nullptr;
  p.num_maps = num_maps; p.maps_f32 = maps_f32; p.heads = heads; p.rr = res * res; p.ldm = ldm; p.ntok = ntok; p.out = out;
  fz::cross_heatmap_kernel<<<dim3(ntok, F), 256, 0, stream>>>(p);
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// CLIP text encoder helpers (the transformer itself runs on fz_layernorm / fz_gemm / fz_attention with causal = 1)
// ---------------------------------------------------------------------------------------------------------------
namespace fz {
__global__ void embed_tokens_kernel(const float* __restrict__ tok, const float* __restrict__ pos, const long long* __restrict__ ids,
                                    __half* __restrict__ out, int rows, int L, int C) {
  const int r = blockIdx.x;
  const long long id = ids[r];
  const float* t = tok + id * C;
  const float* pp = pos + static_cast<long long>(r % L) * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) out[static_cast<long long>(r) * C + c] = __float2half_rn(t[c] + pp[c]);
}
__global__ void quick_gelu_kernel(__half* __restrict__ x, long long n) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float v = __half2float(x[i]);
    x[i] = __float2half_rn(v / (1.0f + __expf(-1.702f * v)));
  }
}
// exact (erf) GELU of the SD-2 text encoders' MLP: 0.5 v (1 + erf(v / sqrt 2)), as torch.nn.functional.gelu(approximate="none")
__global__ void gelu_kernel(__half* __restrict__ x, long long n) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float v = __half2float(x[i]);
    x[i] = __float2half_rn(0.5f * v * (1.0f + erff(v * 0.70710678118654752f)));
  }
}
}  // namespace fz

extern "C" int fz_embed_tokens_f16(const float* tok, const float* pos, const long long* ids, void* out, int rows, int L, int C, cudaStream_t stream) {
  FZ_CHECK_ARG(tok && pos && ids && out && rows > 0 && L > 0 && C > 0, "fz_embed_tokens: bad args");
  fz::embed_tokens_kernel<<<rows, 256, 0, stream>>>(tok, pos, ids, static_cast<__half*>(out), rows, L, C);
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}
extern "C" int fz_quick_gelu_f16(void* x, long long n, cudaStream_t stream) {
  FZ_CHECK_ARG(x && n > 0, "fz_quick_gelu: bad args");
  fz::quick_gelu_kernel<<<static_cast<int>(std::min<long long>((n + 255) / 256, 132 * 8)), 256, 0, stream>>>(static_cast<__half*>(x), n);
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}
extern "C" int fz_gelu_f16(void* x, long long n, cudaStream_t stream) {
  FZ_CHECK_ARG(x && n > 0, "fz_gelu: bad args");
  fz::gelu_kernel<<<static_cast<int>(std::min<long long>((n + 255) / 256, 132 * 8)), 256, 0, stream>>>(static_cast<__half*>(x), n);
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Row softmax in place: x[r, :n] <- softmax(scale * x[r, :n]) (fp32 math, fp16 storage).  The VAE's single-head 512-wide mid-block
// attention (diffusers AttentionBlock: stable_diffusion.py:297-319 decode path) runs as GEMM -> this -> GEMM: its head dim exceeds what
// the fused attention kernel holds in registers (d <= 192).  One warp per row.
// ---------------------------------------------------------------------------------------------------------------
namespace fz {
__global__ void __launch_bounds__(256) softmax_rows_kernel(__half* __restrict__ x, long long rows, int n, long long ld, float scale_log2) {
  const int lane = threadIdx.x & 31;
  const long long r = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  __half* row = x + r * ld;
  float m = -INFINITY;
  for (int c = lane * 8; c < n; c += 256) {
    const Half8 h = *reinterpret_cast<const Half8*>(row + c);
#pragma unroll
    for (int e = 0; e < 8; ++e) m = fmaxf(m, __half2float(h.v[e]));
  }
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  float sum = 0.f;
  for (int c = lane * 8; c < n; c += 256) {
    const Half8 h = *reinterpret_cast<const Half8*>(row + c);
#pragma unroll
    for (int e = 0; e < 8; ++e) sum += exp2f((__half2float(h.v[e]) - m) * scale_log2);
  }
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float inv = 1.0f / sum;
  for (int c = lane * 8; c < n; c += 256) {
    Half8 h = *reinterpret_cast<const Half8*>(row + c);
#pragma unroll
    for (int e = 0; e < 8; ++e) h.v[e] = __float2half_rn(exp2f((__half2float(h.v[e]) - m) * scale_log2) * inv);
    *reinterpret_cast<Half8*>(row + c) = h;
  }
}
}  // namespace fz

extern "C" int fz_softmax_rows_f16(void* x, long long rows, int n, long long ld, float scale, cudaStream_t stream) {
  FZ_CHECK_ARG(x && rows > 0 && n > 0 && n % 8 == 0 && ld % 8 == 0 && scale > 0.f, "fz_softmax_rows: n and ld must be multiples of 8");
  fz::softmax_rows_kernel<<<static_cast<unsigned>((rows + 7) / 8), 256, 0, stream>>>(static_cast<__half*>(x), rows, n, ld, scale * 1.4426950408889634f);
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}
