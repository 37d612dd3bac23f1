// fz_gemm.cu — the "tap-GEMM": one persistent, warp-specialised wgmma kernel that serves every dense contraction of the
// UNet step except attention:
//     D[M, N] = sum_{tap} A_tap[M, K] * W_tap[N, K]^T   (+ bias, + per-batch time-embedding row, + residual, GEGLU, V^T store)
//   * nn.Linear / 1x1 conv ............ 1 tap, A = [M, K] row-major tokens
//   * 3x3 conv (stride 1 / stride 2) .. 9 taps, A = NHWC activation addressed through a 4-D / 5-D TMA map; the tap moves the
//                                       box by (dy, dx) and TMA zero-fills the halo (implicit GEMM, no im2col in HBM)
//   * temporal LoRA Conv1d(k=3) ....... 3 taps along the frame axis of [B, F, HW, C]
// Reference ops replaced: models/resnet.py:57-80 (PseudoConv3d.forward), models/lora.py:46-54, nn.Linear call sites of
// prompt_attention/attention_register.py:81,99-100,124,156-160,214 and diffusers FeedForward/GEGLU (models/attention.py:320).
//
// Structure (per CTA, 384 threads = 3 warpgroups, 1 CTA / SM, grid = min(#tiles, #SMs), static round-robin tile schedule):
//   warpgroup 2    : TMA producer — A box {64ch, rows} + W box {64ch, BLOCK_N} per stage, SWIZZLE_128B, mbarrier complete_tx
//   warpgroups 0-1 : consumers   — wgmma m64 x N=BLOCK_N x k16 on rows [64 wg, 64 wg + 64) of the 128-row tile, fp32 accumulators
//                                  in registers, fused epilogue straight from the accumulator fragment while the producer already
//                                  fills the ring with the next tile's operands
#include "fz_common.cuh"
#include "fz_wgmma.cuh"

#include <algorithm>
#include <climits>
#include <cstdio>
#include <cstring>

#include "../../include/fatezero_b200.h"

namespace fz {

constexpr int kMaxTaps = 9;
constexpr int kBlockM = 128;
constexpr int kBlockK = 64;
constexpr int kATileBytes = kBlockM * kBlockK * 2;  // 16 KiB

struct TapGemmParams {
  CUtensorMap tmA;
  CUtensorMap tmB;
  CUtensorMap tmR[2]; // skip tensors [M, N] folded into the accumulator as extra k-blocks: box {64 cols, 128 rows}
  CUtensorMap tmE;    // identity blocks E[j][n][k] = (n == 64 j + k): (k : 64, n : 256, j : 4), box {64, BLOCK_N, 1}
  int n_res;          // number of folded skip tensors (0..2); the epilogue then sees residual == residual2 == null
  int res_kblocks;    // ceil(BLOCK_N / 64) extra k-blocks per folded skip tensor
  int a_rank;         // 2..5
  int M, N;           // valid output rows / columns (for GEGLU: N = number of OUTPUT columns = half the GEMM columns)
  int rows_per_tile;  // <= 128; tile t covers output rows [t*rows_per_tile, ...)
  int a_box_bytes;    // bytes TMA writes for one A box (rows_per_tile * 128)
  int k_blocks;       // per tap
  int num_taps;
  int n_tiles, m_tiles;
  int ndecomp;        // how many of A's dims 1.. take part in the row decomposition
  int dimsz[4];       // their sizes
  int tap_off[kMaxTaps][5];  // coordinate offsets per tap for A dims 0..4
  const float* bias;         // [gemm columns] fp32 (GEGLU: packed like the weights) or null
  const float* group_bias;   // [M / rows_per_group, N] fp32 or null (time-embedding projection per batch element)
  int rows_per_group;
  const __half* residual;    // [M, ldr] or null
  long long ldr;
  const __half* residual2;   // second skip tensor [M, ldr2] or null
  long long ldr2;
  __half* out;
  long long ldo;
  int mode;          // FZ_EPI_ROWMAJOR / FZ_EPI_GEGLU
  int vt_col_start;  // gemm columns >= this are written transposed (V^T) instead of row-major; INT_MAX = off
  __half* out_vt;    // [BF, heads, d, S]
  int vt_S, vt_d, vt_heads, vt_ld;
};

template <int BLOCK_N>
struct TapGemmCfg {
  static constexpr int kBTileBytes = BLOCK_N * kBlockK * 2;
  static constexpr int kBTilePad = (kBTileBytes + 1023) / 1024 * 1024;
  static constexpr int kStageBytes = kATileBytes + kBTilePad;
  static constexpr int kStagesRaw = (227 * 1024 - 1280) / kStageBytes;
  static constexpr int kStages = kStagesRaw > 8 ? 8 : kStagesRaw;
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
};

// exact-erf GELU (F.gelu default).  erf via Abramowitz-Stegun 7.1.26 (|error| <= 1.5e-7, far below the fp16 output rounding):
// 1 MUFU.RCP + 1 MUFU.EX2 + 8 FMA instead of the ~40-instruction erff().
__device__ __forceinline__ float gelu_erf(float x) {
  const float z = fabsf(x) * 0.70710678118654752f;
  float t, e;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.4426950408889634f * z * z));
  const float erf_abs = fmaf(-poly * t, e, 1.0f);
  return 0.5f * x * (1.0f + copysignf(erf_abs, x));
}

// one output element of the row-major / V^T epilogue (right-edge columns and the V^T part; the paired fast path is inlined below)
__device__ __forceinline__ void epi_store1(const TapGemmParams& p, long long m, int col, float v, const float* gb) {
  if (p.bias) v += __ldg(p.bias + col);
  if (col >= p.vt_col_start) {
    const long long bf = m / p.vt_S;
    const int s = static_cast<int>(m % p.vt_S);
    const int cv = col - p.vt_col_start;
    p.out_vt[((bf * p.vt_heads + cv / p.vt_d) * p.vt_d + cv % p.vt_d) * p.vt_ld + s] = __float2half_rn(v);
  } else {
    if (gb) v += __ldg(gb + col);
    if (p.residual) v += __half2float(p.residual[m * p.ldr + col]);
    if (p.residual2) v += __half2float(p.residual2[m * p.ldr2 + col]);
    p.out[m * p.ldo + col] = __float2half_rn(v);
  }
}

template <int BLOCK_N>
__global__ void __launch_bounds__(384, 1) tapgemm_kernel(const __grid_constant__ TapGemmParams p) {
  using Cfg = TapGemmCfg<BLOCK_N>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStageBytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + Cfg::kStages;

  const int wg = threadIdx.x >> 7;
  pdl_launch_dependents();
  const int num_tiles = p.m_tiles * p.n_tiles;
  const int k_iters = p.num_taps * p.k_blocks + p.n_res * p.res_kblocks;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmA);
    tma_prefetch_desc(&p.tmB);
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);  // one arrive per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();  // everything above overlapped the previous kernel's tail; operands / outputs are touched only from here on

  if (wg == 2) {
    // ===================== TMA producer =====================
    if (threadIdx.x == 256) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int mt = tile / p.n_tiles, nt = tile % p.n_tiles;
        int rem = mt * p.rows_per_tile;
        int base[5] = {0, 0, 0, 0, 0};
        for (int d = 0; d < p.ndecomp; ++d) {
          base[d + 1] = rem % p.dimsz[d];
          rem /= p.dimsz[d];
        }
        const int n0 = nt * BLOCK_N;
        for (int tap = 0; tap < p.num_taps; ++tap) {
          const int c1 = base[1] + p.tap_off[tap][1], c2 = base[2] + p.tap_off[tap][2];
          const int c3 = base[3] + p.tap_off[tap][3], c4 = base[4] + p.tap_off[tap][4];
          for (int kb = 0; kb < p.k_blocks; ++kb) {
            mbar_wait(&empty[stage], phase ^ 1);
            uint8_t* sa = smem + stage * Cfg::kStageBytes;
            uint8_t* sb = sa + kATileBytes;
            mbar_expect_tx(&full[stage], p.a_box_bytes + Cfg::kBTileBytes);
            const int c0 = kb * kBlockK + p.tap_off[tap][0];
            switch (p.a_rank) {
              case 2: tma_load_2d(sa, &p.tmA, &full[stage], c0, c1); break;
              case 3: tma_load_3d(sa, &p.tmA, &full[stage], c0, c1, c2); break;
              case 4: tma_load_4d(sa, &p.tmA, &full[stage], c0, c1, c2, c3); break;
              default: tma_load_5d(sa, &p.tmA, &full[stage], c0, c1, c2, c3, c4); break;
            }
            tma_load_3d(sb, &p.tmB, &full[stage], kb * kBlockK, n0, tap);
            if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
          }
        }
        // Skip connections ride the same pipeline as extra k-blocks: D += R[:, n0 + 64 j ...] * E_j^T with E_j a 0/1 selection block
        // (exact: fp16 x 1.0 accumulated in fp32 after the last tap, the same order as an epilogue add), so the skip tensor is
        // prefetched by the TMA ring like any operand instead of being waited for in the epilogue.
        for (int r = 0; r < p.n_res; ++r) {
          for (int j = 0; j < p.res_kblocks; ++j) {
            mbar_wait(&empty[stage], phase ^ 1);
            uint8_t* sa = smem + stage * Cfg::kStageBytes;
            uint8_t* sb = sa + kATileBytes;
            mbar_expect_tx(&full[stage], kATileBytes + Cfg::kBTileBytes);
            tma_load_2d(sa, &p.tmR[r], &full[stage], n0 + j * kBlockK, mt * p.rows_per_tile);
            tma_load_3d(sb, &p.tmE, &full[stage], 0, 0, j);
            if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }

  // ===================== consumer warpgroups: wgmma mainloop + epilogue =====================
  const int lane = threadIdx.x & 31;
  const int warp_in = (threadIdx.x >> 5) & 3;
  const uint64_t desc0 = wgmma_desc_k_sw128(smem_u32(smem));
  float acc[BLOCK_N / 2];
  int stage = 0;
  uint32_t phase = 0;
  // accumulator fragment: acc[4 i + 2 h + j] = tile row r_base + 8 h, tile column 8 i + c_base + j
  const int r_base = wg * 64 + warp_in * 16 + (lane >> 2);
  const int c_base = 2 * (lane & 3);
  const bool pair_ok = (p.ldo % 2) == 0 && (reinterpret_cast<uintptr_t>(p.out) & 3) == 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int mt = tile / p.n_tiles, nt = tile % p.n_tiles;
    int prev = -1;
    for (int it = 0; it < k_iters; ++it) {
      mbar_wait(&full[stage], phase);
      const uint64_t da = desc0 + static_cast<uint32_t>((stage * Cfg::kStageBytes + wg * 64 * 128) >> 4);
      const uint64_t db = desc0 + static_cast<uint32_t>((stage * Cfg::kStageBytes + kATileBytes) >> 4);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBlockK / 16; ++k) wgmma_f16<BLOCK_N>(acc, da + 2 * k, db + 2 * k, (it | k) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();  // the previous stage's MMAs are done: hand its buffers back to the producer
      if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
      prev = stage;
      if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);

#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = r_base + 8 * h;
      const long long m = static_cast<long long>(mt) * p.rows_per_tile + r;
      if (r >= p.rows_per_tile || m >= p.M) continue;
      if (p.mode == FZ_EPI_GEGLU) {
        // x columns [0, HALF) and gate columns [HALF, BLOCK_N) of the tile sit in the same thread (HALF is a multiple of 8)
        constexpr int HALF = BLOCK_N / 2;
        if constexpr (HALF % 8 == 0) {
          __half* orow = p.out + m * p.ldo;
#pragma unroll
          for (int i = 0; i < HALF / 8; ++i) {
            const int c = 8 * i + c_base;
            const int oc = nt * HALF + c;
            if (oc >= p.N) continue;
            float x0 = acc[4 * i + 2 * h], x1 = acc[4 * i + 2 * h + 1];
            float g0 = acc[4 * (i + HALF / 8) + 2 * h], g1 = acc[4 * (i + HALF / 8) + 2 * h + 1];
            if (p.bias) {
              const float* b = p.bias + nt * BLOCK_N + c;
              x0 += __ldg(b); x1 += __ldg(b + 1); g0 += __ldg(b + HALF); g1 += __ldg(b + HALF + 1);
            }
            const float o0 = x0 * gelu_erf(g0), o1 = x1 * gelu_erf(g1);
            if (pair_ok && oc + 1 < p.N) {
              *reinterpret_cast<__half2*>(orow + oc) = __floats2half2_rn(o0, o1);
            } else {
              orow[oc] = __float2half_rn(o0);
              if (oc + 1 < p.N) orow[oc + 1] = __float2half_rn(o1);
            }
          }
        }
      } else {
        const float* gb = p.group_bias ? p.group_bias + (m / p.rows_per_group) * p.N : nullptr;
        __half* orow = p.out + m * p.ldo;
#pragma unroll
        for (int i = 0; i < BLOCK_N / 8; ++i) {
          const int col = nt * BLOCK_N + 8 * i + c_base;
          if (col >= p.N) continue;
          float v0 = acc[4 * i + 2 * h], v1 = acc[4 * i + 2 * h + 1];
          if (pair_ok && col + 2 <= p.N && col + 2 <= p.vt_col_start) {
            if (p.bias) { v0 += __ldg(p.bias + col); v1 += __ldg(p.bias + col + 1); }
            if (gb) { v0 += __ldg(gb + col); v1 += __ldg(gb + col + 1); }
            if (p.residual) { v0 += __half2float(p.residual[m * p.ldr + col]); v1 += __half2float(p.residual[m * p.ldr + col + 1]); }
            if (p.residual2) { v0 += __half2float(p.residual2[m * p.ldr2 + col]); v1 += __half2float(p.residual2[m * p.ldr2 + col + 1]); }
            *reinterpret_cast<__half2*>(orow + col) = __floats2half2_rn(v0, v1);
          } else {
            epi_store1(p, m, col, v0, gb);
            if (col + 1 < p.N) epi_store1(p, m, col + 1, v1, gb);
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
static int g_num_sms = 0;
static int num_sms() {
  if (g_num_sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_num_sms <= 0) g_num_sms = 132;
  }
  return g_num_sms;
}

template <int BN>
static int launch_tapgemm(const TapGemmParams& p, cudaStream_t stream) {
  using Cfg = TapGemmCfg<BN>;
  static bool configured = false;
  if (!configured) {
    FZ_CUDA(cudaFuncSetAttribute(tapgemm_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    configured = true;
  }
  const int tiles = p.m_tiles * p.n_tiles;
  const int grid = std::min(tiles, num_sms());
  FZ_CUDA(launch_pdl(tapgemm_kernel<BN>, dim3(grid), dim3(384), Cfg::kSmemBytes, stream, p));
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}

// Skip tensors that fold_residuals() turns into extra k-blocks (all present ones, or none): row-major epilogue without V^T, and every
// skip tensor TMA-addressable (16-byte base and row stride).
static int n_foldable(const TapGemmParams& p) {
  if (p.mode != FZ_EPI_ROWMAJOR || p.vt_col_start != INT_MAX) return 0;
  const __half* rs[2] = {p.residual, p.residual2};
  const long long lds[2] = {p.ldr, p.ldr2};
  int n = 0;
  for (int i = 0; i < 2; ++i) {
    if (!rs[i]) continue;
    if ((reinterpret_cast<uintptr_t>(rs[i]) & 15) != 0 || lds[i] % 8 != 0) return 0;
    ++n;
  }
  return n;
}

// k_main = taps x k-blocks of the contraction; p holds the epilogue (fill_epilogue) so the folded skip k-blocks can be counted.
static int pick_block_n(const TapGemmParams& p, int gemm_cols, int forced, int m_tiles, int k_main) {
  if (forced > 0) return forced;
  static const int cands[] = {256, 160, 128, 64, 32, 16};
  if (p.mode == FZ_EPI_GEGLU) return (gemm_cols % 256 == 0) ? 256 : ((gemm_cols % 160 == 0) ? 160 : ((gemm_cols % 128 == 0) ? 128 : ((gemm_cols % 64 == 0) ? 64 : 32)));
  // Cost model: tiles run in waves of one per SM.  Time of a 128 x bn tile with k k-blocks (folded skip blocks included), fitted to
  // per-shape timings of the UNet's linears, 3x3 convs and temporal convs on an H100 80 GB HBM3 (700 W):  bn k + 24 bn + 110 k + 0.15 bn^2.
  // Beyond the MMA term (bn k), the per-tile parts that grow with bn (epilogue, and the ring holding fewer stages of a wider W tile)
  // make narrow tiles win at short K: BLOCK_N 64 for the K <= 640 linears, 160 for the 9-tap convs.
  const int sms = num_sms();
  const int n_fold = n_foldable(p);
  int best = 16;
  double best_cost = 1e30;
  for (int bn : cands) {
    const long long n_tiles = (gemm_cols + bn - 1) / bn;
    const long long tiles = n_tiles * m_tiles;
    const long long waves = (tiles + sms - 1) / sms;
    const double k = k_main + n_fold * ((bn + kBlockK - 1) / kBlockK);
    const double cost = static_cast<double>(waves) * (bn * k + 24.0 * bn + 110.0 * k + 0.15 * bn * bn);
    if (cost < best_cost - 1e-9) { best_cost = cost; best = bn; }
  }
  return best;
}

// Selection blocks for folding skip tensors into the MMA pipeline: E[j][n][k] = 1 if n == 64 j + k (static device memory, filled once).
__device__ __half g_eye[4][256][64];
__global__ void eye_init_kernel() {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < 4 * 256 * 64; i += gridDim.x * blockDim.x) {
    const int k = i % 64, n = (i / 64) % 256, j = i / (64 * 256);
    (&g_eye[0][0][0])[i] = __float2half_rn(n == 64 * j + k ? 1.f : 0.f);
  }
}

// One-time fill of the selection table.  It synchronises the stream, which is illegal under stream capture: fz_init() runs it up front
// (engine construction), so that the first GEMM with a skip tensor may already sit inside a CUDA-graph capture.
static int eye_table(__half** out, cudaStream_t stream) {
  static __half* eye = nullptr;
  if (!eye) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    FZ_CUDA(cudaStreamIsCapturing(stream, &cs));
    FZ_CHECK_ARG(cs == cudaStreamCaptureStatusNone, "fz_init() must run once before the library is used under CUDA-graph capture");
    __half* e = nullptr;
    FZ_CUDA(cudaGetSymbolAddress(reinterpret_cast<void**>(&e), g_eye));
    eye_init_kernel<<<64, 256, 0, stream>>>();
    FZ_CUDA(cudaGetLastError());
    // the table is read by TMA of kernels on ANY stream afterwards: make the one-time fill visible before returning
    FZ_CUDA(cudaStreamSynchronize(stream));
    eye = e;
  }
  *out = eye;
  return FZ_OK;
}

static int fold_residuals(TapGemmParams& p, int bn, cudaStream_t stream) {
  p.n_res = 0;
  p.res_kblocks = 0;
  if (n_foldable(p) == 0) return FZ_OK;  // none, or not TMA-addressable: epilogue path
  const __half* rs[2] = {p.residual, p.residual2};
  const long long lds[2] = {p.ldr, p.ldr2};
  __half* eye = nullptr;
  if (int rc = eye_table(&eye, stream)) return rc;
  {
    uint64_t dims[3] = {64, 256, 4};
    uint64_t strides[2] = {64, 64 * 256};
    uint32_t box[3] = {64, static_cast<uint32_t>(bn), 1};
    if (int rc = encode_tmap_f16(&p.tmE, eye, 3, dims, strides, box, true)) return rc;
  }
  for (int i = 0; i < 2; ++i) {
    if (!rs[i]) continue;
    uint64_t dims[2] = {static_cast<uint64_t>(p.N), static_cast<uint64_t>(p.M)};
    uint64_t strides[1] = {static_cast<uint64_t>(lds[i])};
    uint32_t box[2] = {kBlockK, kBlockM};
    if (int rc = encode_tmap_f16(&p.tmR[p.n_res], rs[i], 2, dims, strides, box, true)) return rc;
    ++p.n_res;
  }
  p.res_kblocks = (bn + kBlockK - 1) / kBlockK;
  p.residual = nullptr;
  p.residual2 = nullptr;
  return FZ_OK;
}

// bn: the caller's pick_block_n() result (its W tensor map already has a {64, bn} box)
static int dispatch_tapgemm(TapGemmParams& p, int gemm_cols, int bn, cudaStream_t stream) {
  if (int rc = check_single_device()) return rc;
  p.n_tiles = (gemm_cols + bn - 1) / bn;
  if (int rc = fold_residuals(p, bn, stream)) return rc;
  switch (bn) {
    case 256: return launch_tapgemm<256>(p, stream);
    case 160: return launch_tapgemm<160>(p, stream);
    case 128: return launch_tapgemm<128>(p, stream);
    case 64: return launch_tapgemm<64>(p, stream);
    case 32: return launch_tapgemm<32>(p, stream);
    case 16: return launch_tapgemm<16>(p, stream);
    default: set_error("unsupported BLOCK_N %d", bn); return FZ_ERR_INVALID;
  }
}

static int fill_epilogue(TapGemmParams& p, const fz_epilogue_t* e, int M, int gemm_cols) {
  p.bias = nullptr; p.group_bias = nullptr; p.rows_per_group = 1; p.residual = nullptr; p.ldr = 0; p.residual2 = nullptr; p.ldr2 = 0;
  p.mode = FZ_EPI_ROWMAJOR; p.vt_col_start = INT_MAX; p.out_vt = nullptr; p.vt_S = p.vt_d = p.vt_heads = p.vt_ld = 1;
  p.N = gemm_cols;
  if (!e) return FZ_OK;
  p.bias = e->bias; p.group_bias = e->group_bias; p.rows_per_group = e->rows_per_group > 0 ? e->rows_per_group : 1;
  p.residual = static_cast<const __half*>(e->residual); p.ldr = e->ldr;
  p.residual2 = static_cast<const __half*>(e->residual2); p.ldr2 = e->ldr2;
  p.mode = e->mode;
  if (e->mode == FZ_EPI_GEGLU) {
    FZ_CHECK_ARG(gemm_cols % 2 == 0, "GEGLU needs an even number of GEMM columns");
    // the GEGLU epilogue applies the bias only: any other term would be dropped without a trace
    FZ_CHECK_ARG(!e->residual && !e->residual2 && !e->group_bias && !e->out_vt,
                 "GEGLU epilogue takes no residual, group bias or V^T output");
    p.N = gemm_cols / 2;
  }
  if (e->out_vt) {
    FZ_CHECK_ARG(e->vt_S > 0 && e->vt_d > 0 && e->vt_heads > 0 && M % e->vt_S == 0, "bad V^T geometry");
    p.vt_col_start = e->vt_col_start; p.out_vt = static_cast<__half*>(e->out_vt);
    p.vt_S = e->vt_S; p.vt_d = e->vt_d; p.vt_heads = e->vt_heads; p.vt_ld = e->vt_ld > 0 ? e->vt_ld : e->vt_S;
  }
  return FZ_OK;
}

}  // namespace fz

using namespace fz;

// One-time device-side initialisation (constant tables).  Idempotent; must have run before the first call under stream capture.
extern "C" int fz_init(cudaStream_t stream) {
  if (int rc = check_single_device()) return rc;
  __half* eye = nullptr;
  return eye_table(&eye, stream);
}

// D[M,N] = A[M,K] * W[N,K]^T (+epilogue).  A, W fp16 row-major (lda, ldw in elements, multiples of 8).
extern "C" int fz_gemm_f16(const void* A, long long lda, const void* W, long long ldw, int M, int N, int K, const fz_epilogue_t* epi,
                           void* out, long long ldo, int force_block_n, cudaStream_t stream) {
  FZ_CHECK_ARG(A && W && out, "fz_gemm_f16: null pointer");
  FZ_CHECK_ARG(M > 0 && N > 0 && K > 0, "fz_gemm_f16: bad shape %d %d %d", M, N, K);
  FZ_CHECK_ARG(lda % 8 == 0 && ldw % 8 == 0 && K % 8 == 0, "fz_gemm_f16: lda/ldw/K must be multiples of 8 (16-byte TMA strides)");
  TapGemmParams p;
  memset(&p, 0, sizeof(p));
  {
    uint64_t dims[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(M)};
    uint64_t strides[1] = {static_cast<uint64_t>(lda)};
    uint32_t box[2] = {kBlockK, kBlockM};
    if (int rc = encode_tmap_f16(&p.tmA, A, 2, dims, strides, box, true)) return rc;
  }
  const int rc0 = fill_epilogue(p, epi, M, N);
  if (rc0) return rc0;
  p.m_tiles = (M + kBlockM - 1) / kBlockM;
  const int bn = pick_block_n(p, N, force_block_n, p.m_tiles, (K + kBlockK - 1) / kBlockK);
  {
    uint64_t dims[3] = {static_cast<uint64_t>(K), static_cast<uint64_t>(N), 1};
    uint64_t strides[2] = {static_cast<uint64_t>(ldw), static_cast<uint64_t>(ldw) * N};
    uint32_t box[3] = {kBlockK, static_cast<uint32_t>(bn), 1};
    if (int rc = encode_tmap_f16(&p.tmB, W, 3, dims, strides, box, true)) return rc;
  }
  p.a_rank = 2; p.M = M; p.rows_per_tile = kBlockM; p.a_box_bytes = kATileBytes;
  p.k_blocks = (K + kBlockK - 1) / kBlockK; p.num_taps = 1;
  p.m_tiles = (M + kBlockM - 1) / kBlockM;
  p.ndecomp = 1; p.dimsz[0] = INT_MAX;
  p.out = static_cast<__half*>(out); p.ldo = ldo;
  return dispatch_tapgemm(p, N, bn, stream);
}

// 3x3 convolution, padding 1, stride 1 or 2, NHWC fp16.  x: [NB, H, W, Cin] (pixel stride ldx >= Cin),
// w: [9][Cout][Cin] (tap-major, tap = ky*3+kx), out: [NB, Ho, Wo, Cout] row-major with row stride ldo.
// asym_pad (stride 2 only): the input is padded by one pixel on the right / bottom ONLY (diffusers Downsample2D with padding = 0 in the VAE
// encoder: F.pad(x, (0, 1, 0, 1)) then a stride-2 conv without padding) instead of symmetrically.
static int conv3x3_impl(const void* x, long long ldx, int NB, int H, int W, int Cin, const void* w, int Cout, int stride, int asym_pad,
                        const fz_epilogue_t* epi, void* out, long long ldo, int force_block_n, cudaStream_t stream) {
  FZ_CHECK_ARG(x && w && out, "fz_conv3x3: null pointer");
  FZ_CHECK_ARG(stride == 1 || stride == 2, "fz_conv3x3: stride must be 1 or 2");
  FZ_CHECK_ARG(Cin % 8 == 0 && ldx % 8 == 0, "fz_conv3x3: Cin/ldx must be multiples of 8");
  FZ_CHECK_ARG(stride == 1 || (H % 2 == 0 && W % 2 == 0), "fz_conv3x3: stride 2 needs even H, W");
  const int Ho = H / stride, Wo = W / stride;
  FZ_CHECK_ARG(!asym_pad || stride == 2, "fz_conv3x3: asymmetric padding is the stride-2 downsample variant");
  // box over (x, y, n): the full output width, as many rows / images as fit 128 GEMM rows.  Wider images (VAE resolutions) are tiled in
  // row segments of bw pixels, bw the largest divisor of Wo up to 128 (Wo 256, 512: 128; 192, 288, 576: 96; 144: 72; 160, 320: 80), so a
  // tile never crosses an image row
  int bw = std::min(Wo, 128);
  while (Wo % bw) --bw;
  FZ_CHECK_ARG(Wo <= 128 || bw >= 8, "fz_conv3x3: output width %d has no divisor in [8, 128] to tile its rows with", Wo);
  int bh = (bw == Wo) ? std::min(Ho, 128 / bw) : 1;
  while (Ho % bh) --bh;
  int bn_img = (bh == Ho) ? std::min(NB, 128 / (bw * bh)) : 1;
  while (NB % bn_img) --bn_img;
  TapGemmParams p;
  memset(&p, 0, sizeof(p));
  const int M = NB * Ho * Wo;
  const int rc0 = fill_epilogue(p, epi, M, Cout);
  if (rc0) return rc0;
  if (stride == 1) {
    uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)NB};
    uint64_t strides[3] = {(uint64_t)ldx, (uint64_t)ldx * W, (uint64_t)ldx * W * H};
    uint32_t box[4] = {kBlockK, (uint32_t)bw, (uint32_t)bh, (uint32_t)bn_img};
    if (int rc = encode_tmap_f16(&p.tmA, x, 4, dims, strides, box, true)) return rc;
    p.a_rank = 4;
    for (int t = 0; t < 9; ++t) {
      p.tap_off[t][0] = 0; p.tap_off[t][1] = t % 3 - 1; p.tap_off[t][2] = t / 3 - 1; p.tap_off[t][3] = 0; p.tap_off[t][4] = 0;
    }
  } else {
    // stride 2: view the input as (c|px : 2*ldx, x' : W/2, y' : H/2, n, py : 2); tap (ky,kx) reads phase (py,px) shifted by {-1,0}
    uint64_t dims[5] = {(uint64_t)(ldx + Cin), (uint64_t)Wo, (uint64_t)Ho, (uint64_t)NB, 2};
    uint64_t strides[4] = {(uint64_t)2 * ldx, (uint64_t)2 * ldx * W, (uint64_t)ldx * W * H, (uint64_t)ldx * W};
    uint32_t box[5] = {kBlockK, (uint32_t)bw, (uint32_t)bh, (uint32_t)bn_img, 1};
    if (int rc = encode_tmap_f16(&p.tmA, x, 5, dims, strides, box, true)) return rc;
    p.a_rank = 5;
    for (int t = 0; t < 9; ++t) {
      const int ky = t / 3, kx = t % 3;
      // symmetric padding 1: input row 2y + ky - 1 -> phase (ky != 1), shift -1 for ky = 0; right/bottom-only padding: input row 2y + ky ->
      // phase ky & 1, shift +1 for ky = 2 (the zero row / column beyond the edge is TMA's out-of-bounds fill)
      const int py = asym_pad ? (ky & 1) : ((ky == 1) ? 0 : 1), px = asym_pad ? (kx & 1) : ((kx == 1) ? 0 : 1);
      p.tap_off[t][0] = px * (int)ldx;
      p.tap_off[t][1] = asym_pad ? (kx >> 1) : ((kx == 0) ? -1 : 0);
      p.tap_off[t][2] = asym_pad ? (ky >> 1) : ((ky == 0) ? -1 : 0);
      p.tap_off[t][3] = 0;
      p.tap_off[t][4] = py;
    }
  }
  p.rows_per_tile = bw * bh * bn_img;
  p.m_tiles = M / p.rows_per_tile;
  const int bn = pick_block_n(p, Cout, force_block_n, p.m_tiles, 9 * ((Cin + kBlockK - 1) / kBlockK));
  {
    uint64_t dims[3] = {(uint64_t)Cin, (uint64_t)Cout, 9};
    uint64_t strides[2] = {(uint64_t)Cin, (uint64_t)Cin * Cout};
    uint32_t box[3] = {kBlockK, (uint32_t)bn, 1};
    if (int rc = encode_tmap_f16(&p.tmB, w, 3, dims, strides, box, true)) return rc;
  }
  p.M = M; p.rows_per_tile = bw * bh * bn_img; p.a_box_bytes = p.rows_per_tile * 128;
  p.k_blocks = (Cin + kBlockK - 1) / kBlockK; p.num_taps = 9;
  p.m_tiles = M / p.rows_per_tile;
  p.ndecomp = 3; p.dimsz[0] = Wo; p.dimsz[1] = Ho; p.dimsz[2] = NB;
  p.out = static_cast<__half*>(out); p.ldo = ldo;
  return dispatch_tapgemm(p, Cout, bn, stream);
}

extern "C" int fz_conv3x3_nhwc_f16(const void* x, long long ldx, int NB, int H, int W, int Cin, const void* w, int Cout, int stride,
                                   const fz_epilogue_t* epi, void* out, long long ldo, int force_block_n, cudaStream_t stream) {
  return conv3x3_impl(x, ldx, NB, H, W, Cin, w, Cout, stride, 0, epi, out, ldo, force_block_n, stream);
}

extern "C" int fz_conv3x3_down_asym_nhwc_f16(const void* x, long long ldx, int NB, int H, int W, int Cin, const void* w, int Cout,
                                             const fz_epilogue_t* epi, void* out, long long ldo, int force_block_n, cudaStream_t stream) {
  return conv3x3_impl(x, ldx, NB, H, W, Cin, w, Cout, 2, 1, epi, out, ldo, force_block_n, stream);
}

// Temporal Conv1d(k=3, padding 1, no bias) over the frame axis: x [B, F, HW, Cin] fp16 (row stride ldx), w [3][Cout][Cin].
// out[b,f,p,:] = sum_t w[t] * x[b, f+t-1, p, :]  (+ epilogue: residual = identity skip of the LoRA, group_bias = time embedding).
// halo = 1 (frame-sharded execution): x is [B, F+2, HW, Cin] whose frames 0 and F+1 hold the neighbour ranks' boundary frames (zeros at
// the ends of the clip, which is what the zero padding of the un-sharded conv reads); the F output frames are the interior ones.
static int tconv3_impl(const void* x, long long ldx, int B, int F, int HW, int Cin, const void* w, int Cout, const fz_epilogue_t* epi,
                       void* out, long long ldo, int force_block_n, int halo, cudaStream_t stream) {
  FZ_CHECK_ARG(x && w && out, "fz_tconv3: null pointer");
  FZ_CHECK_ARG(Cin % 8 == 0 && ldx % 8 == 0, "fz_tconv3: Cin/ldx must be multiples of 8");
  int bp = std::min(HW, 128);
  while (HW % bp) --bp;
  int bf = (bp == HW) ? std::min(F, 128 / bp) : 1;
  while (F % bf) --bf;
  TapGemmParams p;
  memset(&p, 0, sizeof(p));
  const int M = B * F * HW;
  const int rc0 = fill_epilogue(p, epi, M, Cout);
  if (rc0) return rc0;
  const int Fx = F + 2 * halo;
  {
    uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)HW, (uint64_t)Fx, (uint64_t)B};
    uint64_t strides[3] = {(uint64_t)ldx, (uint64_t)ldx * HW, (uint64_t)ldx * HW * Fx};
    uint32_t box[4] = {kBlockK, (uint32_t)bp, (uint32_t)bf, 1};
    if (int rc = encode_tmap_f16(&p.tmA, x, 4, dims, strides, box, true)) return rc;
  }
  p.a_rank = 4;
  for (int t = 0; t < 3; ++t) { p.tap_off[t][2] = t - 1 + halo; }
  p.rows_per_tile = bp * bf;
  p.m_tiles = M / p.rows_per_tile;
  const int bn = pick_block_n(p, Cout, force_block_n, p.m_tiles, 3 * ((Cin + kBlockK - 1) / kBlockK));
  {
    uint64_t dims[3] = {(uint64_t)Cin, (uint64_t)Cout, 3};
    uint64_t strides[2] = {(uint64_t)Cin, (uint64_t)Cin * Cout};
    uint32_t box[3] = {kBlockK, (uint32_t)bn, 1};
    if (int rc = encode_tmap_f16(&p.tmB, w, 3, dims, strides, box, true)) return rc;
  }
  p.M = M; p.rows_per_tile = bp * bf; p.a_box_bytes = p.rows_per_tile * 128;
  p.k_blocks = (Cin + kBlockK - 1) / kBlockK; p.num_taps = 3;
  p.m_tiles = M / p.rows_per_tile;
  p.ndecomp = 3; p.dimsz[0] = HW; p.dimsz[1] = F; p.dimsz[2] = B;
  p.out = static_cast<__half*>(out); p.ldo = ldo;
  return dispatch_tapgemm(p, Cout, bn, stream);
}

extern "C" int fz_tconv3_f16(const void* x, long long ldx, int B, int F, int HW, int Cin, const void* w, int Cout, const fz_epilogue_t* epi,
                             void* out, long long ldo, int force_block_n, cudaStream_t stream) {
  return tconv3_impl(x, ldx, B, F, HW, Cin, w, Cout, epi, out, ldo, force_block_n, 0, stream);
}

extern "C" int fz_tconv3_halo_f16(const void* x_ext, long long ldx, int B, int F, int HW, int Cin, const void* w, int Cout,
                                  const fz_epilogue_t* epi, void* out, long long ldo, int force_block_n, cudaStream_t stream) {
  return tconv3_impl(x_ext, ldx, B, F, HW, Cin, w, Cout, epi, out, ldo, force_block_n, 1, stream);
}
