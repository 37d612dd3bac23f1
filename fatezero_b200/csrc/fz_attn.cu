// fz_attn.cu — fused attention for the FateZero hot path (sm_90a: TMA + wgmma).
//
// One kernel computes  O = f(softmax(scale * Q K^T)) V  for
//   * the spatio-temporal self-attention (K/V of 0..n frames selected per query frame:
//     prompt_attention/attention_register.py:131-218, models/attention.py:366-398), and
//   * the text cross-attention (77 keys: attention_register.py:71-128),
// with the controller hook of attention_register.py:49-51 fused INLINE (no probability tensor in HBM unless it is the cache):
//   STORE      inversion: the fp16 probabilities are written once to the HBM map cache with TMA stores straight from the
//              swizzled P tile that also feeds the PV MMA (attention_store.py:81-93), optional fp16 running sum (:95-101)
//   REPLACE    edit, self-attention inside the replace window: P tile is TMA-loaded from the cache, QK^T/softmax skipped
//              (attention_util.py:80-92 without mask)
//   BLEND      edit, self-attention with a per-(frame,pixel) mask: rows with mask==0 take the cached row (:86-88)
//   CROSSEDIT  edit, cross-attention: Refine gather / Replace 77x77 / Reweight / alpha-lerp in registers (:130-131,213-253,282-286)
// The hook is chosen per row group (fz_attention_grouped_f16: K prompts of one clip in one CFG batch, each group with its own mode, mask,
// running sum and edit tables; fz_attention_grouped_slabs_f16: groups of different clips, each with its own cache slab to store into or
// read from); fz_attention_f16 is the one-group case.
// Hooked rows take two passes over the keys (max and sum first, then probabilities): the normalised fp16 P the reference stores and
// multiplies is reproduced exactly at its rounding point.  Rows that are neither stored nor edited take ONE pass with a running reference
// maximum (online softmax: p = exp2(s c - m_ref c) rounded to fp16 for PV, fp32 row sum l, O / l at the end; m_ref is raised, and O, l
// rescaled, only when a key block exceeds it by more than 2^8, so the rescale is rare and p stays far inside fp16 range).
//
// CTA = 128 query rows of one (frame, head); 9 warps: 0-7 = two consumer warpgroups (warpgroup w owns query rows [64 w, 64 w + 64):
// it issues the wgmma of S = Q K^T and O += P V for them, holds S and O in registers and runs the softmax and the controller hook),
// 8 = TMA producer.  Pipeline granularity = one ATOM of 64 keys.  smem: Q tile, a ring of K chunks / V^T atoms shared by both
// warpgroups, two P buffers per warpgroup (64 rows x 64 keys, swizzled) and two cached-P ("base") buffers for REPLACE / BLEND.
#include "fz_common.cuh"
#include "fz_wgmma.cuh"

#include <algorithm>
#include <cstring>

#include "../../include/fatezero_b200.h"

namespace fz {

constexpr int kMaxSlots = 4;
constexpr int kMaxBF = 64;          // fz_attention_f16
constexpr int kMaxBFGrouped = 128;  // fz_attention_grouped_f16: 8 prompts x CFG 2 x 8 frames
constexpr int kMaxGroups = FZ_ATTN_MAX_GROUPS;
constexpr int kAtomBytes = 128 * 128;  // 128 rows x 64 fp16
constexpr int kHalfAtom = 64 * 128;    // one warpgroup's 64 rows
constexpr int kMaxStages = 12;

struct AttnParams {
  CUtensorMap tmQ;      // (d, heads, S_q, BF)                 box (64, 1, 128, 1)
  CUtensorMap tmK;      // (d, heads, keys_per_slot, SRC)      box (64, 1, 64, 1)
  CUtensorMap tmVt;     // (keys_ld, d, heads, SRC)            box (64, 64 nd, 1, 1)
  // per group: the cache slab it writes (STORE) or reads (REPLACE / BLEND), (keys_ld_cache, slots, S_q, heads, Fc) box (64, 1, 64, 1, 1);
  // a group is never both, so one map per group
  CUtensorMap tmCache[FZ_ATTN_MAX_GROUPS];
  int S_q;              // queries per (frame, head)
  int keys_per_slot;    // S for self-attention, 77 for cross
  int n_slots;          // key/value frames per query frame (self: 1..4, cross: 1)
  int d, nd;            // head dim, number of 64-wide chunks
  int heads, F, BF;
  int ring_stages, ring_stage_bytes;
  float scale_log2;     // scale * log2(e)
  int src_index[kMaxSlots][kMaxBFGrouped];  // K/V source row (frame or text batch) per slot and query frame
  // controller: rows bf >= edit_bf_start form n_groups groups of group_rows rows; row bf belongs to group
  // g = (bf - edit_bf_start) / group_rows and stores / reads cache frame fc = (bf - edit_bf_start) % group_rows of its slab
  int edit_bf_start;
  int group_rows;       // Fc: rows per group (the base / store slabs are [Fc, heads, S_q, cache_ld])
  int n_groups;
  unsigned char row_group[kMaxBFGrouped];  // g of every row (0 for the rows before edit_bf_start)
  int has_base;         // some group is REPLACE / BLEND: the shared-memory plan holds the two cached-P tiles
  int g_row_mode[kMaxGroups];      // FZ_ATTN_* per group
  __half* g_acc[kMaxGroups];       // running sum [Fc, heads, S_q, acc_ld] fp16 or null (cross maps), per group
  const float* g_xedit[kMaxGroups];  // CROSSEDIT tables in device memory (fz_cross_edit_t layout), per group
  const float* g_mask[kMaxGroups];   // BLEND: [Fc, S_q] 1 = keep current row, 0 = take cached row, per group
  long long acc_ld;
  const __half* g_base_rows[FZ_ATTN_MAX_GROUPS];  // CROSSEDIT: cached source map [Fc, heads, S_q, base_ld], per group
  long long base_ld;
  __half* out;          // [BF*S_q, ldo], this head's columns start at head*d
  long long ldo;
  int causal;           // key n visible to query s only if n <= s
  int masked;           // keys_per_slot % 64 != 0 or causal: scores outside the valid keys are set to -inf
};
// a __grid_constant__ parameter block must stay within the classic 4 KiB kernel-parameter space
static_assert(sizeof(AttnParams) <= 4096, "AttnParams exceeds the 4 KiB kernel-parameter limit");

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

struct AtomInfo {
  int slot, k0, valid;
};
__device__ __forceinline__ AtomInfo atom_info(const AttnParams& p, int atoms_per_slot, int A) {
  AtomInfo a;
  if (p.n_slots == 1) {
    a.slot = 0;
    a.k0 = A * 64;
  } else {
    a.slot = A / atoms_per_slot;
    a.k0 = (A - a.slot * atoms_per_slot) * 64;
  }
  a.valid = min(64, p.keys_per_slot - a.k0);
  return a;
}

// O[64 x 64 NCH] (+)= P[64 x 64 keys] V[64 keys x 64 NCH]: the V^T atom holds 64 NCH rows (TMA zero-fills the rows beyond d), so every
// chunk is one fixed-shape wgmma and the issue sequence has no data-dependent branch (which would serialise the asynchronous MMAs).
template <int NCH>
__device__ __forceinline__ void pv_mma(float (&o)[32 * NCH], uint64_t da, uint64_t db, uint32_t accumulate) {
#pragma unroll
  for (int ch = 0; ch < NCH; ++ch) {
    const uint64_t dbc = db + static_cast<uint32_t>((ch * 64 * 128) >> 4);
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_f16<64>(o + 32 * ch, da + 2 * k, dbc + 2 * k, (accumulate | k) ? 1u : 0u);
  }
}

constexpr float kRescaleThreshold = 8.0f;  // log2 units: un-hooked rows raise their reference maximum only past 2^8 (fp16 P stays finite)

// NCH = number of 64-wide chunks of the head dim (1..3): sizes the O accumulator (32 NCH registers per thread).
template <int NCH>
__global__ void __launch_bounds__(288, 1) attn_kernel(const __grid_constant__ AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  pdl_launch_dependents();
  const int q0 = blockIdx.x * 128;
  const int head = blockIdx.y;
  const int bf = blockIdx.z;
  const int grp = p.row_group[bf];
  const int fc = bf - p.edit_bf_start - grp * p.group_rows;
  const bool edited = bf >= p.edit_bf_start && p.g_row_mode[grp] != FZ_ATTN_NONE;
  const int row_mode = edited ? p.g_row_mode[grp] : FZ_ATTN_NONE;
  const bool replace = row_mode == FZ_ATTN_REPLACE;
  const bool blend = row_mode == FZ_ATTN_BLEND;
  const bool exact = row_mode != FZ_ATTN_NONE;  // pass 1 accumulates the sum, pass 2 emits normalised probabilities

  uint8_t* s_q = smem;
  uint8_t* s_ring = s_q + p.nd * kAtomBytes;
  uint8_t* s_p = s_ring + p.ring_stages * p.ring_stage_bytes;  // [warpgroup][2] x 8 KiB
  uint8_t* s_base = s_p + 4 * kHalfAtom;                       // 2 x 16 KiB (REPLACE / BLEND only)
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_base + (p.has_base ? 2 * kAtomBytes : 0));
  uint64_t* ring_full = bars;                   // [kMaxStages]
  uint64_t* ring_empty = bars + kMaxStages;     // [kMaxStages]
  uint64_t* q_full = bars + 2 * kMaxStages;
  uint64_t* base_full = q_full + 1;             // [2]
  uint64_t* base_empty = base_full + 2;         // [2]

  const int atoms_per_slot = (p.keys_per_slot + 63) / 64;
  const int n_atoms = atoms_per_slot * p.n_slots;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmQ);
    tma_prefetch_desc(&p.tmK);
    tma_prefetch_desc(&p.tmVt);
    for (int s = 0; s < p.ring_stages; ++s) {
      mbar_init(&ring_full[s], 1);
      mbar_init(&ring_empty[s], 8);  // every consumer warp releases every stage
    }
    mbar_init(q_full, 1);
    for (int b = 0; b < 2; ++b) {
      mbar_init(&base_full[b], 1);
      mbar_init(&base_empty[b], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();  // prologue above overlaps the previous kernel's tail (programmatic dependent launch)

  if (warp == 8) {
    // =========================================== TMA producer ===========================================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      auto advance = [&]() { if (++stage == p.ring_stages) { stage = 0; phase ^= 1; } };
      auto load_k = [&](int A) {
        const AtomInfo ai = atom_info(p, atoms_per_slot, A);
        for (int c = 0; c < p.nd; ++c) {
          mbar_wait(&ring_empty[stage], phase ^ 1);
          mbar_expect_tx(&ring_full[stage], 64 * 128);
          tma_load_4d(s_ring + stage * p.ring_stage_bytes, &p.tmK, &ring_full[stage], c * 64, head, ai.k0, p.src_index[ai.slot][bf]);
          advance();
        }
      };
      auto load_v = [&](int A) {
        const AtomInfo ai = atom_info(p, atoms_per_slot, A);
        mbar_wait(&ring_empty[stage], phase ^ 1);
        mbar_expect_tx(&ring_full[stage], NCH * 64 * 128);
        tma_load_4d(s_ring + stage * p.ring_stage_bytes, &p.tmVt, &ring_full[stage], ai.k0, 0, head, p.src_index[ai.slot][bf]);
        advance();
      };
      auto load_base = [&](int A) {
        const AtomInfo ai = atom_info(p, atoms_per_slot, A);
        const int b = A & 1;
        mbar_wait(&base_empty[b], ((A >> 1) & 1) ^ 1);
        mbar_expect_tx(&base_full[b], kAtomBytes);
        for (int h = 0; h < 2; ++h)
          tma_load_5d(s_base + b * kAtomBytes + h * kHalfAtom, &p.tmCache[grp], &base_full[b], ai.k0, ai.slot, q0 + 64 * h, head, fc);
      };
      if (!replace) {
        mbar_expect_tx(q_full, p.nd * kAtomBytes);
        for (int c = 0; c < p.nd; ++c) tma_load_4d(s_q + c * kAtomBytes, &p.tmQ, q_full, c * 64, head, q0, bf);
        if (exact)
          for (int A = 0; A < n_atoms; ++A) load_k(A);  // pass 1
        for (int A = 0; A < n_atoms; ++A) {             // pass 2 (the only pass of un-hooked rows)
          load_k(A);
          if (blend) load_base(A);
          load_v(A);
        }
      } else {
        for (int A = 0; A < n_atoms; ++A) {
          load_base(A);
          load_v(A);
        }
      }
    }
    return;
  }

  // =========================================== consumer warpgroups ===========================================
  const int wg = warp >> 2;
  const int st = threadIdx.x & 127;
  const int warp_in = warp & 3;
  // fragment of this thread: rows rl[h] = 16 warp_in + lane / 4 + 8 h of the warpgroup's 64, key / output column 8 i + c_base + j
  // at register 4 i + 2 h + j (fz_wgmma.cuh)
  const int c_base = 2 * (lane & 3);
  int rl[2], q[2];
  bool row_ok[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    rl[h] = 16 * warp_in + (lane >> 2) + 8 * h;
    q[h] = q0 + 64 * wg + rl[h];
    row_ok[h] = q[h] < p.S_q;
  }
  const uint64_t desc0 = wgmma_desc_k_sw128(smem_u32(smem));
  auto desc_of = [&](const uint8_t* ptr) { return desc0 + static_cast<uint32_t>((ptr - smem) >> 4); };
  int stage = 0;
  uint32_t phase = 0;
  auto release = [&]() {
    __syncwarp();
    if (lane == 0) mbar_arrive(&ring_empty[stage]);
    if (++stage == p.ring_stages) { stage = 0; phase ^= 1; }
  };
  const float sc2 = p.scale_log2;
  // S[64 x 64 keys] = Q K^T of atom A (head-dim columns beyond d are TMA zero fill), keys outside the valid range set to -inf
  auto scores = [&](float (&s)[32], int A) {
    for (int c = 0; c < p.nd; ++c) {
      mbar_wait(&ring_full[stage], phase);
      const uint64_t da = desc_of(s_q + c * kAtomBytes + wg * kHalfAtom);
      const uint64_t db = desc_of(s_ring + stage * p.ring_stage_bytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_f16<64>(s, da + 2 * k, db + 2 * k, (c | k) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      release();
    }
    if (p.masked) {
      const AtomInfo ai = atom_info(p, atoms_per_slot, A);
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const int e = 8 * i + c_base + j;
            if (e >= ai.valid || (p.causal && ai.k0 + e > q[h])) s[4 * i + 2 * h + j] = -INFINITY;
          }
    }
  };

  float o[32 * NCH];
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  if (!replace) {
    mbar_wait(q_full, 0);
    // ------------------------------ pass 1 (hooked rows): row max and sum of exponentials ------------------------------
    for (int A = 0; exact && A < n_atoms; ++A) {
      float s[32];
      scores(s, A);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float cm = -INFINITY;
#pragma unroll
        for (int i = 0; i < 8; ++i) cm = fmaxf(cm, fmaxf(s[4 * i + 2 * h], s[4 * i + 2 * h + 1]));
        cm = quad_max(cm);
        const float m_new = fmaxf(m_run[h], cm);
        if (m_new > -INFINITY) {
          const float mb = m_new * sc2;
          float a = 0.f;
#pragma unroll
          for (int i = 0; i < 8; ++i) a += ex2(fmaf(s[4 * i + 2 * h], sc2, -mb)) + ex2(fmaf(s[4 * i + 2 * h + 1], sc2, -mb));
          l_run[h] = l_run[h] * ex2((m_run[h] - m_new) * sc2) + a;  // per-thread partial: the quad shares m_run
        }
        m_run[h] = m_new;
      }
    }
    float inv_l[2], mb2[2], mrow[2];
    // the group's acc / xedit pointers are re-read from the parameter block where they are used (keeping them live spills at d > 128)
    const bool has_acc = edited && p.g_acc[grp] != nullptr;
    const bool row_ops = row_mode == FZ_ATTN_CROSSEDIT || has_acc;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      inv_l[h] = exact ? 1.0f / quad_sum(l_run[h]) : 1.0f;
      mb2[h] = exact ? m_run[h] * sc2 : 0.f;
      mrow[h] = blend ? p.g_mask[grp][static_cast<long long>(fc) * p.S_q + min(q[h], p.S_q - 1)] : 1.f;
      l_run[h] = 0.f;
    }
    // ------------------------ pass 2 (the only pass of un-hooked rows): probabilities -> P tile (-> cache) -> O += P V ------------------------
    for (int A = 0; A < n_atoms; ++A) {
      const AtomInfo ai = atom_info(p, atoms_per_slot, A);
      float pv[32];
      scores(pv, A);
      if (!exact) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float cm = -INFINITY;
#pragma unroll
          for (int i = 0; i < 8; ++i) cm = fmaxf(cm, fmaxf(pv[4 * i + 2 * h], pv[4 * i + 2 * h + 1]));
          cm = quad_max(cm);
          if (m_run[h] == -INFINITY ? cm > -INFINITY : (cm - m_run[h]) * sc2 > kRescaleThreshold) {
            // the PV of the previous atom has completed (wgmma_wait below): O and l of this row are rescaled to the new reference
            const float f = ex2((m_run[h] - cm) * sc2);
            l_run[h] *= f;
            if (A > 0) {
#pragma unroll
              for (int i = 0; i < 8 * NCH; ++i) { o[4 * i + 2 * h] *= f; o[4 * i + 2 * h + 1] *= f; }
            }
            m_run[h] = cm;
            mb2[h] = cm * sc2;
          }
        }
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            float& x = pv[4 * i + 2 * h + j];
            x = ex2(fmaf(x, sc2, -mb2[h]));
            if (exact) x *= inv_l[h];
            else l_run[h] += x;
          }
      if (row_ops) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          // key index n = ai.k0 + 8 i + c_base + j (single slot).  cur = fp16(p); optional running sum; optional edit (in fp32, one rounding)
          const long long rbase = ((static_cast<long long>(fc) * p.heads + head) * p.S_q + min(q[h], p.S_q - 1));
          if (has_acc && row_ok[h]) {
            __half* ap = p.g_acc[grp] + rbase * p.acc_ld;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int n = ai.k0 + 8 * i + c_base;
              if (n < p.acc_ld) {
                const float2 a = __half22float2(*reinterpret_cast<__half2*>(ap + n));
                const float c0 = __half2float(__float2half_rn(pv[4 * i + 2 * h])), c1 = __half2float(__float2half_rn(pv[4 * i + 2 * h + 1]));
                *reinterpret_cast<__half2*>(ap + n) = __floats2half2_rn(a.x + c0, a.y + c1);
              }
            }
          }
          if (row_mode == FZ_ATTN_CROSSEDIT) {
            const __half* brow = p.g_base_rows[grp] + rbase * p.base_ld;
            const float* xe = p.g_xedit[grp];
            const int xmode = static_cast<int>(xe[0]);  // 0 refine, 1 replace
            const float* x_alpha = xe + 8;              // [80] cross_replace_alpha of this step
            const float* x_eq = xe + 8 + 80;            // [80] equalizer (1 when absent)
            const float* x_a = xe + 8 + 160;            // [80] refine alphas
            const float* x_map = xe + 8 + 240;          // [80] refine mapper (as float)
            const float* x_M = xe + 8 + 320;            // [80][80] replace matrix M[w][n]
            float rr[16];
            if (xmode == 1) {
#pragma unroll
              for (int e = 0; e < 16; ++e) rr[e] = 0.f;
              for (int w = 0; w < p.keys_per_slot; ++w) {
                const float bw = __half2float(brow[w]);
                const float* mrow_p = x_M + w * 80;
#pragma unroll
                for (int i = 0; i < 8; ++i)
#pragma unroll
                  for (int j = 0; j < 2; ++j) {
                    const int n = ai.k0 + 8 * i + c_base + j;
                    if (n < 80) rr[2 * i + j] += bw * __ldg(mrow_p + n);
                  }
              }
            }
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
              for (int j = 0; j < 2; ++j) {
                const int n = ai.k0 + 8 * i + c_base + j;
                if (n < p.keys_per_slot) {
                  float& x = pv[4 * i + 2 * h + j];
                  const float cur = __half2float(__float2half_rn(x));
                  float R;
                  if (xmode == 1) R = rr[2 * i + j];
                  else {
                    int mi = static_cast<int>(__ldg(x_map + n));
                    if (mi < 0) mi += p.keys_per_slot;  // python negative index (masked by a[n] == 0)
                    const float an = __ldg(x_a + n);
                    R = __half2float(brow[mi]) * an + cur * (1.f - an);
                  }
                  R *= __ldg(x_eq + n);
                  const float al = __ldg(x_alpha + n);
                  x = R * al + (1.f - al) * cur;
                }
              }
          }
        }
      }
      // P buffer pb of this warpgroup: its PV two atoms ago is complete (wgmma_wait below); for STORE its TMA store must be done reading
      const int pb = A & 1;
      uint8_t* ptile = s_p + (wg * 2 + pb) * kHalfAtom;
      if (row_mode == FZ_ATTN_STORE) {
        if (st == 0) tma_store_wait_read<1>();
        named_bar_sync(1 + wg, 128);
      }
      // swizzled stores: 16-byte chunk i of row r lands at chunk (i ^ (r & 7))
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 8; ++i)
          *reinterpret_cast<uint32_t*>(ptile + rl[h] * 128 + ((i ^ (rl[h] & 7)) << 4) + c_base * 2) =
              pack_half2(pv[4 * i + 2 * h], pv[4 * i + 2 * h + 1]);
      if (blend) {
        mbar_wait(&base_full[A & 1], (A >> 1) & 1);
        const uint8_t* btile = s_base + (A & 1) * kAtomBytes + wg * kHalfAtom;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (mrow[h] == 0.f) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int off = rl[h] * 128 + ((i ^ (rl[h] & 7)) << 4) + c_base * 2;
              *reinterpret_cast<uint32_t*>(ptile + off) = *reinterpret_cast<const uint32_t*>(btile + off);
            }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&base_empty[A & 1]);
      }
      fence_proxy_async_smem();
      named_bar_sync(1 + wg, 128);
      if (row_mode == FZ_ATTN_STORE && st == 0) {
        tma_store_5d(&p.tmCache[grp], ptile, ai.k0, ai.slot, q0 + 64 * wg, head, fc);
        tma_store_commit();
      }
      mbar_wait(&ring_full[stage], phase);
      wgmma_fence();
      pv_mma<NCH>(o, desc_of(ptile), desc_of(s_ring + stage * p.ring_stage_bytes), A ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      release();
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) l_run[h] = quad_sum(l_run[h]);
  } else {
    for (int A = 0; A < n_atoms; ++A) {
      mbar_wait(&base_full[A & 1], (A >> 1) & 1);
      mbar_wait(&ring_full[stage], phase);
      wgmma_fence();
      pv_mma<NCH>(o, desc_of(s_base + (A & 1) * kAtomBytes + wg * kHalfAtom), desc_of(s_ring + stage * p.ring_stage_bytes), A ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      release();
      __syncwarp();
      if (lane == 0) mbar_arrive(&base_empty[A & 1]);
    }
  }
  // ------------------------------ epilogue: O (registers) -> fp16 -> global ------------------------------
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (!row_ok[h]) continue;
    const float o_scale = (!replace && !exact) ? (1.0f / l_run[h]) : 1.0f;
    __half* orow = p.out + (static_cast<long long>(bf) * p.S_q + q[h]) * p.ldo + head * p.d;
#pragma unroll
    for (int i = 0; i < 8 * NCH; ++i) {
      const int c = 8 * i + c_base;
      if (c < p.d) *reinterpret_cast<uint32_t*>(orow + c) = pack_half2(o[4 * i + 2 * h] * o_scale, o[4 * i + 2 * h + 1] * o_scale);
    }
  }
  if (row_mode == FZ_ATTN_STORE && st == 0) tma_store_wait_all<0>();
}

}  // namespace fz

using namespace fz;

static int encode_cache_map(CUtensorMap* tm, const void* base, int keys_ld_slot, int n_slots, int S_q, int heads, int Fc, long long row_ld) {
  // cache slab [Fc, heads, S_q, row_ld] fp16; a row holds n_slots runs of keys_ld_slot keys (self) or one run (cross)
  uint64_t dims[5] = {(uint64_t)keys_ld_slot, (uint64_t)n_slots, (uint64_t)S_q, (uint64_t)heads, (uint64_t)Fc};
  uint64_t strides[4] = {(uint64_t)keys_ld_slot, (uint64_t)row_ld, (uint64_t)row_ld * S_q, (uint64_t)row_ld * S_q * heads};
  uint32_t box[5] = {64, 1, 64, 1, 1};
  return encode_tmap_f16(tm, base, 5, dims, strides, box, true);
}

// One launcher for every entry.  `g` carries the controller hook per row group; rows [edit_bf_start, BF) form g->n_groups groups of
// group_rows rows.  Group k stores into / reads the slab [group_rows, heads, S_q, cache_ld] slabs->store[k] / slabs->base[k], or the slab
// of `a` where that is NULL (slabs == NULL: every group uses the slabs of `a`).
static int attention_launch(const fz_attn_args_t* a, const fz_attn_groups_t* g, const fz_attn_slabs_t* slabs, int group_rows,
                            cudaStream_t stream) {
  AttnParams p;
  memset(&p, 0, sizeof(p));
  p.S_q = a->S_q; p.keys_per_slot = a->keys_per_slot; p.n_slots = a->n_slots;
  p.d = a->d; p.nd = (a->d + 63) / 64;
  p.heads = a->heads; p.F = a->F; p.BF = a->BF;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  for (int s = 0; s < a->n_slots; ++s)
    for (int i = 0; i < a->BF; ++i) p.src_index[s][i] = a->src_index[s * a->BF + i];
  p.edit_bf_start = a->edit_bf_start;
  p.group_rows = std::max(1, group_rows);
  p.n_groups = g->n_groups;
  for (int i = std::max(0, a->edit_bf_start); i < a->BF; ++i) p.row_group[i] = static_cast<unsigned char>((i - a->edit_bf_start) / p.group_rows);
  bool any_slab = false, any_self_base = false, any_hook = false;
  const void* store_of[kMaxGroups];
  const void* base_of[kMaxGroups];
  for (int k = 0; k < g->n_groups; ++k) {
    const fz_attn_group_t& gr = g->g[k];
    store_of[k] = slabs && slabs->store[k] ? slabs->store[k] : a->store;
    base_of[k] = slabs && slabs->base[k] ? slabs->base[k] : a->base;
    FZ_CHECK_ARG(gr.row_mode >= FZ_ATTN_NONE && gr.row_mode <= FZ_ATTN_CROSSEDIT, "fz_attention: group %d: row_mode %d unknown", k, gr.row_mode);
    p.g_row_mode[k] = gr.row_mode;
    p.g_acc[k] = static_cast<__half*>(gr.acc);
    p.g_xedit[k] = gr.xedit;
    p.g_mask[k] = gr.mask;
    p.g_base_rows[k] = static_cast<const __half*>(base_of[k]);
    const bool reads_base = gr.row_mode == FZ_ATTN_REPLACE || gr.row_mode == FZ_ATTN_BLEND || gr.row_mode == FZ_ATTN_CROSSEDIT;
    if (gr.row_mode == FZ_ATTN_STORE) FZ_CHECK_ARG(store_of[k], "fz_attention: STORE needs a cache slab (group %d)", k);
    if (reads_base) FZ_CHECK_ARG(base_of[k], "fz_attention: REPLACE/BLEND/CROSSEDIT need the cached source map (group %d)", k);
    any_slab |= store_of[k] != nullptr || base_of[k] != nullptr;
    any_self_base |= gr.row_mode == FZ_ATTN_REPLACE || gr.row_mode == FZ_ATTN_BLEND;
    any_hook |= gr.row_mode != FZ_ATTN_NONE || gr.acc != nullptr;
    if (gr.row_mode == FZ_ATTN_BLEND) FZ_CHECK_ARG(gr.mask, "fz_attention: BLEND needs a mask");
    if (gr.row_mode == FZ_ATTN_CROSSEDIT) FZ_CHECK_ARG(gr.xedit && a->n_slots == 1 && a->keys_per_slot <= 80, "fz_attention: CROSSEDIT needs tables, one slot, <= 80 keys");
    if (gr.acc) FZ_CHECK_ARG(a->n_slots == 1 && a->acc_ld % 8 == 0, "fz_attention: running sum only for single-slot maps");
  }
  p.has_base = any_self_base;
  p.acc_ld = a->acc_ld;
  p.base_ld = a->cache_ld;
  p.out = static_cast<__half*>(a->out); p.ldo = a->ldo;
  p.causal = a->causal;
  p.masked = a->causal || a->keys_per_slot % 64 != 0;
  if (a->causal) FZ_CHECK_ARG(a->n_slots == 1 && !any_hook, "fz_attention: causal masking needs one slot and no controller hook");
  const int Fc = group_rows;
  if (any_slab || a->store || a->base)
    FZ_CHECK_ARG(a->cache_ld > 0 && a->cache_ld % a->n_slots == 0 && a->cache_ld / a->n_slots >= a->keys_per_slot,
                 "fz_attention: cache_ld=%lld must split into n_slots=%d runs of >= keys_per_slot=%d keys", a->cache_ld, a->n_slots,
                 a->keys_per_slot);
  {
    uint64_t dims[4] = {(uint64_t)a->d, (uint64_t)a->heads, (uint64_t)a->S_q, (uint64_t)a->BF};
    uint64_t strides[3] = {(uint64_t)a->d, (uint64_t)a->ldq, (uint64_t)a->ldq * a->S_q};
    uint32_t box[4] = {64, 1, 128, 1};
    if (int rc = encode_tmap_f16(&p.tmQ, a->q, 4, dims, strides, box, true)) return rc;
  }
  {
    uint64_t dims[4] = {(uint64_t)a->d, (uint64_t)a->heads, (uint64_t)a->keys_per_slot, (uint64_t)a->n_src};
    uint64_t strides[3] = {(uint64_t)a->d, (uint64_t)a->ldk, (uint64_t)a->ldk * a->keys_per_slot};
    uint32_t box[4] = {64, 1, 64, 1};
    if (int rc = encode_tmap_f16(&p.tmK, a->k, 4, dims, strides, box, true)) return rc;
  }
  {
    uint64_t dims[4] = {(uint64_t)a->keys_per_slot, (uint64_t)a->d, (uint64_t)a->heads, (uint64_t)a->n_src};
    uint64_t strides[3] = {(uint64_t)a->vt_ld, (uint64_t)a->vt_ld * a->d, (uint64_t)a->vt_ld * a->d * a->heads};
    uint32_t box[4] = {64, (uint32_t)(64 * p.nd), 1, 1};  // rows beyond d: zero fill (fixed-shape PV wgmma)
    if (int rc = encode_tmap_f16(&p.tmVt, a->vt, 4, dims, strides, box, true)) return rc;
  }
  // cache geometry: a row of the slab is n_slots * keys_ld_slot wide, keys_ld_slot = cache_ld / n_slots.  Groups that share a slab share
  // its encoded map; groups without a TMA-accessed slab (NONE, CROSSEDIT) get a placeholder that is never used.
  for (int k = 0; k < kMaxGroups; ++k) {
    const int mode = k < g->n_groups ? g->g[k].row_mode : FZ_ATTN_NONE;
    const void* slab = mode == FZ_ATTN_STORE ? store_of[k] : (mode == FZ_ATTN_REPLACE || mode == FZ_ATTN_BLEND) ? base_of[k] : nullptr;
    int same = -1;
    for (int j = 0; j < k && slab; ++j) {
      const int mj = g->g[j].row_mode;
      const void* sj = mj == FZ_ATTN_STORE ? store_of[j] : (mj == FZ_ATTN_REPLACE || mj == FZ_ATTN_BLEND) ? base_of[j] : nullptr;
      if (sj == slab) { same = j; break; }
    }
    if (!slab) {
      p.tmCache[k] = p.tmQ;
    } else if (same >= 0) {
      p.tmCache[k] = p.tmCache[same];
    } else if (int rc = encode_cache_map(&p.tmCache[k], slab, (int)(a->cache_ld / a->n_slots), a->n_slots, a->S_q, a->heads, Fc, a->cache_ld)) {
      return rc;
    }
  }
  // shared memory plan: Q + ring + 4 half P tiles (+ 2 base tiles) + barriers
  const int stage_bytes = p.nd * 64 * 128;
  const int fixed = p.nd * kAtomBytes + 4 * kHalfAtom + (p.has_base ? 2 * kAtomBytes : 0) + 1024 + 512;
  int stages = kMaxStages;
  while (stages > 2 && fixed + stages * stage_bytes > 227 * 1024) --stages;
  FZ_CHECK_ARG(fixed + stages * stage_bytes <= 227 * 1024, "fz_attention: shared memory plan does not fit (d=%d)", a->d);
  p.ring_stages = stages; p.ring_stage_bytes = stage_bytes;
  const int smem = fixed + stages * stage_bytes;
  static bool configured = false;
  if (!configured) {
    FZ_CUDA(cudaFuncSetAttribute(attn_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    FZ_CUDA(cudaFuncSetAttribute(attn_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    FZ_CUDA(cudaFuncSetAttribute(attn_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    configured = true;
  }
  dim3 grid((a->S_q + 127) / 128, a->heads, a->BF);
  auto kernel = p.nd == 1 ? attn_kernel<1> : p.nd == 2 ? attn_kernel<2> : attn_kernel<3>;
  FZ_CUDA(launch_pdl(kernel, grid, dim3(288), smem, stream, p));
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}

static int check_common(const fz_attn_args_t* a, int max_bf) {
  if (int rc = check_single_device()) return rc;
  FZ_CHECK_ARG(a && a->q && a->k && a->vt && a->out, "fz_attention: null pointer");
  FZ_CHECK_ARG(a->d % 8 == 0 && a->d >= 8 && a->d <= 192, "fz_attention: head dim %d unsupported", a->d);
  FZ_CHECK_ARG(a->n_slots >= 1 && a->n_slots <= kMaxSlots && a->BF <= max_bf, "fz_attention: n_slots=%d BF=%d unsupported", a->n_slots, a->BF);
  FZ_CHECK_ARG(a->ldq % 8 == 0 && a->ldk % 8 == 0 && a->vt_ld % 8 == 0 && a->ldo % 8 == 0, "fz_attention: leading dims must be multiples of 8");
  FZ_CHECK_ARG(a->keys_per_slot >= 1 && a->keys_per_slot <= a->vt_ld, "fz_attention: keys_per_slot > vt_ld");
  return FZ_OK;
}

extern "C" int fz_attention_f16(const fz_attn_args_t* a, cudaStream_t stream) {
  if (int rc = check_common(a, kMaxBF)) return rc;
  fz_attn_groups_t g;
  memset(&g, 0, sizeof(g));
  g.n_groups = 1;
  g.g[0].row_mode = a->row_mode;
  g.g[0].xedit = a->xedit;
  g.g[0].mask = a->mask;
  g.g[0].acc = a->acc;
  return attention_launch(a, &g, nullptr, a->BF - a->edit_bf_start, stream);
}

extern "C" int fz_attention_grouped_slabs_f16(const fz_attn_args_t* a, const fz_attn_groups_t* g, const fz_attn_slabs_t* slabs,
                                              cudaStream_t stream) {
  if (int rc = check_common(a, kMaxBFGrouped)) return rc;
  FZ_CHECK_ARG(g && g->n_groups >= 1 && g->n_groups <= kMaxGroups, "fz_attention_grouped: n_groups=%d unsupported (1..%d)", g ? g->n_groups : 0,
               kMaxGroups);
  FZ_CHECK_ARG(a->F >= 1 && a->edit_bf_start >= 0 && a->BF - a->edit_bf_start == g->n_groups * a->F,
               "fz_attention_grouped: BF - edit_bf_start = %d rows must be n_groups * F = %d * %d", a->BF - a->edit_bf_start, g->n_groups, a->F);
  return attention_launch(a, g, slabs, a->F, stream);
}

extern "C" int fz_attention_grouped_f16(const fz_attn_args_t* a, const fz_attn_groups_t* g, cudaStream_t stream) {
  return fz_attention_grouped_slabs_f16(a, g, nullptr, stream);
}
