// fz_p2p.cu — frame-sharded execution over the GPUs of one NVSwitch box: peer-memory exchange kernels.
//
// The frames of ONE clip are split over the ranks (one process per GPU).  Every op of the UNet forward is per-frame except
//   (1) the sparse-causal self-attention reading K / V of other frames        (attention_register.py:162-193),
//   (2) the joint-frame GroupNorm statistics                                  (resnet.py:338,369; unet_3d_condition.py:439),
//   (3) the temporal Conv1d(k=3) over frames (LoRA down / up, full conv)      (resnet.py:72-78, lora.py:46-54),
//   (4) the temporal attention over frames                                    (models/attention.py:327-337).
// All four are served by ONE primitive over a symmetric arena (a cudaMalloc'd slab per rank, mapped into every peer with CUDA IPC, same
// offsets everywhere): the producer PUSHES 2-D segments straight into the consumers' buffers with 16-byte stores over NVLink and raises
// a flag in the consumer's memory (system-scope release) from the last CTA that finished writing to that consumer; the consumer runs a
// one-warp kernel that spins on its local flags (system-scope acquire) and clears them — it is their only reader, so no sequence
// numbers are needed and the same launch sequence can sit in a CUDA graph.  Every exchange site owns its buffers and flags; a site is
// reused one UNet forward later, by which time every rank has consumed it (each forward contains all-to-all GroupNorm exchanges that
// order all ranks).  No NCCL call sits on the data path.
#include "fz_common.cuh"

#include <algorithm>
#include <cstring>

#include "../../include/fatezero_b200.h"

namespace fz {

constexpr int kP2PMaxSegs = 96;  // 4.7 KiB of kernel parameters (CUDA >= 12.1 allows 32 KiB)
constexpr int kP2PMaxDst = 16;
#ifndef FZ_P2P_TIMEOUT_NS
#define FZ_P2P_TIMEOUT_NS 30000000000ull  // a peer that never arrives becomes a trap after 30 s, not a hung box
#endif

struct P2PSeg {
  const uint8_t* src;
  uint8_t* dst;
  long long src_pitch, dst_pitch;
  int rows, row_bytes;  // row_bytes % 16 == 0
  int dst_slot;         // index into flags / counters, -1 = local copy without a flag
};
struct P2PPushParams {
  P2PSeg seg[kP2PMaxSegs];
  int n_segs;
  int n_dst;
  unsigned* flag[kP2PMaxDst];  // flag word in the DESTINATION rank's arena (peer pointer)
  unsigned* counter;           // local arrival counter (zero between launches)
  unsigned* wait_flags;        // local flag words of this site (32, one per source rank), or null
  unsigned wait_mask;          // sources this rank expects data from at this site
};

__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void spin_until_raised(unsigned* flag, const char* what, int who) {
  const uint64_t t0 = global_timer_ns();
  unsigned spins = 0;
  while (ld_acquire_sys(flag) == 0u) {
    if ((++spins & 0x3ff) == 0 && global_timer_ns() - t0 > FZ_P2P_TIMEOUT_NS) {
      printf("fz: %s of peer %d never arrived (frame-sharded exchange)\n", what, who);
      __trap();
    }
  }
  *flag = 0u;  // this thread is the flag's only reader
}

// Exchange = push + wait in ONE launch: every CTA copies its share of the segments into the peers (16-byte stores over NVLink); the CTA
// that arrives last raises the flags of all destinations (system-scope release after a system fence) and then waits for this rank's own
// incoming flags, so that the next kernel of the stream (programmatic dependent launch: griddepcontrol.wait = completion of this grid)
// finds the neighbours' data in place.  Raising before waiting makes the exchange deadlock-free.
__global__ void __launch_bounds__(256) p2p_push_kernel(const __grid_constant__ P2PPushParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const P2PSeg& s = p.seg[blockIdx.y];
  const int vec_per_row = s.row_bytes >> 4;
  const long long total = static_cast<long long>(s.rows) * vec_per_row;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / vec_per_row;
    const int c = static_cast<int>(i - r * vec_per_row);
    const uint4 v = *reinterpret_cast<const uint4*>(s.src + r * s.src_pitch + (static_cast<long long>(c) << 4));
    *reinterpret_cast<uint4*>(s.dst + r * s.dst_pitch + (static_cast<long long>(c) << 4)) = v;
  }
  __threadfence_system();  // this thread's peer stores are performed before the arrival below
  __syncthreads();
  __shared__ bool s_last;
  if (threadIdx.x == 0) s_last = atomicAdd(p.counter, 1u) == gridDim.x * gridDim.y - 1u;
  __syncthreads();
  if (!s_last) return;
  if (threadIdx.x == 0) *p.counter = 0;  // ready for the next launch (stream order)
  __threadfence_system();
  if (threadIdx.x < p.n_dst) st_release_sys(p.flag[threadIdx.x], 1u);
  if (p.wait_flags && threadIdx.x < 32 && ((p.wait_mask >> threadIdx.x) & 1u)) spin_until_raised(p.wait_flags + threadIdx.x, "data", threadIdx.x);
}

// One warp: lane i (bit i of mask) spins until its flag is raised, then clears it.
__global__ void p2p_wait_kernel(unsigned* flags, unsigned mask) {
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x;
  if (lane < 32 && ((mask >> lane) & 1u)) spin_until_raised(flags + lane, "data", lane);
}

// GroupNorm statistics exchange in ONE single-CTA launch, low-latency ("LL") protocol: every per-image (sum, sumsq) pair travels as two
// 8-byte words {value bits, epoch} written straight into the peers' inboxes — an aligned 8-byte store is single-copy atomic, so each
// word carries its own validity and NO system fence or separate flag is needed (the fence pair + flag round trip of the generic exchange
// cost 10-20 us per GroupNorm at 8 GPUs; this is one NVLink store latency).  The epoch is a per-site counter in local device memory that
// every rank advances once per use (all ranks execute the same launch sequence), so the protocol is replay-safe inside CUDA graphs.
// The receiver polls its own inbox, adds the peers' statistics to the local ones and leaves the fp64 total of every statistics set in the
// slot of its first local image of `totals` (the layout fz_groupnorm_apply_sums64_f16 consumes; the other slots of the set are zeroed).  The
// totals stay in fp64, as the single-GPU apply keeps its fp64 sum of the per-image fp32 sums: a total rounded to fp32 moves the mean of a
// constant group by up to 2^-24 |mean|, which rstd = eps^-1/2 turns into ~100 fp16 ulps of a small beta.
// inbox: [world][NB * G][2] uint2 in this rank's arena (slot `me` unused); peer_inbox[r]: rank r's inbox slot for THIS rank.
struct GnXchgParams {
  uint2* peer_inbox[32];
  const uint2* inbox;    // local
  unsigned* epoch;       // local per-site use counter
  const float2* sums;    // [NB * G] this rank's per-image (sum, sumsq)
  double2* totals;       // [NB * G] out: set totals in the first image of each set, 0 elsewhere
  int NB, F_loc, G, world, me;
};
__device__ __forceinline__ uint2 ld_relaxed_sys_v2(const uint2* p) {
  uint2 v;
  asm volatile("ld.relaxed.sys.global.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_sys_v2(uint2* p, uint2 v) {
  asm volatile("st.relaxed.sys.global.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(v.x), "r"(v.y) : "memory");
}
__global__ void __launch_bounds__(1024) gn_combine_kernel(const __grid_constant__ GnXchgParams p) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ double gx_smem[];  // [NB * G][2]
  const int n = p.NB * p.G;
  const unsigned ep = *p.epoch + 1u;
  const int i = threadIdx.x;
  double sa = 0.0, sb = 0.0;
  if (i < n) {
    const float2 mine = p.sums[i];
    sa = mine.x;
    sb = mine.y;
    for (int r = 0; r < p.world; ++r) {
      if (r == p.me) continue;
      st_relaxed_sys_v2(p.peer_inbox[r] + 2 * i, make_uint2(__float_as_uint(mine.x), ep));
      st_relaxed_sys_v2(p.peer_inbox[r] + 2 * i + 1, make_uint2(__float_as_uint(mine.y), ep));
    }
    const uint64_t t0 = global_timer_ns();
    for (int r = 0; r < p.world; ++r) {
      if (r == p.me) continue;
      const uint2* in = p.inbox + (static_cast<long long>(r) * n + i) * 2;
      uint2 a, b;
      unsigned spins = 0;
      for (;;) {
        a = ld_relaxed_sys_v2(in);
        b = ld_relaxed_sys_v2(in + 1);
        if (a.y == ep && b.y == ep) break;
        if ((++spins & 0x3ff) == 0 && global_timer_ns() - t0 > FZ_P2P_TIMEOUT_NS) {
          printf("fz: GroupNorm statistics of peer %d never arrived (epoch %u, have %u / %u)\n", r, ep, a.y, b.y);
          __trap();
        }
      }
      sa += __uint_as_float(a.x);
      sb += __uint_as_float(b.x);
    }
    gx_smem[2 * i] = sa;
    gx_smem[2 * i + 1] = sb;
  }
  __syncthreads();
  if (threadIdx.x == 0) *p.epoch = ep;  // every thread has read the old value (it is read before the barrier)
  const int sets = p.NB / p.F_loc, G = p.G, F_loc = p.F_loc;
  if (i < sets * G) {
    const int b = i / G, g = i - b * G;
    double ta = 0.0, tb = 0.0;
    for (int f = 0; f < F_loc; ++f) {
      ta += gx_smem[2 * ((b * F_loc + f) * G + g)];
      tb += gx_smem[2 * ((b * F_loc + f) * G + g) + 1];
    }
    p.totals[(b * F_loc) * G + g] = make_double2(ta, tb);
    for (int f = 1; f < F_loc; ++f) p.totals[(b * F_loc + f) * G + g] = make_double2(0.0, 0.0);
  }
}

}  // namespace fz

using namespace fz;

extern "C" int fz_p2p_alloc(long long nbytes, void** ptr) {
  FZ_CHECK_ARG(ptr && nbytes > 0, "fz_p2p_alloc: bad args");
  FZ_CUDA(cudaMalloc(ptr, static_cast<size_t>(nbytes)));
  FZ_CUDA(cudaMemset(*ptr, 0, static_cast<size_t>(nbytes)));
  FZ_CUDA(cudaDeviceSynchronize());
  return FZ_OK;
}
extern "C" int fz_p2p_free(void* ptr) {
  FZ_CUDA(cudaFree(ptr));
  return FZ_OK;
}
extern "C" int fz_p2p_export(void* ptr, void* handle64) {
  FZ_CHECK_ARG(ptr && handle64, "fz_p2p_export: null pointer");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  cudaIpcMemHandle_t h;
  FZ_CUDA(cudaIpcGetMemHandle(&h, ptr));
  memcpy(handle64, &h, 64);
  return FZ_OK;
}
extern "C" int fz_p2p_import(const void* handle64, void** ptr) {
  FZ_CHECK_ARG(ptr && handle64, "fz_p2p_import: null pointer");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  FZ_CUDA(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return FZ_OK;
}
extern "C" int fz_p2p_unimport(void* ptr) {
  FZ_CUDA(cudaIpcCloseMemHandle(ptr));
  return FZ_OK;
}

extern "C" int fz_p2p_push(const fz_p2p_seg_t* segs, int n_segs, void* const* flags, void* counter, int n_dst, void* wait_flags, unsigned wait_mask,
                           cudaStream_t stream) {
  FZ_CHECK_ARG(segs && n_segs >= 1 && n_segs <= kP2PMaxSegs && n_dst >= 0 && n_dst <= kP2PMaxDst && counter, "fz_p2p_push: %d segments / %d destinations unsupported",
               n_segs, n_dst);
  P2PPushParams p;
  memset(&p, 0, sizeof(p));
  long long max_vec = 1;
  for (int i = 0; i < n_segs; ++i) {
    const fz_p2p_seg_t& s = segs[i];
    FZ_CHECK_ARG(s.src && s.dst && s.rows > 0 && s.row_bytes > 0 && s.row_bytes % 16 == 0 && s.src_pitch % 16 == 0 && s.dst_pitch % 16 == 0 &&
                     (reinterpret_cast<uintptr_t>(s.src) & 15) == 0 && (reinterpret_cast<uintptr_t>(s.dst) & 15) == 0,
                 "fz_p2p_push: segment %d is not 16-byte addressable", i);
    p.seg[i].src = static_cast<const uint8_t*>(s.src); p.seg[i].dst = static_cast<uint8_t*>(s.dst);
    p.seg[i].src_pitch = s.src_pitch; p.seg[i].dst_pitch = s.dst_pitch; p.seg[i].rows = s.rows; p.seg[i].row_bytes = s.row_bytes;
    p.seg[i].dst_slot = s.dst_slot;
    max_vec = std::max(max_vec, static_cast<long long>(s.rows) * (s.row_bytes >> 4));
  }
  p.n_segs = n_segs;
  p.n_dst = n_dst;
  // ~8 vectors per thread; large local re-layouts get up to two waves of CTAs, halo-sized segments a handful
  int gx = static_cast<int>(std::min<long long>(296 / std::max(1, n_segs) + 1, (max_vec + 256 * 8 - 1) / (256 * 8)));
  if (gx < 1) gx = 1;
  for (int d = 0; d < n_dst; ++d) {
    FZ_CHECK_ARG(flags[d], "fz_p2p_push: null flag");
    p.flag[d] = static_cast<unsigned*>(flags[d]);
  }
  p.counter = static_cast<unsigned*>(counter);
  p.wait_flags = static_cast<unsigned*>(wait_flags);
  p.wait_mask = wait_flags ? wait_mask : 0u;
  FZ_CUDA(launch_pdl(p2p_push_kernel, dim3(gx, n_segs), dim3(256), 0, stream, p));
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}

extern "C" int fz_p2p_wait(void* flags, unsigned mask, cudaStream_t stream) {
  FZ_CHECK_ARG(flags, "fz_p2p_wait: null pointer");
  if (mask == 0) return FZ_OK;
  FZ_CUDA(launch_pdl(p2p_wait_kernel, dim3(1), dim3(32), 0, stream, static_cast<unsigned*>(flags), mask));
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}

extern "C" int fz_gn_combine(void* epoch, void* const* peer_inbox, const void* inbox, const void* sums, void* totals, int NB, int F_loc, int G,
                             int world, int me, cudaStream_t stream) {
  FZ_CHECK_ARG(epoch && peer_inbox && inbox && sums && totals && F_loc >= 1 && NB % F_loc == 0 && world >= 1 && world <= 32 && me >= 0 && me < world,
               "fz_gn_combine: bad args");
  const int n = NB * G;
  FZ_CHECK_ARG(n <= 1024, "fz_gn_combine: %d images x groups > 1024", n);
  GnXchgParams p;
  memset(&p, 0, sizeof(p));
  for (int r = 0; r < world; ++r) {
    if (r == me) continue;
    FZ_CHECK_ARG(peer_inbox[r], "fz_gn_combine: null peer pointer");
    p.peer_inbox[r] = static_cast<uint2*>(peer_inbox[r]);
  }
  p.inbox = static_cast<const uint2*>(inbox); p.epoch = static_cast<unsigned*>(epoch); p.sums = static_cast<const float2*>(sums);
  p.totals = static_cast<double2*>(totals);
  p.NB = NB; p.F_loc = F_loc; p.G = G; p.world = world; p.me = me;
  const int threads = std::max(64, (n + 31) / 32 * 32);
  FZ_CUDA(launch_pdl(gn_combine_kernel, dim3(1), dim3(threads), static_cast<size_t>(n) * 16, stream, p));
  FZ_CUDA(cudaGetLastError());
  return FZ_OK;
}
