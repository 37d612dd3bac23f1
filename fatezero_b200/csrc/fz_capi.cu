// fz_capi.cu — error plumbing, device probe and the host-side TMA tensor-map encoder of libfatezero_b200.so
#include <cstdarg>
#include <cstdio>

#include "fz_common.cuh"
#include "../../include/fatezero_b200.h"

namespace fz {

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_encode = nullptr;

int encode_tmap_f16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_elems,
                    const uint32_t* box, bool swizzle128) {
  return encode_tmap_f16_sw(out, base, rank, dims, strides_elems, box, swizzle128 ? 128 : 0);
}

int encode_tmap_f16_sw(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_elems,
                       const uint32_t* box, int swizzle_bytes) {
  if (!g_encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn) {
      set_error("cuTensorMapEncodeTiled entry point unavailable (%s)", cudaGetErrorString(e));
      return FZ_ERR_CUDA;
    }
    g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  }
  cuuint64_t gdims[5];
  cuuint64_t gstrides[4];
  cuuint32_t gbox[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdims[i] = dims[i];
    gbox[i] = box[i];
    estr[i] = 1;
    if (box[i] == 0 || box[i] > 256) {
      set_error("tensor map: box[%d]=%u out of range", i, box[i]);
      return FZ_ERR_INVALID;
    }
  }
  for (int i = 0; i + 1 < rank; ++i) {
    gstrides[i] = strides_elems[i] * 2;
    if (gstrides[i] % 16 != 0) {
      set_error("tensor map: stride[%d]=%llu bytes is not a multiple of 16", i, (unsigned long long)gstrides[i]);
      return FZ_ERR_INVALID;
    }
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) {
    set_error("tensor map: base pointer not 16-byte aligned");
    return FZ_ERR_INVALID;
  }
  CUresult r = g_encode(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank, const_cast<void*>(base), gdims, gstrides, gbox, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE,
                        swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                        : swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (rank %d dims %llu %llu box %u %u)", (int)r, rank,
              (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0), box[0], rank > 1 ? box[1] : 0);
    return FZ_ERR_CUDA;
  }
  return FZ_OK;
}

}  // namespace fz

namespace fz {
int check_single_device() {
  static int first = -1;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    set_error("no CUDA device");
    return FZ_ERR_CUDA;
  }
  if (first < 0) first = dev;
  if (dev != first) {
    set_error("libfatezero_b200 was first used on device %d and is now called on device %d: it caches per-device state, run one process per GPU", first, dev);
    return FZ_ERR_INVALID;
  }
  return FZ_OK;
}
}  // namespace fz

extern "C" const char* fz_last_error(void) { return fz::g_err; }
extern "C" int fz_version(void) { return 100; }
extern "C" int fz_device_check(void) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) {
    fz::set_error("no CUDA device: %s", cudaGetErrorString(e));
    return FZ_ERR_CUDA;
  }
  int major = 0, minor = 0;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  if (major != 9 || minor != 0) {
    fz::set_error("libfatezero_b200 is built for sm_90a (H100) and needs an sm_90 GPU (found sm_%d%d)", major, minor);
    return FZ_ERR_INVALID;
  }
  return FZ_OK;
}
