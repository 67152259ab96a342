// Error state, device check and the TMA tensor-map encoder (driver entry point resolved at
// run time through the runtime API, so the library links against libcudart only).
#include "common.cuh"

#include <string.h>

namespace adp {

static thread_local char g_err[512] = "";
int g_pdl = 1;

int set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return 1;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e =
      cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !p) return nullptr;
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                   const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  ADP_CHECK(fn != nullptr, "cuTensorMapEncodeTiled entry point not available");
  ADP_CHECK((reinterpret_cast<uintptr_t>(base) & 15) == 0, "TMA base pointer not 16B aligned");
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bdim[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = 1;
    ADP_CHECK(box[i] >= 1 && box[i] <= 256, "TMA box dim %d = %u out of range", i, box[i]);
  }
  for (int i = 0; i + 1 < rank; ++i) {
    gstr[i] = strides_bytes[i];
    ADP_CHECK(strides_bytes[i] % 16 == 0, "TMA stride %d = %llu not a multiple of 16 bytes", i,
              (unsigned long long)strides_bytes[i]);
  }
  CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_NONE;
  if (swizzle_bytes == 32) sw = CU_TENSOR_MAP_SWIZZLE_32B;
  else if (swizzle_bytes == 64) sw = CU_TENSOR_MAP_SWIZZLE_64B;
  else if (swizzle_bytes == 128) sw = CU_TENSOR_MAP_SWIZZLE_128B;
  else ADP_CHECK(swizzle_bytes == 0, "bad swizzle %d", swizzle_bytes);
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, static_cast<cuuint32_t>(rank),
                  const_cast<void*>(base), gdim, gstr, bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  ADP_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with CUresult %d (rank %d dims "
            "%llu,%llu box %u,%u swizzle %d)", (int)r, rank, (unsigned long long)dims[0],
            (unsigned long long)(rank > 1 ? dims[1] : 0), box[0], rank > 1 ? box[1] : 0,
            swizzle_bytes);
  return 0;
}

int num_sms() {
  static int n[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) dev = 0;
  int& v = n[dev & 63];
  if (v <= 0 && (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0))
    v = 132;
  return v;
}

}  // namespace adp

extern "C" {

int adp_version(void) { return 1; }

const char* adp_last_error(void) { return adp::g_err; }

int adp_device_check(void) {
  int dev = 0;
  ADP_CUDA(cudaGetDevice(&dev));
  int major = 0, minor = 0;
  ADP_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  ADP_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  ADP_CHECK(major == 9 && minor == 0, "libadp_b200 is built for sm_90a (H100), found sm_%d%d",
            major, minor);
  return 0;
}

}  // extern "C"
