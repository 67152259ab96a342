// Host-side helpers shared by the launchers: error reporting, TMA tensor-map encoding.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/adp_b200.h"

namespace adp {

int set_error(const char* fmt, ...);  // returns non-zero, records the message (thread-local)

#define ADP_CHECK(cond, ...)                         \
  do {                                               \
    if (!(cond)) return ::adp::set_error(__VA_ARGS__); \
  } while (0)

#define ADP_CUDA(expr)                                                                   \
  do {                                                                                   \
    cudaError_t e_ = (expr);                                                             \
    if (e_ != cudaSuccess) {                                                             \
      (void)cudaGetLastError();  /* a refused launch's error is not the next launch's */ \
      return ::adp::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_),    \
                              __FILE__, __LINE__);                                       \
    }                                                                                    \
  } while (0)

#define ADP_LAUNCH_CHECK() ADP_CUDA(cudaGetLastError())

// bf16 tensor map, up to 4 dims.  dims[0] is the contiguous dimension; strides_bytes[i] is
// the byte stride of dims[i+1].  swizzle_bytes in {0, 32, 64, 128}.
int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                   const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes);

inline cudaStream_t as_stream(adp_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device attribute: remember the largest
// value set so far for each device (one static cache per kernel instantiation at the call site).
struct SmemAttrCache { size_t set[64] = {}; };
template <typename Kern>
inline cudaError_t ensure_dyn_smem(Kern kernel, size_t bytes, SmemAttrCache& cache) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  size_t& cur = cache.set[dev & 63];
  // always opt in on first use: static + dynamic shared memory together may exceed the 48 KB
  // default even when the dynamic part alone does not
  if (bytes <= cur) return cudaSuccess;
  e = cudaFuncSetAttribute((const void*)kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e == cudaSuccess) cur = bytes;
  return e;
}

// Every kernel is launched with the programmatic-dependent-launch attribute: kernel N+1 may
// start (set up smem / mbarriers, prefetch tensor maps) while kernel N drains; it calls
// griddepcontrol.wait before its first global-memory access.  adp_debug_set(6, 0) disables.
extern int g_pdl;
template <typename Kern, typename... Args>
inline cudaError_t launch_k(Kern kernel, dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                            Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = g_pdl ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  void* ptrs[] = {(void*)&args...};
  return cudaLaunchKernelExC(&cfg, (const void*)kernel, ptrs);
}

// streaming multiprocessors of the current device (grid sizing of persistent / capped grids)
int num_sms();

// grid.x of a persistent (tile-looping) kernel launched as grid(gx, B): exactly one wave of
// resident blocks (a grid larger than occupancy * SMs would run a second, mostly empty wave)
template <typename K>
inline int one_wave_gx(K kernel, int threads, size_t smem, int B, int n_tiles) {
  int occ = 1;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, threads, smem) != cudaSuccess || occ < 1)
    occ = 1;
  int gx = (occ * num_sms()) / B;
  if (gx < 1) gx = 1;
  if (gx > n_tiles) gx = n_tiles;
  return gx;
}

// grid.x of a tile loop launched as grid(gx, B, z): about 4 blocks per SM in total
inline int blocks_per_batch(int n_tiles, int B, int z = 1) {
  int gx = (num_sms() * 4 + B * z - 1) / (B * z);
  if (gx > n_tiles) gx = n_tiles;
  return gx < 1 ? 1 : gx;
}

// Row layout of the LayerNorm row kernels (ln_film, ln_film_bwd), C a multiple of 8: the C/8
// vectors of a row spread over lpr lanes, vpl vectors per lane, lpr a power of two.  Up to 32
// vectors: one per lane on the next power of two of lanes; more: 32 lanes, ceil(C/256) vectors
// each.  Returns true when lpr * vpl > C/8, i.e. the kernel masks the vectors past the row end.
inline bool ln_row_layout(int C, int* lpr, int* vpl) {
  const int vpr = C / 8;
  if (vpr <= 32) {
    int p = 1;
    while (p < vpr) p <<= 1;
    *lpr = p; *vpl = 1;
  } else {
    *lpr = 32; *vpl = (vpr + 31) / 32;
  }
  return *lpr * *vpl != vpr;
}

// 1-D grid-stride launch over n items: one item per thread, at most 16 blocks per SM
inline int capped_grid(int64_t n, int threads) {
  int64_t g = (n + threads - 1) / threads;
  if (g < 1) g = 1;
  if (g > num_sms() * 16) g = num_sms() * 16;
  return static_cast<int>(g);
}

}  // namespace adp
