// adp_wgrad: weight-gradient GEMM on wgmma (backward of adp_conv_gemm w.r.t. W).
//
//   dW[n = out channel][k = in channel] += sum_{b,t} G[b, t, g_col0 + n] * X[b, t + off, x_col0 + k]
//
// The reduction runs over TIME, which is the strided dimension of both channels-last
// operands, so both are fed to the tensor core as MN-major tiles exactly as they lie in
// memory (no transposes): a 64-time-step chunk of G is the A operand (M = 128 out channels =
// two 64-channel swizzle chunks, one per consumer warpgroup), the row-shifted chunk of X the B
// operand (N = BN in channels, 64-channel chunks LBO apart).  TMA zero-fills rows outside
// [0,T) (conv padding) and channels beyond the tensor (C < 64), so narrow levels just run
// padded tiles.  fp32 accumulation in registers over the CTA's share of the (batch, time)
// chunks, then fp32 atomics into dW (split-K over time across CTAs).  Warp roles: 0-7 the two
// consumer warpgroups, 8 the TMA producer.
#include "common.cuh"
#include "ptx.cuh"

namespace adp {

constexpr int kWgChunk = 64;          // time steps per pipeline stage
constexpr int kWgBoxBytes = 64 * 128; // one TMA box: 64 rows x 64 channels bf16
constexpr int kWgMaxStages = 8;
constexpr int kWgThreads = 288;

struct WgradParams {
  float* dw;
  long long tap_stride;    // floats between the dW slabs of consecutive taps (fused 3-tap mode)
  int ldw;                 // row pitch of dW in floats
  int n_valid, k_valid;    // real out / in channel counts (tile masks)
  int T, chunks_per_batch, total_chunks, chunks_per_split;
  int g_col0, x_col0, off;
  int n_stages, nb;        // nb = BN / 64 boxes of X per stage
};

// NT = 3: the three taps of a k=3 convolution in ONE launch.  The X box carries 2 extra time rows;
// tap j is the same smem tile read through a descriptor whose start is advanced by j rows (the
// 128-byte swizzle is a function of the absolute address, as for the shifted-tap forward GEMM), and
// accumulates into its own registers.  G and X are read once instead of three times.
template <int BN, int NT>
__global__ void __launch_bounds__(kWgThreads, 1)
wgrad_kernel(const __grid_constant__ CUtensorMap tmG, const __grid_constant__ CUtensorMap tmX,
             const WgradParams p) {
  constexpr int NB = BN / 64;
  constexpr int XBOX = NT == 1 ? kWgBoxBytes : 9 * 1024;        // (64 + NT - 1) rows x 128 B, 1 KB-rounded
  constexpr int STAGE_BYTES = 2 * kWgBoxBytes + NB * XBOX;
  static_assert(NT * BN <= 256, "accumulators of all taps must fit the register file");
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t full_bar[kWgMaxStages], empty_bar[kWgMaxStages];

  pdl_launch_dependents();
  const int warp = warp_id_uniform();
  const int lane = threadIdx.x & 31;
  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* ring = smem_raw + ((1024u - (raw & 1023u)) & 1023u);

  const int n0 = blockIdx.x * 128;             // out-channel tile
  const int k0 = blockIdx.y * BN;              // in-channel tile
  const int chunk_begin = blockIdx.z * p.chunks_per_split;
  int chunk_end = chunk_begin + p.chunks_per_split;
  if (chunk_end > p.total_chunks) chunk_end = p.total_chunks;

  if (warp == 8 && lane == 0) {
    for (int s = 0; s < p.n_stages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }
    fence_mbar_init();
    tma_prefetch_desc(&tmG);
    tma_prefetch_desc(&tmX);
  }
  __syncthreads();
  pdl_wait();

  if (warp == 8) {
    // whole warp runs the loop (uniform control flow), one elected lane issues: see ptx.cuh
    int s = 0;
    uint32_t ph = 0;
    for (int c = chunk_begin; c < chunk_end; ++c) {
      const int b = c / p.chunks_per_batch;
      const int t0 = (c - b * p.chunks_per_batch) * kWgChunk;
      mbar_wait(&empty_bar[s], ph ^ 1);
      if (elect_one()) {
        uint8_t* st = ring + s * STAGE_BYTES;
        // bytes actually written: the X boxes are (64 + NT - 1) rows of 128 B (the stage slot is
        // rounded up to 1 KB)
        mbar_arrive_expect_tx(&full_bar[s], 2 * kWgBoxBytes + NB * (kWgChunk + NT - 1) * 128);
        tma_load_3d(st, &tmG, &full_bar[s], p.g_col0 + n0, t0, b);
        tma_load_3d(st + kWgBoxBytes, &tmG, &full_bar[s], p.g_col0 + n0 + 64, t0, b);
#pragma unroll
        for (int i = 0; i < NB; ++i)
          tma_load_3d(st + 2 * kWgBoxBytes + i * XBOX, &tmX, &full_bar[s], p.x_col0 + k0 + i * 64,
                      t0 + p.off, b);
      }
      __syncwarp();
      if (++s == p.n_stages) { s = 0; ph ^= 1; }
    }
    return;
  }

  // -------------------------------------------------------------------------- consumers
  const int wg = threadIdx.x >> 7;             // out channels [64*wg, 64*wg + 64) of the tile
  // MN-major SW128: G box of this warpgroup (one 64-channel chunk); X chunks XBOX apart (LBO);
  // 8-row groups 1024 B apart (SBO); 16 time steps per MMA = 2048 B
  const uint64_t gdesc0 = gmma_desc_mnmajor_sw128(smem_u32(ring) + wg * kWgBoxBytes, kWgBoxBytes);
  const uint64_t xdesc0 = gmma_desc_mnmajor_sw128(smem_u32(ring) + 2 * kWgBoxBytes, XBOX);
  float acc[NT][BN / 2];
  int s = 0;
  uint32_t ph = 0, accumulate = 0;
  for (int c = chunk_begin; c < chunk_end; ++c) {
    mbar_wait(&full_bar[s], ph);
    const uint64_t gdesc = gdesc0 + static_cast<uint64_t>((s * STAGE_BYTES) >> 4);
    const uint64_t xdesc = xdesc0 + static_cast<uint64_t>((s * STAGE_BYTES) >> 4);
    wgmma_fence();
#pragma unroll
    for (int tap = 0; tap < NT; ++tap) {
#pragma unroll
      for (int kk = 0; kk < kWgChunk / 16; ++kk)
        Wgmma<BN>::template ss<1, 1>(acc[tap], gdesc + ((kk * 2048) >> 4),
                                     xdesc + ((tap * 128 + kk * 2048) >> 4), accumulate | (kk != 0));
    }
    wgmma_commit();
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[s]);
    accumulate = 1;
    if (++s == p.n_stages) { s = 0; ph ^= 1; }
  }
  if (chunk_end <= chunk_begin) return;        // an empty split contributes nothing
#pragma unroll
  for (int tap = 0; tap < NT; ++tap) acc_fence(acc[tap]);

  // dW += the product.  With one split this thread is the only writer of its elements: a plain
  // read-modify-write instead of atomics
  const bool single = gridDim.z == 1;
  const bool pairs = (p.ldw & 1) == 0 && (p.tap_stride & 1) == 0;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int n = n0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * r;
    if (n >= p.n_valid) continue;
#pragma unroll
    for (int tap = 0; tap < NT; ++tap) {
      float* drow = p.dw + tap * p.tap_stride + static_cast<size_t>(n) * p.ldw;
#pragma unroll
      for (int jb = 0; jb < BN / 8; ++jb) {
        const int k = k0 + 8 * jb + 2 * (lane & 3);
        const float v0 = acc[tap][4 * jb + 2 * r], v1 = acc[tap][4 * jb + 2 * r + 1];
        if (k + 1 < p.k_valid && pairs) {
          float2* d2 = reinterpret_cast<float2*>(drow + k);
          if (single) {
            const float2 o = *d2;
            *d2 = make_float2(o.x + v0, o.y + v1);
          } else {
            atomicAdd(d2, make_float2(v0, v1));
          }
        } else {
          if (k < p.k_valid) { if (single) drow[k] += v0; else atomicAdd(drow + k, v0); }
          if (k + 1 < p.k_valid) { if (single) drow[k + 1] += v1; else atomicAdd(drow + k + 1, v1); }
        }
      }
    }
  }
}

template <int BN, int NT>
static int launch_wgrad(const adp_wgrad_args& a, cudaStream_t stream) {
  constexpr int NB = BN / 64;
  constexpr int XBOX = NT == 1 ? kWgBoxBytes : 9 * 1024;
  constexpr int STAGE_BYTES = 2 * kWgBoxBytes + NB * XBOX;
  CUtensorMap tmG, tmX;
  const uint32_t box[3] = {64, (uint32_t)kWgChunk, 1};
  const uint32_t xbox[3] = {64, (uint32_t)(kWgChunk + NT - 1), 1};
  {
    const uint64_t dims[3] = {(uint64_t)a.g_cols, (uint64_t)a.T, (uint64_t)a.B};
    const uint64_t str[2] = {(uint64_t)a.ldg * 2, (uint64_t)a.T * a.ldg * 2};
    if (int e = make_tmap_bf16(&tmG, a.g, 3, dims, str, box, 128)) return e;
  }
  {
    const uint64_t dims[3] = {(uint64_t)a.x_cols, (uint64_t)a.T, (uint64_t)a.B};
    const uint64_t str[2] = {(uint64_t)a.ldx * 2, (uint64_t)a.T * a.ldx * 2};
    if (int e = make_tmap_bf16(&tmX, a.x, 3, dims, str, xbox, 128)) return e;
  }
  WgradParams p;
  p.dw = a.dw;
  p.tap_stride = a.tap_stride;
  p.ldw = a.ldw;
  p.n_valid = a.n;
  p.k_valid = a.k;
  p.T = a.T;
  p.chunks_per_batch = (a.T + kWgChunk - 1) / kWgChunk;
  p.total_chunks = a.B * p.chunks_per_batch;
  p.g_col0 = a.g_col0;
  p.x_col0 = a.x_col0;
  p.off = a.off;
  p.nb = NB;
  int n_stages = (192 * 1024) / STAGE_BYTES;
  if (n_stages > kWgMaxStages) n_stages = kWgMaxStages;
  p.n_stages = n_stages;
  const int n_tiles = (a.n + 127) / 128, k_tiles = (a.k + BN - 1) / BN;
  const int sms = num_sms();
  // split-K over time: every split ends in NT x 128 x BN fp32 reductions into dW.  Narrow outputs
  // (few tiles) need many splits to fill the SMs; wide outputs pay for every split in atomics:
  // cap the total reduction traffic at ~4 M elements and keep >= 4 chunks per CTA
  int splits = (2 * sms) / (n_tiles * k_tiles);
  const long out_elems = (long)NT * a.n * a.k;
  const long by_atomics = (4L << 20) / (out_elems > 0 ? out_elems : 1);
  if (splits > by_atomics) splits = (int)(by_atomics < 1 ? 1 : by_atomics);
  if (splits > p.total_chunks / 4) splits = p.total_chunks / 4;
  if (splits < 1) splits = 1;
  p.chunks_per_split = (p.total_chunks + splits - 1) / splits;
  splits = (p.total_chunks + p.chunks_per_split - 1) / p.chunks_per_split;
  const size_t smem = static_cast<size_t>(n_stages) * STAGE_BYTES + 1024;
  static SmemAttrCache smem_cache;
  ADP_CUDA(ensure_dyn_smem(wgrad_kernel<BN, NT>, smem, smem_cache));
  dim3 grid(n_tiles, k_tiles, splits);
  ADP_CUDA(launch_k(wgrad_kernel<BN, NT>, grid, dim3(kWgThreads), smem, stream, tmG, tmX, p));
  return 0;
}

}  // namespace adp

extern "C" int adp_wgrad(const adp_wgrad_args* args, adp_stream_t stream) {
  using namespace adp;
  ADP_CHECK(args && args->g && args->x && args->dw, "adp_wgrad: null pointer");
  const adp_wgrad_args& a = *args;
  ADP_CHECK(a.B > 0 && a.T > 0 && a.n > 0 && a.k > 0, "adp_wgrad: bad sizes");
  ADP_CHECK(a.ldg % 8 == 0 && a.ldx % 8 == 0 && a.g_cols % 8 == 0 && a.x_cols % 8 == 0,
            "adp_wgrad: pitches / extents must be multiples of 8");
  ADP_CHECK(a.g_col0 % 8 == 0 && a.x_col0 % 8 == 0, "adp_wgrad: column offsets must be multiples of 8");
  ADP_CHECK(a.g_col0 + a.n <= a.g_cols && a.x_col0 + a.k <= a.x_cols, "adp_wgrad: columns out of range");
  ADP_CHECK(a.ntaps == 0 || a.ntaps == 1 || a.ntaps == 3, "adp_wgrad: ntaps must be 1 or 3");
  cudaStream_t s = as_stream(stream);
  if (a.ntaps == 3) {        // all taps of a k=3 conv: three register accumulators of 64 columns
    ADP_CHECK(a.tap_stride >= (long long)a.n * a.ldw, "adp_wgrad: tap_stride smaller than one dW slab");
    return launch_wgrad<64, 3>(a, s);
  }
  if (a.k > 128) return launch_wgrad<256, 1>(a, s);
  if (a.k > 64) return launch_wgrad<128, 1>(a, s);
  return launch_wgrad<64, 1>(a, s);
}
