// Level-0 ("stem") pieces shared by stem.cu, stem_bwd.cu and the fp32 twins in verify_f32*.cu:
// the size envelope of the stem entry points, which sizes the narrow kernels take, the block-input
// gather and the stem_out epilogue.
#pragma once
#include "common.cuh"
#include "ptx.cuh"

namespace adp {

// ---------------------------------------------------------------------------- envelope
// Sizes every stem entry point accepts (adp_stem_in / _out / _in_bwd / _out_bwd); B200UNet.MAX_*
// states the same limits on the Python side.
constexpr int kStemMaxCin = 64;    // cx + ca, the block input channels
constexpr int kStemMaxIn = 128;    // (cx + ca) * f, the inputs of one stem_in output position
constexpr int kStemMaxC0 = 256;    // level-0 width, a multiple of 8
constexpr int kStemMaxCo = 64;     // outputs, co <= cx

// Refuses sizes outside the envelope, naming the entry point `fn`.  co: the outputs of the
// stem_out side; the stem_in side passes co = 1.
inline int check_stem_envelope(const char* fn, int cx, int ca, int c0, int f, int T, int co) {
  const int cin = cx + ca;
  ADP_CHECK(cx >= 1 && ca >= 0 && cin <= kStemMaxCin && f >= 1 && cin * f <= kStemMaxIn && T % f == 0 &&
                c0 >= 8 && c0 % 8 == 0 && c0 <= kStemMaxC0 && co >= 1 && co <= kStemMaxCo && co <= cx,
            "%s: cx=%d ca=%d c0=%d f=%d co=%d unsupported (cx+ca <= %d, (cx+ca)*f <= %d, T %% f == 0, "
            "c0 <= %d and a multiple of 8, co <= cx, co <= %d)",
            fn, cx, ca, c0, f, co, kStemMaxCin, kStemMaxIn, kStemMaxC0, kStemMaxCo);
  return 0;
}

// Sizes the narrow kernels take (register arrays sized at compile time); every other size of the
// envelope runs on the wide kernels.
constexpr int kStemInNarrowIn = 32;     // stem_in_kernel: (cx+ca)*f inputs per output position
constexpr int kStemOutNarrowCo = 4;     // stem_out_kernel: outputs ...
constexpr int kStemOutNarrowCin = 8;    // ... and block input channels per position
inline bool stem_in_narrow(const adp_stem_in_args& a) { return (a.cx + a.ca) * a.f <= kStemInNarrowIn; }
inline bool stem_out_narrow(const adp_stem_out_args& a) {
  return a.co <= kStemOutNarrowCo && a.cx + a.ca <= kStemOutNarrowCin;
}
// stem_out_bwd_kernel: 256-position tiles holding whole low-rate rows, at most 4 parameter
// gradients per thread
inline bool stem_out_bwd_narrow(const adp_stem_out_bwd_args& a) {
  const int cin = a.cx + a.ca;
  return a.co <= 4 && a.c0 <= 64 && cin <= 8 && 256 % a.f == 0 && a.co * a.c0 * 3 + 3 * a.co + a.co * cin <= 4 * 256;
}
// stem_in_bwd_kernel: at most 9 parameter gradients per thread, (cx+ca)*f*c0 + c0 <= 9 * 256
inline bool stem_in_bwd_narrow(const adp_stem_in_bwd_args& a) { return (a.cx + a.ca) * a.f <= 32 && a.c0 <= 64; }

// ------------------------------------------------------------------------- block input
// Channel c of the block input cat([x(_noisy), append]) of batch element b at position t;
// x_noisy = al*x + be*noise when args.noise is set (reference diffusion.py:91).  kLdg: read
// through the read-only data cache.  Every stem argument struct has these field names.
template <bool kLdg = false, typename Args>
__device__ __forceinline__ float block_input(const Args& a, int b, int c, size_t t, float al, float be) {
  auto ld = [](const float* p) { return kLdg ? __ldg(p) : *p; };
  if (c < a.cx) {
    const size_t idx = (static_cast<size_t>(b) * a.cx + c) * a.T + t;
    float v = ld(a.x + idx);
    if (a.noise) v = al * v + be * ld(a.noise + idx);
    return v;
  }
  return ld(a.append + (static_cast<size_t>(b) * a.ca + (c - a.cx)) * a.T + t);
}

// ---------------------------------------------------------------------- stem_out epilogue
// Output o at position t of batch element b, given the skip path `skip`, the conv branch y (ym:
// the unconditional row of the guidance pair) and xin = block input channel o: MergeModulate, the
// CFG combine, v_out, the sampler update x_next (reference diffusion.py:185-187) and the
// VDiffusion loss term (diffusion.py:92,95) with dL/dv.  al / be: the noising of batch element b.
// The loss reads x after x_next is stored, so the entry points refuse the two together.
__device__ __forceinline__ void stem_out_finish(const adp_stem_out_args& a, int b, int o, int t, float skip,
                                                float y, float ym, float xin, float al, float be,
                                                double& lsum) {
  const int ldg = a.ld_gate > 0 ? a.ld_gate : a.co;
  float v = skip + a.gate[static_cast<size_t>(b) * ldg + o] * y;               // MergeModulate
  if (a.cfg) {
    const float vm = skip + a.gate[static_cast<size_t>(b + a.B) * ldg + o] * ym;
    v = vm + (v - vm) * a.cfg_scale;                                           // CFG combine
  }
  const size_t oidx = (static_cast<size_t>(b) * a.co + o) * a.T + t;
  if (a.v_out) a.v_out[oidx] = v;
  if (a.x_next) {
    const float a0 = a.ab[0], b0 = a.ab[1], a1 = a.ab[2], b1 = a.ab[3];
    a.x_next[oidx] = a1 * (a0 * xin - b0 * v) + b1 * (b0 * xin + a0 * v);
  }
  if (a.loss_sum) {
    const size_t xidx = (static_cast<size_t>(b) * a.cx + o) * a.T + t;
    const float d = v - (al * a.noise[xidx] - be * a.x[xidx]);
    lsum += static_cast<double>(d) * d;
    if (a.dv) a.dv[oidx] = 2.f * d / (static_cast<float>(a.B) * a.co * a.T);
  }
}

// Block sum of the per-thread loss terms -> *loss_sum, one fp64 atomic per block.  Every thread of
// the block (at most 256) calls.
__device__ __forceinline__ void block_loss_flush(double lsum, double* loss_sum) {
  __shared__ double s_loss[8];
  for (int o = 16; o > 0; o >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
  if ((threadIdx.x & 31) == 0) s_loss[threadIdx.x >> 5] = lsum;
  __syncthreads();
  if (threadIdx.x == 0) {
    double tot = 0.0;
    for (int i = 0; i < (blockDim.x >> 5); ++i) tot += s_loss[i];
    atomicAdd(loss_sum, tot);
  }
}

}  // namespace adp
