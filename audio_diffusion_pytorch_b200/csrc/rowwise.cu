// Bandwidth-bound row/elementwise kernels (CUDA cores): GroupNorm apply + SiLU, GroupNorm
// statistics, LayerNorm over channels + FiLM (a_unet Modulation), the small conditioning
// linears, NumberEmbedder features and the stand-alone VSampler update.
// All activations are channels-last bf16, moved as 16-byte vectors (8 channels).
#include "common.cuh"
#include "ptx.cuh"

namespace adp {

constexpr int kMaxC = 2048;

// --------------------------------------------------------------------------- gn_silu
// y = silu(x * a[b,c] + d[b,c]),  a = gamma*rstd, d = beta - mean*a  from (sum, sumsq).
// Each CTA streams tiles of 1024 vectors, four independent 16-byte loads in flight per thread
// plus the next tile's.  REG: C/8 divides 256, so a thread meets the SAME 8 channels in every
// vector it touches and keeps their coefficients in registers — the statistics / gamma / beta
// loads go out together with the first data loads (one latency round, no smem, no barrier; the
// deep levels' launches are latency-, not bandwidth-bound).  Otherwise coefficients of all C
// channels are staged in smem.
template <bool REG, int NV>      // NV = 16-byte vectors per thread per tile (1 for small tensors)
__global__ void __launch_bounds__(256)
gn_silu_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, const double* __restrict__ stats,
               const float* __restrict__ gamma, const float* __restrict__ beta, int T, int C,
               int groups, float eps) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ __align__(16) float s_a[REG ? 8 : kMaxC];
  __shared__ __align__(16) float s_d[REG ? 8 : kMaxC];
  const int b = blockIdx.y;
  const int gsz = C / groups;
  const int vpr = C >> 3;  // vectors per row
  const uint32_t nvec = static_cast<uint32_t>(T) * vpr;          // < 2^31 (checked by the host)
  const uint4* xb = x + static_cast<size_t>(b) * nvec;
  uint4* yb = y + static_cast<size_t>(b) * nvec;
  constexpr uint32_t TILE = 256u * NV;
  uint4 u[NV];
  uint32_t base = blockIdx.x * TILE;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const uint32_t i = base + k * 256 + threadIdx.x;
    u[k] = i < nvec ? __ldg(xb + i) : make_uint4(0, 0, 0, 0);
  }
  const double inv_n = 1.0 / (static_cast<double>(gsz) * T);
  float ca[8], cd[8];
  if constexpr (REG) {
    const int c0 = (threadIdx.x & (vpr - 1)) << 3;      // vpr is a power of two dividing 256
    const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + c0));
    const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma + c0 + 4));
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + c0));
    const float4 b1 = __ldg(reinterpret_cast<const float4*>(beta + c0 + 4));
    const float gm[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
    const float bt[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
    if (gsz >= 8) {            // the 8 channels share one group
      const int g = c0 / gsz;
      const double s = stats[(static_cast<size_t>(b) * groups + g) * 2];
      const double q = stats[(static_cast<size_t>(b) * groups + g) * 2 + 1];
      const double mean = s * inv_n;                    // fp64 only where cancellation bites
      const float var = fmaxf(static_cast<float>(q * inv_n - mean * mean), 0.f);
      const float rstd = rsqrtf(var + eps), fm = static_cast<float>(mean);
#pragma unroll
      for (int j = 0; j < 8; ++j) { ca[j] = gm[j] * rstd; cd[j] = bt[j] - fm * ca[j]; }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int g = (c0 + j) / gsz;
        const double s = stats[(static_cast<size_t>(b) * groups + g) * 2];
        const double q = stats[(static_cast<size_t>(b) * groups + g) * 2 + 1];
        const double mean = s * inv_n;
        const float var = fmaxf(static_cast<float>(q * inv_n - mean * mean), 0.f);
        ca[j] = gm[j] * rsqrtf(var + eps);
        cd[j] = bt[j] - static_cast<float>(mean) * ca[j];
      }
    }
  } else {
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      const int g = c / gsz;
      const double s = stats[(static_cast<size_t>(b) * groups + g) * 2];
      const double q = stats[(static_cast<size_t>(b) * groups + g) * 2 + 1];
      const double mean = s * inv_n;
      const float var = fmaxf(static_cast<float>(q * inv_n - mean * mean), 0.f);
      const float a = gamma[c] * rsqrtf(var + eps);
      s_a[c] = a;
      s_d[c] = beta[c] - static_cast<float>(mean) * a;
    }
    __syncthreads();
  }
  for (; base < nvec; base += gridDim.x * TILE) {
    const uint32_t nbase = base + gridDim.x * TILE;
    uint4 un[NV];
    if (nbase < nvec) {
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        const uint32_t i = nbase + k * 256 + threadIdx.x;
        un[k] = i < nvec ? __ldg(xb + i) : make_uint4(0, 0, 0, 0);
      }
    }
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const uint32_t i = base + k * 256 + threadIdx.x;
      if (i >= nvec) continue;
      if constexpr (!REG) {
        const int c = static_cast<int>(i % static_cast<uint32_t>(vpr)) << 3;
#pragma unroll
        for (int j = 0; j < 8; ++j) { ca[j] = s_a[c + j]; cd[j] = s_d[c + j]; }
      }
      const float2 f0 = unpack_bf16(u[k].x), f1 = unpack_bf16(u[k].y);
      const float2 f2 = unpack_bf16(u[k].z), f3 = unpack_bf16(u[k].w);
      uint4 o;
      o.x = pack_bf16(silu_f(f0.x * ca[0] + cd[0]), silu_f(f0.y * ca[1] + cd[1]));
      o.y = pack_bf16(silu_f(f1.x * ca[2] + cd[2]), silu_f(f1.y * ca[3] + cd[3]));
      o.z = pack_bf16(silu_f(f2.x * ca[4] + cd[4]), silu_f(f2.y * ca[5] + cd[5]));
      o.w = pack_bf16(silu_f(f3.x * ca[6] + cd[6]), silu_f(f3.y * ca[7] + cd[7]));
      yb[i] = o;
    }
#pragma unroll
    for (int k = 0; k < NV; ++k) u[k] = un[k];
  }
}

// -------------------------------------------------------------------------- gn_stats
__global__ void __launch_bounds__(256)
gn_stats_kernel(const uint4* __restrict__ x, double* __restrict__ stats, int T, int C,
                int groups) {
  pdl_launch_dependents();
  pdl_wait();
  // each thread keeps a fixed channel-vector (stride is a multiple of vectors-per-row)
  __shared__ float s_acc[2 * 64];
  const int b = blockIdx.y;
  const int gsz = C / groups;
  const int vpr = C >> 3;
  if (threadIdx.x < 2 * groups) s_acc[threadIdx.x] = 0.f;
  __syncthreads();
  const size_t nvec = static_cast<size_t>(T) * vpr;
  const uint4* xb = x + static_cast<size_t>(b) * nvec;
  // make the per-thread stride a multiple of vpr so its channels never change
  const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t stride = nthreads / vpr * vpr;      // round DOWN: threads >= stride sit out (host: vpr <= 256)
  float s[8], q[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { s[j] = 0.f; q[j] = 0.f; }
  if (tid < stride) {
    for (size_t i = tid; i < nvec; i += stride) {
      const uint4 u = __ldg(xb + i);
      const uint32_t in[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16(in[j]);
        s[2 * j] += f.x; q[2 * j] += f.x * f.x;
        s[2 * j + 1] += f.y; q[2 * j + 1] += f.y * f.y;
      }
    }
    const int c = static_cast<int>(tid % vpr) << 3;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int g = (c + j) / gsz;
      atomicAdd(&s_acc[2 * g], s[j]);
      atomicAdd(&s_acc[2 * g + 1], q[j]);
    }
  }
  __syncthreads();
  if (threadIdx.x < 2 * groups)
    atomicAdd(stats + static_cast<size_t>(b) * 2 * groups + threadIdx.x,
              static_cast<double>(s_acc[threadIdx.x]));
}

// --------------------------------------------------------------------------- ln_film
// One row = C channels = C/8 vectors spread over LPR lanes (VPL vectors per lane); UNR
// independent row groups per warp iteration keep several 16-byte loads in flight per lane.
constexpr int kMaxLnC = 1024;
template <int VPL, bool PER_CH, int UNR>
__global__ void __launch_bounds__(256)
ln_film_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, const float* __restrict__ ss,
               int ss_stride, double* __restrict__ stats, int T, int C, int lpr, int groups,
               float eps, uint4* __restrict__ y2, float eps2) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float s_acc[2 * 64];
  __shared__ __align__(16) float s_fs[kMaxLnC];
  __shared__ __align__(16) float s_ft[kMaxLnC];
  const int b = blockIdx.y;
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int rpw = 32 / lpr;          // rows per warp per group
  const int sub = lane / lpr;        // which of those rows
  const int l = lane - sub * lpr;    // lane inside the row
  const int vpr = C >> 3;
  const int gsz = groups > 0 ? C / groups : C;
  const bool do_stats = stats != nullptr;
  if (threadIdx.x < 128) s_acc[threadIdx.x] = 0.f;

  constexpr int NACC = PER_CH ? 8 : VPL;
  float as[NACC], aq[NACC];
#pragma unroll
  for (int j = 0; j < NACC; ++j) { as[j] = 0.f; aq[j] = 0.f; }

  const uint4* xb = x + static_cast<size_t>(b) * T * vpr;
  uint4* yb = y + static_cast<size_t>(b) * T * vpr;
  const int warps_total = gridDim.x * (blockDim.x >> 5);
  const float inv_c = 1.f / static_cast<float>(C);
  const int step = warps_total * rpw * UNR;
  auto load_rows = [&](int base, uint4 (&dst)[UNR][VPL]) {
#pragma unroll
    for (int un = 0; un < UNR; ++un) {
      const int row = base + un * rpw + sub;
#pragma unroll
      for (int it = 0; it < VPL; ++it) {
        dst[un][it] = make_uint4(0, 0, 0, 0);
        if (row < T) dst[un][it] = __ldg(xb + static_cast<size_t>(row) * vpr + it * lpr + l);
      }
    }
  };
  // the first rows are requested BEFORE the FiLM coefficients are staged (the two global
  // latencies of this latency-bound kernel overlap), later rows one iteration ahead
  int base = (blockIdx.x * (blockDim.x >> 5) + warp) * rpw * UNR;
  uint4 u[UNR][VPL];
  load_rows(base, u);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {   // FiLM coefficients of this batch row
    s_fs[c] = ss ? 1.f + ss[static_cast<size_t>(b) * ss_stride + c] : 1.f;
    s_ft[c] = ss ? ss[static_cast<size_t>(b) * ss_stride + C + c] : 0.f;
  }
  __syncthreads();
  for (; base < T; base += step) {
    uint4 unx[UNR][VPL];
    if (base + step < T) load_rows(base + step, unx);
#pragma unroll
    for (int un = 0; un < UNR; ++un) {
      const int row = base + un * rpw + sub;
      const bool ok = row < T;
      float v[VPL][8];
      float sum = 0.f;
#pragma unroll
      for (int it = 0; it < VPL; ++it) {
        const uint32_t in[4] = {u[un][it].x, u[un][it].y, u[un][it].z, u[un][it].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = unpack_bf16(in[j]);
          v[it][2 * j] = f.x; v[it][2 * j + 1] = f.y;
          sum += f.x + f.y;
        }
      }
      for (int o = lpr >> 1; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      const float mean = sum * inv_c;
      float sq = 0.f;
#pragma unroll
      for (int it = 0; it < VPL; ++it)
#pragma unroll
        for (int j = 0; j < 8; ++j) { const float d = v[it][j] - mean; sq += d * d; }
      for (int o = lpr >> 1; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
      const float rstd = rsqrtf(sq * inv_c + eps);
#pragma unroll
      for (int it = 0; it < VPL; ++it) {
        const int c = (it * lpr + l) << 3;
        const float4 f0 = *reinterpret_cast<const float4*>(&s_fs[c]);
        const float4 f1 = *reinterpret_cast<const float4*>(&s_fs[c + 4]);
        const float4 t0 = *reinterpret_cast<const float4*>(&s_ft[c]);
        const float4 t1 = *reinterpret_cast<const float4*>(&s_ft[c + 4]);
        const float fs[8] = {f0.x, f0.y, f0.z, f0.w, f1.x, f1.y, f1.z, f1.w};
        const float ft[8] = {t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w};
        uint32_t o4[4];
        float r[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float y0 = (v[it][2 * j] - mean) * rstd * fs[2 * j] + ft[2 * j];
          const float y1 = (v[it][2 * j + 1] - mean) * rstd * fs[2 * j + 1] + ft[2 * j + 1];
          o4[j] = pack_bf16(y0, y1);
          const float2 rr = unpack_bf16(o4[j]);   // statistics of what is stored
          r[2 * j] = rr.x; r[2 * j + 1] = rr.y;
          v[it][2 * j] = rr.x; v[it][2 * j + 1] = rr.y;   // kept for the second LayerNorm
        }
        if (ok) {
          yb[static_cast<size_t>(row) * vpr + it * lpr + l] = make_uint4(o4[0], o4[1], o4[2], o4[3]);
          if (do_stats) {
            if constexpr (PER_CH) {
#pragma unroll
              for (int j = 0; j < 8; ++j) { as[j] += r[j]; aq[j] += r[j] * r[j]; }
            } else {
#pragma unroll
              for (int j = 0; j < 8; ++j) { as[it] += r[j]; aq[it] += r[j] * r[j]; }
            }
          }
        }
      }
      if (y2) {   // y2 = LayerNorm(y; eps2) of the stored (rounded) y: the attention pre-norm
        float sum2 = 0.f;
#pragma unroll
        for (int it = 0; it < VPL; ++it)
#pragma unroll
          for (int j = 0; j < 8; ++j) sum2 += v[it][j];
        for (int o = lpr >> 1; o > 0; o >>= 1) sum2 += __shfl_xor_sync(0xffffffffu, sum2, o);
        const float mean2 = sum2 * inv_c;
        float sq2 = 0.f;
#pragma unroll
        for (int it = 0; it < VPL; ++it)
#pragma unroll
          for (int j = 0; j < 8; ++j) { const float d = v[it][j] - mean2; sq2 += d * d; }
        for (int o = lpr >> 1; o > 0; o >>= 1) sq2 += __shfl_xor_sync(0xffffffffu, sq2, o);
        const float rstd2 = rsqrtf(sq2 * inv_c + eps2);
        if (ok) {
#pragma unroll
          for (int it = 0; it < VPL; ++it) {
            uint4 o;
            o.x = pack_bf16((v[it][0] - mean2) * rstd2, (v[it][1] - mean2) * rstd2);
            o.y = pack_bf16((v[it][2] - mean2) * rstd2, (v[it][3] - mean2) * rstd2);
            o.z = pack_bf16((v[it][4] - mean2) * rstd2, (v[it][5] - mean2) * rstd2);
            o.w = pack_bf16((v[it][6] - mean2) * rstd2, (v[it][7] - mean2) * rstd2);
            y2[static_cast<size_t>(b) * T * vpr + static_cast<size_t>(row) * vpr + it * lpr + l] = o;
          }
        }
      }
    }
#pragma unroll
    for (int un = 0; un < UNR; ++un)
#pragma unroll
      for (int it = 0; it < VPL; ++it) u[un][it] = unx[un][it];
  }
  if (do_stats) {
    // lanes l, l+lpr, l+2*lpr, ... hold the same channels: fold them before touching smem
#pragma unroll
    for (int j = 0; j < NACC; ++j)
      for (int o = lpr; o < 32; o <<= 1) {
        as[j] += __shfl_xor_sync(0xffffffffu, as[j], o);
        aq[j] += __shfl_xor_sync(0xffffffffu, aq[j], o);
      }
    if (sub == 0) {
      if constexpr (PER_CH) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int g = ((l << 3) + j) / gsz;
          atomicAdd(&s_acc[2 * g], as[j]);
          atomicAdd(&s_acc[2 * g + 1], aq[j]);
        }
      }
    }
    if constexpr (!PER_CH) {
      // gsz/8 consecutive lanes of a row hold channels of the SAME group: reduce them with
      // shuffles so that one lane per (warp, group) touches the 2*groups shared bins (at
      // C = 1024 the per-lane version queued 16 lanes on every bin and tripled the kernel time)
      const int lpg = gsz >> 3;                               // lanes (vectors) per group
      const int span = lpg < lpr ? lpg : lpr;                 // lanes to fold
      const bool tree = span > 0 && (span & (span - 1)) == 0 && (lpg >= lpr ? lpg % lpr == 0 : lpr % lpg == 0);
#pragma unroll
      for (int it = 0; it < VPL; ++it) {
        float sa = as[it], sq = aq[it];
        if (tree) {
          for (int o = span >> 1; o > 0; o >>= 1) {
            sa += __shfl_xor_sync(0xffffffffu, sa, o);
            sq += __shfl_xor_sync(0xffffffffu, sq, o);
          }
        }
        if (sub == 0 && (!tree || (l & (span - 1)) == 0)) {
          const int g = ((it * lpr + l) << 3) / gsz;
          atomicAdd(&s_acc[2 * g], sa);
          atomicAdd(&s_acc[2 * g + 1], sq);
        }
      }
    }
    __syncthreads();
    if (threadIdx.x < 2 * groups)
      atomicAdd(stats + static_cast<size_t>(b) * 2 * groups + threadIdx.x,
                static_cast<double>(s_acc[threadIdx.x]));
  }
}

// --------------------------------------------------------------------- skinny_linear
// y[b][n] = out_act(sum_k in_act(x[b][k]) * w[n][k] + bias[n]); 16 batch rows per CTA in smem,
// one warp per output column, 16-value butterfly reduction.
constexpr int kSkinnyRows = 16;
__device__ __forceinline__ float apply_act(float v, int act) {
  if (act == ADP_ACT_GELU) return gelu_erf_f(v);
  if (act == ADP_ACT_SILU) return silu_f(v);
  return v;
}
__global__ void __launch_bounds__(256)
skinny_linear_kernel(const float* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                     const float* __restrict__ bias, float* __restrict__ y, int B, int K, int N,
                     int ldx, int ldw, int ldy, int in_act, int out_act) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float s_x[];  // [16][K]
  const int b0 = blockIdx.y * kSkinnyRows;
  for (int i = threadIdx.x; i < kSkinnyRows * K; i += blockDim.x) {
    const int r = i / K, k = i - r * K;
    float v = 0.f;
    if (b0 + r < B) v = apply_act(x[static_cast<size_t>(b0 + r) * ldx + k], in_act);
    s_x[i] = v;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int nwarps = gridDim.x * (blockDim.x >> 5);
  const int kvecs = K >> 3;
  for (int n = blockIdx.x * (blockDim.x >> 5) + warp; n < N; n += nwarps) {
    float acc[kSkinnyRows];
#pragma unroll
    for (int r = 0; r < kSkinnyRows; ++r) acc[r] = 0.f;
    const uint4* wr = reinterpret_cast<const uint4*>(w + static_cast<size_t>(n) * ldw);
    for (int kv = lane; kv < kvecs; kv += 32) {
      const uint4 u = __ldg(wr + kv);
      const float2 w0 = unpack_bf16(u.x), w1 = unpack_bf16(u.y);
      const float2 w2 = unpack_bf16(u.z), w3 = unpack_bf16(u.w);
#pragma unroll
      for (int r = 0; r < kSkinnyRows; ++r) {
        const float4 xa = *reinterpret_cast<const float4*>(s_x + r * K + (kv << 3));
        const float4 xb = *reinterpret_cast<const float4*>(s_x + r * K + (kv << 3) + 4);
        acc[r] += xa.x * w0.x + xa.y * w0.y + xa.z * w1.x + xa.w * w1.y + xb.x * w2.x +
                  xb.y * w2.y + xb.z * w3.x + xb.w * w3.y;
      }
    }
    // butterfly: after offsets 16,8,4,2 each lane holds one of the 16 row sums
#pragma unroll
    for (int off = 16, cnt = kSkinnyRows; off >= 2; off >>= 1) {
      cnt >>= 1;
      const bool hi = (lane & off) != 0;
#pragma unroll
      for (int j = 0; j < cnt; ++j) {
        const float send = hi ? acc[j] : acc[j + cnt];
        const float keep = hi ? acc[j + cnt] : acc[j];
        acc[j] = keep + __shfl_xor_sync(0xffffffffu, send, off);
      }
    }
    acc[0] += __shfl_xor_sync(0xffffffffu, acc[0], 1);
    const int r = ((lane & 16) ? 8 : 0) + ((lane & 8) ? 4 : 0) + ((lane & 4) ? 2 : 0) +
                  ((lane & 2) ? 1 : 0);
    if ((lane & 1) == 0 && b0 + r < B) {
      float v = acc[0] + (bias ? bias[n] : 0.f);
      y[static_cast<size_t>(b0 + r) * ldy + n] = apply_act(v, out_act);
    }
  }
}

// ---------------------------------------------------------------------- time_features
__global__ void time_features_kernel(const float* __restrict__ sigma,
                                     const float* __restrict__ freqs, float* __restrict__ out,
                                     int B, int nfreq, int ld_out) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x;
  const float s = sigma[b];
  for (int j = threadIdx.x; j < ld_out; j += blockDim.x) {
    float v = 0.f;
    if (j == 0) v = s;
    else if (j <= nfreq) v = sinf(s * freqs[j - 1] * 2.f * 3.14159265358979323846f);
    else if (j <= 2 * nfreq) v = cosf(s * freqs[j - 1 - nfreq] * 2.f * 3.14159265358979323846f);
    out[static_cast<size_t>(b) * ld_out + j] = v;
  }
}

// ----------------------------------------------------------------------- sampler_step
__global__ void sampler_step_kernel(const float* __restrict__ x, const float* __restrict__ v,
                                    const float* __restrict__ ab, float* __restrict__ xn,
                                    int64_t n) {
  pdl_launch_dependents();
  pdl_wait();
  const float a0 = ab[0], b0 = ab[1], a1 = ab[2], b1 = ab[3];
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float xv = x[i], vv = v[i];
    const float x_pred = a0 * xv - b0 * vv;   // reference diffusion.py:185
    const float n_pred = b0 * xv + a0 * vv;   // :186
    xn[i] = a1 * x_pred + b1 * n_pred;        // :187
  }
}

// Per-step inputs of the captured sampling step, selected ON THE DEVICE: the step graph is the same
// for every step (and several steps can be captured back to back), the host only replays it.
//   ctrl[0] = address of the conditioning table rows [n][ss_elems] (fp32), ctrl[1] = steps that
//   share one table row (VInpainter resamples), ctrl[2] = n (rows; the index is clamped to it, so a
//   replay past the end of the block re-uses the last row instead of reading out of bounds),
//   step = iterations done since the host reset it
__global__ void step_select_kernel(const int* __restrict__ step, const long long* __restrict__ ctrl,
                                   const float* __restrict__ ab_table, float* __restrict__ ab_out,
                                   float* __restrict__ ss_out, int64_t ss_elems) {
  pdl_launch_dependents();
  pdl_wait();
  const float* table = reinterpret_cast<const float*>(ctrl[0]);
  const long long div = ctrl[1] > 0 ? ctrl[1] : 1;
  const long long n_it = (ctrl[2] > 0 ? ctrl[2] : 1) * div;
  const long long it = *step < n_it ? *step : n_it - 1;
  const float4* src = reinterpret_cast<const float4*>(table + static_cast<size_t>(it / div) * ss_elems);
  float4* dst = reinterpret_cast<float4*>(ss_out);
  const int64_t n4 = ss_elems >> 2;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    dst[i] = src[i];
  if (blockIdx.x == 0 && threadIdx.x < 4) ab_out[threadIdx.x] = ab_table[static_cast<size_t>(it) * 4 + threadIdx.x];
}
__global__ void step_advance_kernel(int* step) {
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x == 0) *step += 1;
}

// VInpainter (reference diffusion.py:349-350): where mask, x := a1*source + b1*noise (the known
// region re-noised to the level the sampler just stepped to); elsewhere x keeps the sampler's value
__global__ void inpaint_blend_kernel(float* __restrict__ x, const float* __restrict__ source,
                                     const float* __restrict__ noise, const uint8_t* __restrict__ mask,
                                     const float* __restrict__ ab, int64_t n) {
  pdl_launch_dependents();
  pdl_wait();
  const float a1 = ab[2], b1 = ab[3];
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    if (mask[i]) x[i] = a1 * source[i] + b1 * noise[i];
}

// ARVSampler step (reference diffusion.py:231-235): every position carries its own noise level.
// chan fp32 [B, C+1, T] is the net input: channels 0..C-1 = current, channel C = sigma_i.  With
// a = cos(sigma pi/2), b = sin(sigma pi/2):  x_pred = a_i x - b_i v, n_pred = b_i x + a_i v,
// current' = a_n x_pred + b_n n_pred; current' and sigma_{i+1} are written back into chan, which
// is then the next step's net input.  One thread per (batch, position).
__global__ void arv_step_kernel(float* __restrict__ chan, const float* __restrict__ v,
                                const float* __restrict__ sig_next, int B, int C, int T) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t n = static_cast<int64_t>(B) * T;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int b = static_cast<int>(i / T);
    const int t = static_cast<int>(i - static_cast<int64_t>(b) * T);
    float* cb = chan + static_cast<size_t>(b) * (C + 1) * T + t;
    const float* vb = v + static_cast<size_t>(b) * C * T + t;
    const float s0 = cb[static_cast<size_t>(C) * T], s1 = sig_next[i];
    const float a0 = cospif(0.5f * s0), b0 = sinpif(0.5f * s0);
    const float a1 = cospif(0.5f * s1), b1 = sinpif(0.5f * s1);
    for (int c = 0; c < C; ++c) {
      const float x = cb[static_cast<size_t>(c) * T], vv = vb[static_cast<size_t>(c) * T];
      const float xp = a0 * x - b0 * vv, np = b0 * x + a0 * vv;
      cb[static_cast<size_t>(c) * T] = a1 * xp + b1 * np;
    }
    cb[static_cast<size_t>(C) * T] = s1;
  }
}

__global__ void silu_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                 int64_t n) {
  pdl_launch_dependents();
  pdl_wait();
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    y[i] = __float2bfloat16(silu_f(x[i]));
}

static int pick_grid(size_t work_items, int per_block, int cap) {
  size_t g = (work_items + per_block - 1) / per_block;
  if (g < 1) g = 1;
  if (g > static_cast<size_t>(cap)) g = cap;
  return static_cast<int>(g);
}

}  // namespace adp

using namespace adp;

extern "C" int adp_gn_silu(const void* x, void* y, const double* stats, const float* gamma,
                           const float* beta, int32_t B, int32_t T, int32_t C, int32_t groups,
                           float eps, adp_stream_t stream) {
  ADP_CHECK(x && y && stats && gamma && beta, "adp_gn_silu: null pointer");
  ADP_CHECK(C % 8 == 0 && C <= kMaxC && groups > 0 && C % groups == 0,
            "adp_gn_silu: C=%d groups=%d unsupported", C, groups);
  const size_t nvec = static_cast<size_t>(T) * (C / 8);
  ADP_CHECK(nvec < (1ull << 31), "adp_gn_silu: T*C/8 = %zu does not fit 31 bits", nvec);
  const int vpr = C / 8;
  const bool reg = vpr <= 256 && (vpr & (vpr - 1)) == 0;
  // small tensors (the deep levels) are latency-bound: one vector per thread, many blocks
  const bool small = static_cast<size_t>(B) * nvec <= static_cast<size_t>(num_sms()) * 2048 * 2;
  const int tile = small ? 256 : 1024;
  dim3 grid(pick_grid(nvec, tile, num_sms() * 16 / (B < 16 ? B : 16) + 1), B);
#define ADP_GN(REG, NV)                                                                         \
  ADP_CUDA(launch_k(gn_silu_kernel<REG, NV>, grid, dim3(256), (size_t)0, as_stream(stream),     \
                    static_cast<const uint4*>(x), static_cast<uint4*>(y), stats, gamma, beta,    \
                    (int)T, (int)C, (int)groups, eps))
  if (reg && small) ADP_GN(true, 1);
  else if (reg) ADP_GN(true, 4);
  else if (small) ADP_GN(false, 1);
  else ADP_GN(false, 4);
#undef ADP_GN
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_gn_stats(const void* x, double* stats, int32_t B, int32_t T, int32_t C,
                            int32_t groups, adp_stream_t stream) {
  ADP_CHECK(x && stats, "adp_gn_stats: null pointer");
  ADP_CHECK(C % 8 == 0 && C <= 2048 && groups > 0 && groups <= 64 && C % groups == 0,
            "adp_gn_stats: C=%d groups=%d unsupported", C, groups);
  const size_t nvec = static_cast<size_t>(T) * (C / 8);
  dim3 grid(pick_grid(nvec, 256 * 8, num_sms() * 8 / (B < 8 ? B : 8) + 1), B);
  ADP_CUDA(launch_k(gn_stats_kernel, grid, dim3(256), (size_t)0, as_stream(stream),
                    static_cast<const uint4*>(x), stats, (int)T, (int)C, (int)groups));
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_ln_film(const void* x, void* y, const float* scale_shift, int32_t ss_stride,
                           double* stats_out, int32_t B, int32_t T, int32_t C, int32_t groups,
                           float eps, adp_stream_t stream) {
  return adp_ln_film_dual(x, y, nullptr, scale_shift, ss_stride, stats_out, B, T, C, groups, eps,
                          0.f, stream);
}

extern "C" int adp_ln_film_dual(const void* x, void* y, void* y2, const float* scale_shift,
                                int32_t ss_stride, double* stats_out, int32_t B, int32_t T,
                                int32_t C, int32_t groups, float eps, float eps2,
                                adp_stream_t stream) {
  ADP_CHECK(x && y, "adp_ln_film: null pointer");
  ADP_CHECK(C % 8 == 0, "adp_ln_film: C=%d must be a multiple of 8", C);
  const int vpr = C / 8;
  int lpr, vpl;
  if (vpr <= 32) {
    ADP_CHECK((vpr & (vpr - 1)) == 0, "adp_ln_film: C/8=%d must be a power of two (<=32)", vpr);
    lpr = vpr; vpl = 1;
  } else {
    ADP_CHECK(vpr % 32 == 0 && vpr / 32 <= 4, "adp_ln_film: C=%d unsupported (need C%%256==0, "
              "C<=1024)", C);
    lpr = 32; vpl = vpr / 32;
  }
  bool per_ch = false;
  if (stats_out) {
    ADP_CHECK(groups > 0 && groups <= 64 && C % groups == 0, "adp_ln_film: groups=%d", groups);
    const int gsz = C / groups;
    per_ch = gsz < 8;
    ADP_CHECK(per_ch ? (vpl == 1) : (gsz % 8 == 0), "adp_ln_film: group size %d unsupported", gsz);
  }
  ADP_CHECK(C <= kMaxLnC, "adp_ln_film: C=%d > %d", C, kMaxLnC);
  const int unr = vpl <= 2 ? 2 : 1;
  const int rows_per_block = 8 * (32 / lpr) * unr;
  // deep levels have few rows: one pass per warp (all SMs busy) instead of two
  const bool few = static_cast<size_t>(B) * ((T + rows_per_block - 1) / rows_per_block) <= num_sms() * 4;
  dim3 grid(pick_grid(T, few ? rows_per_block : rows_per_block * 2, num_sms() * 16 / (B < 16 ? B : 16) + 1), B);
  const uint4* xi = static_cast<const uint4*>(x);
  uint4* yo = static_cast<uint4*>(y);
  cudaStream_t s = as_stream(stream);
#define ADP_LN(VPL, PC)                                                                         \
  ADP_CUDA(launch_k(ln_film_kernel<VPL, PC, (VPL <= 2 ? 2 : 1)>, grid, dim3(256), (size_t)0, s, \
                    xi, yo, scale_shift, (int)ss_stride, stats_out, (int)T, (int)C, (int)lpr,   \
                    (int)groups, eps, static_cast<uint4*>(y2), eps2))
  if (per_ch) ADP_LN(1, true);
  else if (vpl == 1) ADP_LN(1, false);
  else if (vpl == 2) ADP_LN(2, false);
  else if (vpl == 3) ADP_LN(3, false);
  else ADP_LN(4, false);
#undef ADP_LN
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_skinny_linear(const float* x, const void* w, const float* bias, float* y,
                                 int32_t B, int32_t K, int32_t N, int32_t ldx, int32_t ldw,
                                 int32_t ldy, int32_t in_act, int32_t out_act,
                                 adp_stream_t stream) {
  ADP_CHECK(x && w && y, "adp_skinny_linear: null pointer");
  ADP_CHECK(K % 8 == 0 && ldw % 8 == 0 && K <= 3072 && K <= ldx && K <= ldw,
            "adp_skinny_linear: K=%d ldx=%d ldw=%d unsupported", K, ldx, ldw);
  const size_t smem = static_cast<size_t>(kSkinnyRows) * K * sizeof(float);
  static SmemAttrCache smem_cache;
  ADP_CUDA(ensure_dyn_smem(skinny_linear_kernel, smem, smem_cache));
  dim3 grid(pick_grid(N, 8, num_sms() * 2), (B + kSkinnyRows - 1) / kSkinnyRows);
  ADP_CUDA(launch_k(skinny_linear_kernel, grid, dim3(256), smem, as_stream(stream), x,
                    static_cast<const __nv_bfloat16*>(w), bias, y, (int)B, (int)K, (int)N, (int)ldx,
                    (int)ldw, (int)ldy, (int)in_act, (int)out_act));
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_time_features(const float* sigma, const float* freqs, float* out, int32_t B,
                                 int32_t nfreq, int32_t ld_out, adp_stream_t stream) {
  ADP_CHECK(sigma && freqs && out && ld_out >= 2 * nfreq + 1, "adp_time_features: bad args");
  ADP_CUDA(launch_k(time_features_kernel, dim3(B), dim3(128), (size_t)0, as_stream(stream), sigma,
                    freqs, out, (int)B, (int)nfreq, (int)ld_out));
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_silu_bf16(const float* x, void* y, int64_t n, adp_stream_t stream) {
  ADP_CHECK(x && y && n > 0, "adp_silu_bf16: bad args");
  ADP_CUDA(launch_k(silu_bf16_kernel, dim3(pick_grid(static_cast<size_t>(n), 256, num_sms() * 4)),
                    dim3(256), (size_t)0, as_stream(stream), x, static_cast<__nv_bfloat16*>(y), n));
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_step_select(const int32_t* step, const int64_t* ctrl, const float* ab_table,
                               float* ab_out, float* ss_out, int64_t ss_elems, adp_stream_t stream) {
  ADP_CHECK(step && ctrl && ab_table && ab_out && ss_out && ss_elems > 0 && ss_elems % 4 == 0,
            "adp_step_select: bad args");
  ADP_CUDA(launch_k(step_select_kernel, dim3(pick_grid(static_cast<size_t>(ss_elems / 4), 256 * 4, num_sms() * 4)),
                    dim3(256), (size_t)0, as_stream(stream), step, reinterpret_cast<const long long*>(ctrl),
                    ab_table, ab_out, ss_out, ss_elems));
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_step_advance(int32_t* step, adp_stream_t stream) {
  ADP_CHECK(step != nullptr, "adp_step_advance: null");
  ADP_CUDA(launch_k(step_advance_kernel, dim3(1), dim3(32), (size_t)0, as_stream(stream), step));
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_inpaint_blend(float* x, const float* source, const float* noise, const uint8_t* mask,
                                 const float* ab, int64_t n, adp_stream_t stream) {
  ADP_CHECK(x && source && noise && mask && ab && n > 0, "adp_inpaint_blend: bad args");
  ADP_CUDA(launch_k(inpaint_blend_kernel, dim3(pick_grid(static_cast<size_t>(n), 256 * 4, num_sms() * 8)),
                    dim3(256), (size_t)0, as_stream(stream), x, source, noise, mask, ab, n));
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_arv_step(float* chan, const float* v, const float* sig_next, int B, int C, int T,
                            adp_stream_t stream) {
  ADP_CHECK(chan && v && sig_next && B > 0 && C > 0 && T > 0, "adp_arv_step: bad args");
  ADP_CUDA(launch_k(arv_step_kernel, dim3(pick_grid(static_cast<size_t>(B) * T, 256, num_sms() * 8)), dim3(256),
                    (size_t)0, as_stream(stream), chan, v, sig_next, B, C, T));
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_sampler_step(const float* x, const float* v, const float* ab, float* x_next,
                                int64_t n, adp_stream_t stream) {
  ADP_CHECK(x && v && ab && x_next && n > 0, "adp_sampler_step: bad args");
  ADP_CUDA(launch_k(sampler_step_kernel, dim3(pick_grid(static_cast<size_t>(n), 256 * 4, num_sms() * 8)),
                    dim3(256), (size_t)0, as_stream(stream), x, v, ab, x_next, n));
  ADP_LAUNCH_CHECK();
  return 0;
}
