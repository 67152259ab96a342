// Bandwidth-bound backward kernels of the UNetV0 training step (CUDA cores):
//   adp_gn_silu_bwd / adp_gn_bwd_apply   GroupNorm+SiLU backward (two passes: sums, apply)
//   adp_ln_film_bwd                      LayerNorm_C + FiLM backward (a_unet Modulation)
//   adp_colsum                           per-channel sums (conv bias gradients)
//   adp_skip_gate / adp_skip_gate_bwd    MergeModulate  out = skip + gate*y  (training forward)
//   adp_cond_bwd                         the concatenated conditioning projection backward
// All activations / activation gradients are channels-last bf16; parameter gradients and
// statistics accumulate in fp32 / fp64 with atomics (pre-zeroed by the caller).
#include "common.cuh"
#include "ptx.cuh"

namespace adp {

constexpr int kBwMaxC = 1024;

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  const float2 a = unpack_bf16(u.x), b = unpack_bf16(u.y), c = unpack_bf16(u.z), d = unpack_bf16(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  return make_uint4(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]),
                    pack_bf16(f[6], f[7]));
}

// The streaming kernels below give every thread 8 fixed channels (c0 = (global tid % vpr) * 8,
// vpr = C/8 vectors per row).  When vpr < 32 the lanes l, l+vpr, l+2vpr, ... of a warp own the
// SAME channels: fold their partial sums with shuffles so that one lane per channel touches the
// block's shared-memory bins (at C = 32 the unfolded version sent 64 threads to every bin and
// the kernel ran far below HBM bandwidth).
__device__ __forceinline__ bool fold_ok(int vpr) { return vpr < 32 && (32 % vpr) == 0; }
__device__ __forceinline__ float fold_lanes(float v, int vpr) {
  for (int o = vpr; o < 32; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// per-(batch, channel) GroupNorm coefficients -> smem: mean[c], rstd[c]
__device__ __forceinline__ void gn_coeffs(const double* stats, int b, int T, int C, int groups,
                                          float eps, float* s_mean, float* s_rstd) {
  const int gsz = C / groups;
  const double inv_n = 1.0 / (static_cast<double>(gsz) * T);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int g = c / gsz;
    const double s = stats[(static_cast<size_t>(b) * groups + g) * 2];
    const double q = stats[(static_cast<size_t>(b) * groups + g) * 2 + 1];
    const double mean = s * inv_n;
    const float var = fmaxf(static_cast<float>(q * inv_n - mean * mean), 0.f);
    s_mean[c] = static_cast<float>(mean);
    s_rstd[c] = rsqrtf(var + eps);
  }
}

// ----------------------------------------------------------------------- gn_silu_bwd
// a = silu(z), z = xhat*gamma + beta.  Given da: dz = da*silu'(z); writes dxh = dz*gamma and
// accumulates dgamma += sum dz*xhat, dbeta += sum dz, S[b,g] += (sum dxh, sum dxh*xhat).
__global__ void __launch_bounds__(256)
gn_silu_bwd_kernel(const uint4* __restrict__ da, const uint4* __restrict__ x,
                   const double* __restrict__ stats, const float* __restrict__ gamma,
                   const float* __restrict__ beta, uint4* __restrict__ dxh,
                   float* __restrict__ dgamma, float* __restrict__ dbeta, double* __restrict__ S,
                   int T, int C, int groups, float eps) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float s_mean[kBwMaxC], s_rstd[kBwMaxC];
  __shared__ float s_dg[kBwMaxC], s_db[kBwMaxC];
  __shared__ float s_s1[kBwMaxC], s_s2[kBwMaxC];      // per-channel sums of dxh, dxh*xhat
  const int b = blockIdx.y;
  gn_coeffs(stats, b, T, C, groups, eps, s_mean, s_rstd);
  for (int c = threadIdx.x; c < C; c += blockDim.x) { s_dg[c] = 0.f; s_db[c] = 0.f; s_s1[c] = 0.f; s_s2[c] = 0.f; }
  __syncthreads();
  const int gsz = C / groups;
  const int vpr = C >> 3;
  const size_t nvec = static_cast<size_t>(T) * vpr;
  const uint4* dab = da + static_cast<size_t>(b) * nvec;
  const uint4* xb = x + static_cast<size_t>(b) * nvec;
  uint4* ob = dxh + static_cast<size_t>(b) * nvec;
  // per-thread stride is a multiple of vectors-per-row: the thread's 8 channels never change
  const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t stride = (nthreads + vpr - 1) / vpr * vpr;
  const int c0 = static_cast<int>(tid % vpr) << 3;
  float g8[8], b8[8], m8[8], r8[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    g8[j] = gamma[c0 + j]; b8[j] = beta[c0 + j]; m8[j] = s_mean[c0 + j]; r8[j] = s_rstd[c0 + j];
  }
  float adg[8], adb[8], as1[8], as2[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { adg[j] = 0.f; adb[j] = 0.f; as1[j] = 0.f; as2[j] = 0.f; }
  for (size_t i = tid; i < nvec; i += stride) {
    float fa[8], fx[8], o[8];
    unpack8(__ldg(dab + i), fa);
    unpack8(__ldg(xb + i), fx);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float xh = (fx[j] - m8[j]) * r8[j];
      const float z = xh * g8[j] + b8[j];
      const float sg = 1.f / (1.f + __expf(-z));
      const float dz = fa[j] * sg * (1.f + z * (1.f - sg));
      o[j] = dz * g8[j];
      adg[j] += dz * xh; adb[j] += dz;
    }
    const uint4 ov = pack8(o);
    ob[i] = ov;
    float orr[8];
    unpack8(ov, orr);                       // sums of what the second pass will read
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float xh = (fx[j] - m8[j]) * r8[j];
      as1[j] += orr[j]; as2[j] += orr[j] * xh;
    }
  }
  {
    const bool fold = fold_ok(vpr);
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float v0 = adg[j], v1 = adb[j], v2 = as1[j], v3 = as2[j];
      if (fold) {
        v0 = fold_lanes(v0, vpr); v1 = fold_lanes(v1, vpr);
        v2 = fold_lanes(v2, vpr); v3 = fold_lanes(v3, vpr);
      }
      if (!fold || lane < vpr) {
        atomicAdd(&s_dg[c0 + j], v0);
        atomicAdd(&s_db[c0 + j], v1);
        atomicAdd(&s_s1[c0 + j], v2);
        atomicAdd(&s_s2[c0 + j], v3);
      }
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    atomicAdd(dgamma + c, s_dg[c]);
    atomicAdd(dbeta + c, s_db[c]);
  }
  if (threadIdx.x < 2 * groups) {      // thread (g, which) sums its group's channels: no contention
    const int g = threadIdx.x >> 1, which = threadIdx.x & 1;
    const float* src = which ? s_s2 : s_s1;
    float tot = 0.f;
    for (int c = g * gsz; c < (g + 1) * gsz; ++c) tot += src[c];
    atomicAdd(S + static_cast<size_t>(b) * 2 * groups + threadIdx.x, static_cast<double>(tot));
  }
}

// ---------------------------------------------------------------------- gn_bwd_apply
// dx = rstd * (dxh - S1/n - xhat * S2/n) [+ dres];  optional colsum[c] += sum dx.
__global__ void __launch_bounds__(256)
gn_bwd_apply_kernel(const uint4* __restrict__ dxh, const uint4* __restrict__ x,
                    const double* __restrict__ stats, const double* __restrict__ S,
                    const uint4* __restrict__ dres, uint4* __restrict__ dx,
                    float* __restrict__ colsum, int T, int C, int groups, float eps) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float s_mean[kBwMaxC], s_rstd[kBwMaxC], s_c1[kBwMaxC], s_c2[kBwMaxC];
  __shared__ float s_cs[kBwMaxC];
  const int b = blockIdx.y;
  gn_coeffs(stats, b, T, C, groups, eps, s_mean, s_rstd);
  const int gsz = C / groups;
  const double inv_n = 1.0 / (static_cast<double>(gsz) * T);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int g = c / gsz;
    s_c1[c] = static_cast<float>(S[(static_cast<size_t>(b) * groups + g) * 2] * inv_n);
    s_c2[c] = static_cast<float>(S[(static_cast<size_t>(b) * groups + g) * 2 + 1] * inv_n);
    s_cs[c] = 0.f;
  }
  __syncthreads();
  const int vpr = C >> 3;
  const size_t nvec = static_cast<size_t>(T) * vpr;
  const size_t boff = static_cast<size_t>(b) * nvec;
  const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t stride = (nthreads + vpr - 1) / vpr * vpr;
  const int c0 = static_cast<int>(tid % vpr) << 3;
  float acs[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acs[j] = 0.f;
  for (size_t i = tid; i < nvec; i += stride) {
    float fd[8], fx[8], fr[8], o[8];
    unpack8(__ldg(dxh + boff + i), fd);
    unpack8(__ldg(x + boff + i), fx);
    if (dres) unpack8(__ldg(dres + boff + i), fr);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = c0 + j;
      const float xh = (fx[j] - s_mean[c]) * s_rstd[c];
      o[j] = s_rstd[c] * (fd[j] - s_c1[c] - xh * s_c2[c]);
      if (dres) o[j] += fr[j];
    }
    const uint4 ov = pack8(o);
    dx[boff + i] = ov;
    if (colsum) {
      float orr[8];
      unpack8(ov, orr);
#pragma unroll
      for (int j = 0; j < 8; ++j) acs[j] += o[j];   // bias gradients sum the unrounded fp32 values
    }
  }
  if (colsum) {
    const bool fold = fold_ok(vpr);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float v = fold ? fold_lanes(acs[j], vpr) : acs[j];
      if (!fold || (threadIdx.x & 31) < vpr) atomicAdd(&s_cs[c0 + j], v);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) atomicAdd(colsum + c, s_cs[c]);
  }
}

// ----------------------------------------------------------------------- ln_film_bwd
// y = xhat*(1+s) + t per row.  dx = rstd*(g - mean(g) - xhat*mean(g*xhat)), g = dy*(1+s);
// dss[b, c] += sum_t dy*xhat, dss[b, C+c] += sum_t dy;  optional colsum[c] += sum dx.
template <int VPL>
__global__ void __launch_bounds__(256)
ln_film_bwd_kernel(const uint4* __restrict__ dy, const uint4* __restrict__ x,
                   const float* __restrict__ ss, int ss_stride, uint4* __restrict__ dx,
                   float* __restrict__ dss, int dss_stride, float* __restrict__ colsum,
                   const uint4* __restrict__ dres, int T, int C, int lpr, float eps) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ __align__(16) float s_fs[kBwMaxC];
  __shared__ float s_ds[kBwMaxC], s_dt[kBwMaxC], s_cs[kBwMaxC];
  const int b = blockIdx.y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int rpw = 32 / lpr, sub = lane / lpr, l = lane - sub * lpr;
  const int vpr = C >> 3;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    s_fs[c] = ss ? 1.f + ss[static_cast<size_t>(b) * ss_stride + c] : 1.f;
    s_ds[c] = 0.f; s_dt[c] = 0.f; s_cs[c] = 0.f;
  }
  __syncthreads();
  float ads[VPL][8], adt[VPL][8], acs[VPL][8];
#pragma unroll
  for (int it = 0; it < VPL; ++it)
#pragma unroll
    for (int j = 0; j < 8; ++j) { ads[it][j] = 0.f; adt[it][j] = 0.f; acs[it][j] = 0.f; }
  const size_t boff = static_cast<size_t>(b) * T * vpr;
  const int warps_total = gridDim.x * (blockDim.x >> 5);
  const float inv_c = 1.f / static_cast<float>(C);
  for (int base = (blockIdx.x * (blockDim.x >> 5) + warp) * rpw; base < T; base += warps_total * rpw) {
    const int row = base + sub;
    const bool ok = row < T;
    float vx[VPL][8], vg[VPL][8], vd[VPL][8];
    float sum = 0.f;
#pragma unroll
    for (int it = 0; it < VPL; ++it) {
      uint4 ux = make_uint4(0, 0, 0, 0), ud = make_uint4(0, 0, 0, 0);
      if (ok) {
        ux = __ldg(x + boff + static_cast<size_t>(row) * vpr + it * lpr + l);
        ud = __ldg(dy + boff + static_cast<size_t>(row) * vpr + it * lpr + l);
      }
      unpack8(ux, vx[it]);
      unpack8(ud, vd[it]);
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += vx[it][j];
    }
    for (int o = lpr >> 1; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum * inv_c;
    float sq = 0.f;
#pragma unroll
    for (int it = 0; it < VPL; ++it)
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float d = vx[it][j] - mean; sq += d * d; }
    for (int o = lpr >> 1; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    const float rstd = rsqrtf(sq * inv_c + eps);
    float m1 = 0.f, m2 = 0.f;
#pragma unroll
    for (int it = 0; it < VPL; ++it) {
      const int c = (it * lpr + l) << 3;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float xh = (vx[it][j] - mean) * rstd;
        vx[it][j] = xh;
        const float g = vd[it][j] * s_fs[c + j];
        vg[it][j] = g;
        m1 += g; m2 += g * xh;
        if (ok) { ads[it][j] += vd[it][j] * xh; adt[it][j] += vd[it][j]; }
      }
    }
    for (int o = lpr >> 1; o > 0; o >>= 1) {
      m1 += __shfl_xor_sync(0xffffffffu, m1, o);
      m2 += __shfl_xor_sync(0xffffffffu, m2, o);
    }
    m1 *= inv_c; m2 *= inv_c;
#pragma unroll
    for (int it = 0; it < VPL; ++it) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = rstd * (vg[it][j] - m1 - vx[it][j] * m2);
      if (dres != nullptr && ok) {        // gradient arriving on a parallel (residual) path
        float fr[8];
        unpack8(__ldg(dres + boff + static_cast<size_t>(row) * vpr + it * lpr + l), fr);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] += fr[j];
      }
      const uint4 ov = pack8(o);
      if (ok) {
        dx[boff + static_cast<size_t>(row) * vpr + it * lpr + l] = ov;
        if (colsum) {
          float orr[8];
          unpack8(ov, orr);
#pragma unroll
          for (int j = 0; j < 8; ++j) acs[it][j] += o[j];
        }
      }
    }
  }
  // lanes l, l+lpr, ... hold the same channels: fold, then one smem atomic per channel
#pragma unroll
  for (int it = 0; it < VPL; ++it)
#pragma unroll
    for (int j = 0; j < 8; ++j)
      for (int o = lpr; o < 32; o <<= 1) {
        ads[it][j] += __shfl_xor_sync(0xffffffffu, ads[it][j], o);
        adt[it][j] += __shfl_xor_sync(0xffffffffu, adt[it][j], o);
        acs[it][j] += __shfl_xor_sync(0xffffffffu, acs[it][j], o);
      }
  if (sub == 0) {
#pragma unroll
    for (int it = 0; it < VPL; ++it)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = ((it * lpr + l) << 3) + j;
        atomicAdd(&s_ds[c], ads[it][j]);
        atomicAdd(&s_dt[c], adt[it][j]);
        atomicAdd(&s_cs[c], acs[it][j]);
      }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    if (dss) {
      atomicAdd(dss + static_cast<size_t>(b) * dss_stride + c, s_ds[c]);
      atomicAdd(dss + static_cast<size_t>(b) * dss_stride + C + c, s_dt[c]);
    }
    if (colsum) atomicAdd(colsum + c, s_cs[c]);
  }
}

// ---------------------------------------------------------------------------- colsum
constexpr int kColsumMaxC = 2048;     // fused q|k|v gradient rows are 3*512 wide
__global__ void __launch_bounds__(256)
colsum_kernel(const uint4* __restrict__ x, const float* __restrict__ gate, int ld_gate,
              float* __restrict__ out, int T, int C) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float s_cs[kColsumMaxC];
  const int b = blockIdx.y;
  for (int c = threadIdx.x; c < C; c += blockDim.x) s_cs[c] = 0.f;
  __syncthreads();
  const int vpr = C >> 3;
  const size_t nvec = static_cast<size_t>(T) * vpr;
  const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t stride = (nthreads + vpr - 1) / vpr * vpr;
  const int c0 = static_cast<int>(tid % vpr) << 3;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  for (size_t i = tid; i < nvec; i += stride) {
    float f[8];
    unpack8(__ldg(x + static_cast<size_t>(b) * nvec + i), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] += f[j];
  }
  {
    const bool fold = fold_ok(vpr);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float v = gate ? acc[j] * gate[static_cast<size_t>(b) * ld_gate + c0 + j] : acc[j];
      if (fold) v = fold_lanes(v, vpr);
      if (!fold || (threadIdx.x & 31) < vpr) atomicAdd(&s_cs[c0 + j], v);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) atomicAdd(out + c, s_cs[c]);
}

// ------------------------------------------------------------------------- skip_gate
// forward (training): out = skip + gate[b,c]*y, with the GroupNorm statistics of out.
__global__ void __launch_bounds__(256)
skip_gate_kernel(const uint4* __restrict__ y, const uint4* __restrict__ skip,
                 const float* __restrict__ gate, int ld_gate, uint4* __restrict__ out,
                 double* __restrict__ stats, int T, int C, int groups) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float s_s1[kBwMaxC], s_s2[kBwMaxC];      // per-channel sum / sum of squares of out
  const int b = blockIdx.y;
  for (int c = threadIdx.x; c < C; c += blockDim.x) { s_s1[c] = 0.f; s_s2[c] = 0.f; }
  __syncthreads();
  const int vpr = C >> 3, gsz = groups > 0 ? C / groups : C;
  const size_t nvec = static_cast<size_t>(T) * vpr, boff = static_cast<size_t>(b) * nvec;
  const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t stride = (nthreads + vpr - 1) / vpr * vpr;
  const int c0 = static_cast<int>(tid % vpr) << 3;
  float g8[8], s1[8], s2[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { g8[j] = gate[static_cast<size_t>(b) * ld_gate + c0 + j]; s1[j] = 0.f; s2[j] = 0.f; }
  for (size_t i = tid; i < nvec; i += stride) {
    float fy[8], fs[8], o[8];
    unpack8(__ldg(y + boff + i), fy);
    unpack8(__ldg(skip + boff + i), fs);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = fs[j] + g8[j] * fy[j];
    const uint4 ov = pack8(o);
    out[boff + i] = ov;
    if (stats) {
      float orr[8];
      unpack8(ov, orr);
#pragma unroll
      for (int j = 0; j < 8; ++j) { s1[j] += orr[j]; s2[j] += orr[j] * orr[j]; }
    }
  }
  if (stats) {
    const bool fold = fold_ok(vpr);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float v1 = s1[j], v2 = s2[j];
      if (fold) { v1 = fold_lanes(v1, vpr); v2 = fold_lanes(v2, vpr); }
      if (!fold || (threadIdx.x & 31) < vpr) {
        atomicAdd(&s_s1[c0 + j], v1);
        atomicAdd(&s_s2[c0 + j], v2);
      }
    }
    __syncthreads();
    if (threadIdx.x < 2 * groups) {
      const int g = threadIdx.x >> 1, which = threadIdx.x & 1;
      const float* src = which ? s_s2 : s_s1;
      float tot = 0.f;
      for (int c = g * gsz; c < (g + 1) * gsz; ++c) tot += src[c];
      atomicAdd(stats + static_cast<size_t>(b) * 2 * groups + threadIdx.x, static_cast<double>(tot));
    }
  }
}

// backward: dys = gate*dout (bf16), dgate[b,c] += sum_t dout*y.  (d skip = dout, aliased)
__global__ void __launch_bounds__(256)
skip_gate_bwd_kernel(const uint4* __restrict__ dout, const uint4* __restrict__ y,
                     const float* __restrict__ gate, int ld_gate, uint4* __restrict__ dys,
                     float* __restrict__ dgate, int ld_dgate, int T, int C) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float s_dg[kBwMaxC];
  const int b = blockIdx.y;
  for (int c = threadIdx.x; c < C; c += blockDim.x) s_dg[c] = 0.f;
  __syncthreads();
  const int vpr = C >> 3;
  const size_t nvec = static_cast<size_t>(T) * vpr, boff = static_cast<size_t>(b) * nvec;
  const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t stride = (nthreads + vpr - 1) / vpr * vpr;
  const int c0 = static_cast<int>(tid % vpr) << 3;
  float g8[8], adg[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { g8[j] = gate[static_cast<size_t>(b) * ld_gate + c0 + j]; adg[j] = 0.f; }
  for (size_t i = tid; i < nvec; i += stride) {
    float fd[8], fy[8], o[8];
    unpack8(__ldg(dout + boff + i), fd);
    unpack8(__ldg(y + boff + i), fy);
#pragma unroll
    for (int j = 0; j < 8; ++j) { o[j] = g8[j] * fd[j]; adg[j] += fd[j] * fy[j]; }
    dys[boff + i] = pack8(o);
  }
  {
    const bool fold = fold_ok(vpr);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float v = fold ? fold_lanes(adg[j], vpr) : adg[j];
      if (!fold || (threadIdx.x & 31) < vpr) atomicAdd(&s_dg[c0 + j], v);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x)
    atomicAdd(dgate + static_cast<size_t>(b) * ld_dgate + c, s_dg[c]);
}

// -------------------------------------------------------------------------- cond_bwd
// ss[b][n] = sum_k cond[b][k] * W[n][k] + bias[n]:
//   dW[n][k] = sum_b dss[b][n]*cond[b][k],  dbias[n] = sum_b dss[b][n]
//   dcond[b][k] += sum_n dss[b][n]*W[n][k]
// Pure streaming (W read once as bf16, dW written once as fp32): every thread owns 4 consecutive
// k, so W arrives as 8-byte and dW leaves as 16-byte vectors; cond[.][k..k+3] stays in registers.
constexpr int kCondMaxB = 8;          // batch rows per pass of the in-graph (local) call
constexpr int kCondGatherB = 32;      // ... of the data-parallel call on all-gathered rows (no dcond)
template <int MAXB, bool DC>
__global__ void __launch_bounds__(256)
cond_bwd_kernel(const float* __restrict__ dss, int ld_dss, const float* __restrict__ cond,
                const __nv_bfloat16* __restrict__ w, float* __restrict__ dw,
                float* __restrict__ dbias, float* __restrict__ dcond, int B, int N, int K,
                int rows_per_block, int accumulate) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float s_d[];       // dss slab [MAXB][rows_per_block], zero beyond B
  const int n0 = blockIdx.x * rows_per_block;
  const int nr = min(rows_per_block, N - n0);
  for (int i = threadIdx.x; i < MAXB * rows_per_block; i += blockDim.x) {
    const int bb = i / rows_per_block, r = i - bb * rows_per_block;
    s_d[i] = (bb < B && r < nr) ? dss[static_cast<size_t>(bb) * ld_dss + n0 + r] : 0.f;
  }
  __syncthreads();
  if (threadIdx.x < nr) {
    float t = 0.f;
    for (int bb = 0; bb < B; ++bb) t += s_d[bb * rows_per_block + threadIdx.x];
    dbias[n0 + threadIdx.x] = accumulate ? dbias[n0 + threadIdx.x] + t : t;
  }
  for (int k4 = threadIdx.x * 4; k4 < K; k4 += blockDim.x * 4) {
    float4 c4[MAXB], dc[DC ? MAXB : 1];
#pragma unroll
    for (int bb = 0; bb < MAXB; ++bb) {
      c4[bb] = bb < B ? *reinterpret_cast<const float4*>(cond + static_cast<size_t>(bb) * K + k4)
                      : make_float4(0.f, 0.f, 0.f, 0.f);
      if constexpr (DC) dc[bb] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll 2
    for (int r = 0; r < nr; ++r) {
      const uint2 wu = __ldg(reinterpret_cast<const uint2*>(w + static_cast<size_t>(n0 + r) * K + k4));
      const float2 w01 = unpack_bf16(wu.x), w23 = unpack_bf16(wu.y);
      float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int bb = 0; bb < MAXB; ++bb) {
        const float d = s_d[bb * rows_per_block + r];       // zero rows beyond B: no branch needed
        g.x += d * c4[bb].x; g.y += d * c4[bb].y; g.z += d * c4[bb].z; g.w += d * c4[bb].w;
        if constexpr (DC) {
          dc[bb].x += d * w01.x; dc[bb].y += d * w01.y; dc[bb].z += d * w23.x; dc[bb].w += d * w23.y;
        }
      }
      float4* dwp = reinterpret_cast<float4*>(dw + static_cast<size_t>(n0 + r) * K + k4);
      if (accumulate) {
        const float4 o = *dwp;
        g.x += o.x; g.y += o.y; g.z += o.z; g.w += o.w;
      }
      *dwp = g;
    }
    if constexpr (DC) {
#pragma unroll
      for (int bb = 0; bb < MAXB; ++bb)
        if (bb < B) {
          float* dp = dcond + static_cast<size_t>(bb) * K + k4;
          atomicAdd(dp, dc[bb].x); atomicAdd(dp + 1, dc[bb].y);
          atomicAdd(dp + 2, dc[bb].z); atomicAdd(dp + 3, dc[bb].w);
        }
    }
  }
}

static int grid_for(size_t nvec, int B) {
  // every block ends in 2C global atomics: a few hundred blocks in total, each streaming many rows
  size_t g = (nvec + 256 * 4 - 1) / (256 * 4);
  const size_t cap = num_sms() * 3 / (B < 8 ? B : 8) + 1;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return static_cast<int>(g);
}

}  // namespace adp

using namespace adp;

extern "C" int adp_gn_silu_bwd(const void* da, const void* x, const double* stats,
                               const float* gamma, const float* beta, void* dxh, float* dgamma,
                               float* dbeta, double* S, int32_t B, int32_t T, int32_t C,
                               int32_t groups, float eps, adp_stream_t stream) {
  ADP_CHECK(da && x && stats && gamma && beta && dxh && dgamma && dbeta && S, "adp_gn_silu_bwd: null");
  ADP_CHECK(C % 8 == 0 && C <= kBwMaxC && groups > 0 && groups <= 64 && C % groups == 0,
            "adp_gn_silu_bwd: C=%d groups=%d", C, groups);
  dim3 grid(grid_for(static_cast<size_t>(T) * (C / 8), B), B);
  ADP_CUDA(launch_k(gn_silu_bwd_kernel, grid, dim3(256), (size_t)0, as_stream(stream),
                    static_cast<const uint4*>(da), static_cast<const uint4*>(x), stats, gamma, beta,
                    static_cast<uint4*>(dxh), dgamma, dbeta, S, (int)T, (int)C, (int)groups, eps));
  return 0;
}

extern "C" int adp_gn_bwd_apply(const void* dxh, const void* x, const double* stats,
                                const double* S, const void* dres, void* dx, float* colsum,
                                int32_t B, int32_t T, int32_t C, int32_t groups, float eps,
                                adp_stream_t stream) {
  ADP_CHECK(dxh && x && stats && S && dx, "adp_gn_bwd_apply: null");
  ADP_CHECK(C % 8 == 0 && C <= kBwMaxC && groups > 0 && C % groups == 0, "adp_gn_bwd_apply: C=%d", C);
  dim3 grid(grid_for(static_cast<size_t>(T) * (C / 8), B), B);
  ADP_CUDA(launch_k(gn_bwd_apply_kernel, grid, dim3(256), (size_t)0, as_stream(stream),
                    static_cast<const uint4*>(dxh), static_cast<const uint4*>(x), stats, S,
                    static_cast<const uint4*>(dres), static_cast<uint4*>(dx), colsum, (int)T,
                    (int)C, (int)groups, eps));
  return 0;
}

extern "C" int adp_ln_film_bwd(const void* dy, const void* x, const float* scale_shift,
                               int32_t ss_stride, void* dx, float* dss, int32_t dss_stride,
                               float* colsum, const void* dres, int32_t B, int32_t T, int32_t C,
                               float eps, adp_stream_t stream) {
  ADP_CHECK(dy && x && dx, "adp_ln_film_bwd: null");
  ADP_CHECK(C % 8 == 0 && C <= kBwMaxC, "adp_ln_film_bwd: C=%d", C);
  const int vpr = C / 8;
  int lpr, vpl;
  if (vpr <= 32) {
    ADP_CHECK((vpr & (vpr - 1)) == 0, "adp_ln_film_bwd: C/8=%d must be a power of two", vpr);
    lpr = vpr; vpl = 1;
  } else {
    ADP_CHECK(vpr % 32 == 0 && vpr / 32 <= 4, "adp_ln_film_bwd: C=%d unsupported", C);
    lpr = 32; vpl = vpr / 32;
  }
  const int rows_per_block = 8 * (32 / lpr);
  // few rows (deep levels): one pass per warp so that every SM gets a block; many rows: persistent
  // blocks (each ends in 3C global atomics)
  const size_t g1 = (static_cast<size_t>(T) + rows_per_block - 1) / rows_per_block;
  size_t g = g1 * B <= num_sms() * 2 ? g1 : (static_cast<size_t>(T) + rows_per_block * 4 - 1) / (rows_per_block * 4);
  const size_t cap = num_sms() * 4 / (B < 8 ? B : 8) + 1;
  if (g > cap) g = cap;
  dim3 grid(static_cast<unsigned>(g < 1 ? 1 : g), B);
  const uint4* pdy = static_cast<const uint4*>(dy);
  const uint4* px = static_cast<const uint4*>(x);
  uint4* pdx = static_cast<uint4*>(dx);
  cudaStream_t s = as_stream(stream);
#define ADP_LNB(VPL)                                                                              \
  ADP_CUDA(launch_k(ln_film_bwd_kernel<VPL>, grid, dim3(256), (size_t)0, s, pdy, px, scale_shift, \
                    (int)ss_stride, pdx, dss, (int)dss_stride, colsum,                            \
                    static_cast<const uint4*>(dres), (int)T, (int)C, (int)lpr, eps))
  if (vpl == 1) ADP_LNB(1);
  else if (vpl == 2) ADP_LNB(2);
  else if (vpl == 3) ADP_LNB(3);
  else ADP_LNB(4);
#undef ADP_LNB
  return 0;
}

extern "C" int adp_colsum(const void* x, const float* gate, int32_t ld_gate, float* out, int32_t B,
                          int32_t T, int32_t C, adp_stream_t stream) {
  ADP_CHECK(x && out && C % 8 == 0 && C <= kColsumMaxC, "adp_colsum: bad args (C=%d)", C);
  dim3 grid(grid_for(static_cast<size_t>(T) * (C / 8), B), B);
  ADP_CUDA(launch_k(colsum_kernel, grid, dim3(256), (size_t)0, as_stream(stream),
                    static_cast<const uint4*>(x), gate, (int)ld_gate, out, (int)T, (int)C));
  return 0;
}

extern "C" int adp_skip_gate(const void* y, const void* skip, const float* gate, int32_t ld_gate,
                             void* out, double* stats, int32_t B, int32_t T, int32_t C,
                             int32_t groups, adp_stream_t stream) {
  ADP_CHECK(y && skip && gate && out && C % 8 == 0, "adp_skip_gate: bad args");
  ADP_CHECK(!stats || (groups > 0 && groups <= 64 && C % groups == 0 && C <= kBwMaxC), "adp_skip_gate: groups");
  dim3 grid(grid_for(static_cast<size_t>(T) * (C / 8), B), B);
  ADP_CUDA(launch_k(skip_gate_kernel, grid, dim3(256), (size_t)0, as_stream(stream),
                    static_cast<const uint4*>(y), static_cast<const uint4*>(skip), gate,
                    (int)ld_gate, static_cast<uint4*>(out), stats, (int)T, (int)C, (int)groups));
  return 0;
}

extern "C" int adp_skip_gate_bwd(const void* dout, const void* y, const float* gate,
                                 int32_t ld_gate, void* dys, float* dgate, int32_t ld_dgate,
                                 int32_t B, int32_t T, int32_t C, adp_stream_t stream) {
  ADP_CHECK(dout && y && gate && dys && dgate && C % 8 == 0 && C <= kBwMaxC, "adp_skip_gate_bwd: bad args");
  dim3 grid(grid_for(static_cast<size_t>(T) * (C / 8), B), B);
  ADP_CUDA(launch_k(skip_gate_bwd_kernel, grid, dim3(256), (size_t)0, as_stream(stream),
                    static_cast<const uint4*>(dout), static_cast<const uint4*>(y), gate,
                    (int)ld_gate, static_cast<uint4*>(dys), dgate, (int)ld_dgate, (int)T, (int)C));
  return 0;
}

template <int MAXB, bool DC>
static int launch_cond_bwd(const float* dss, int ld_dss, const float* cond, const void* w, float* dw,
                           float* dbias, float* dcond, int B, int N, int K, cudaStream_t stream) {
  const int rows_per_block = 64;
  static SmemAttrCache smem_cache;
  dim3 grid((N + rows_per_block - 1) / rows_per_block);
  const size_t smem = static_cast<size_t>(MAXB) * rows_per_block * sizeof(float);
  ADP_CUDA(ensure_dyn_smem(cond_bwd_kernel<MAXB, DC>, smem, smem_cache));
  // batches beyond MAXB rows run as further passes that accumulate into dw / dbias
  for (int b0 = 0; b0 < B; b0 += MAXB) {
    const int bc = B - b0 < MAXB ? B - b0 : MAXB;
    ADP_CUDA(launch_k(cond_bwd_kernel<MAXB, DC>, grid, dim3(256), smem, stream,
                      dss + static_cast<size_t>(b0) * ld_dss, ld_dss, cond + static_cast<size_t>(b0) * K,
                      static_cast<const __nv_bfloat16*>(w), dw, dbias,
                      dcond ? dcond + static_cast<size_t>(b0) * K : nullptr, bc, N, K, rows_per_block,
                      (int)(b0 > 0)));
  }
  return 0;
}

extern "C" int adp_cond_bwd(const float* dss, int32_t ld_dss, const float* cond, const void* w,
                            float* dw, float* dbias, float* dcond, int32_t B, int32_t N, int32_t K,
                            adp_stream_t stream) {
  ADP_CHECK(dss && cond && w && dw && dbias, "adp_cond_bwd: null");   // dcond may be NULL (not wanted)
  ADP_CHECK(B >= 1, "adp_cond_bwd: B=%d", B);
  ADP_CHECK(K % 4 == 0, "adp_cond_bwd: K=%d must be a multiple of 4", K);
  cudaStream_t s = as_stream(stream);
  if (dcond == nullptr)       // parameter gradients only (all-gathered rows of a data-parallel step):
    return launch_cond_bwd<kCondGatherB, false>(dss, ld_dss, cond, w, dw, dbias, nullptr, B, N, K, s);
  return launch_cond_bwd<kCondMaxB, true>(dss, ld_dss, cond, w, dw, dbias, dcond, B, N, K, s);
}
