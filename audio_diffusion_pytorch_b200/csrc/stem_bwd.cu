// Backward of the network-boundary / narrow-level kernels of stem.cu (CUDA cores).
// Pattern: stage the tile's activations and output gradients in shared memory, then
//   (1) one thread per position for the data gradient, (2) one thread per parameter for the
//   weight gradient (a 256-step dot product out of smem), one atomic per parameter per CTA.
#include "common.cuh"
#include "ptx.cuh"

namespace adp {

constexpr int kTB = 256;

// blocks per batch element for the persistent tile loops: ~4 blocks per SM in total
static int persistent_blocks(int n_tiles, int B) {
  int g = (num_sms() * 4 + B - 1) / B;
  if (g > n_tiles) g = n_tiles;
  return g < 1 ? 1 : g;
}

// ---------------------------------------------------------------------- narrow_conv_bwd
// forward: y = conv3(a) + bias, a = silu(xhat*gamma + beta), C == 8.  Given dy:
//   dxh = (conv3^T dy) * silu'(z) * gamma  (first GroupNorm-backward pass, see adp_gn_bwd_apply)
//   dgamma, dbeta, S[b,g] = (sum dxh, sum dxh*xhat), dw[co][ci][k], dbias[co].
template <int C>
__global__ void __launch_bounds__(kTB)
narrow_conv_bwd_kernel(const adp_narrow_conv_bwd_args a) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ __align__(16) float s_a[(kTB + 2) * C];    // activated input, rows t0-1 .. t0+TB
  __shared__ __align__(16) float s_dy[(kTB + 2) * C];   // output gradient, same rows
  __shared__ __align__(16) float s_w[3 * C * C];        // [k][co][ci]
  __shared__ float s_ga[C], s_be[C], s_mean[C], s_rstd[C];
  __shared__ float s_red[4 * C];                        // dgamma, dbeta, S1, S2 per channel
  const int b = blockIdx.y;
  // persistent over row tiles: the parameter gradients stay in registers / smem and reach global
  // memory with ONE atomic per parameter per block (one block per tile meant 4096 same-address
  // atomics per parameter)
  const int n_tiles = (a.T + kTB - 1) / kTB;
  static_assert(C == 8, "register layout of the weight-gradient accumulators assumes C = 8");
  float gwr[2][C][3], gb[2] = {0.f, 0.f};              // dw[2 co][C ci][3 taps], dbias[2 co]
#pragma unroll
  for (int c2 = 0; c2 < 2; ++c2)
#pragma unroll
    for (int ci = 0; ci < C; ++ci) { gwr[c2][ci][0] = 0.f; gwr[c2][ci][1] = 0.f; gwr[c2][ci][2] = 0.f; }
  for (int i = threadIdx.x; i < 3 * C * C; i += kTB) {
    const int k = i / (C * C), r = i - k * C * C, co = r / C, ci = r - co * C;
    s_w[i] = a.w[(co * C + ci) * 3 + k];
  }
  if (threadIdx.x < C) {
    const int c = threadIdx.x, gsz = C / a.groups, g = c / gsz;
    const double inv_n = 1.0 / (static_cast<double>(gsz) * a.T);
    const double mean = a.stats_in[(static_cast<size_t>(b) * a.groups + g) * 2] * inv_n;
    const float var = fmaxf(static_cast<float>(
        a.stats_in[(static_cast<size_t>(b) * a.groups + g) * 2 + 1] * inv_n - mean * mean), 0.f);
    s_mean[c] = static_cast<float>(mean);
    s_rstd[c] = rsqrtf(var + a.gn_eps);
    s_ga[c] = a.gamma[c];
    s_be[c] = a.beta[c];
  }
  if (threadIdx.x < 4 * C) s_red[threadIdx.x] = 0.f;
  __syncthreads();
  const __nv_bfloat16* xb = static_cast<const __nv_bfloat16*>(a.x) + static_cast<size_t>(b) * a.T * C;
  const __nv_bfloat16* dyb = static_cast<const __nv_bfloat16*>(a.dy) + static_cast<size_t>(b) * a.T * C;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
  const int t0 = tile * kTB;
  __syncthreads();                                     // previous tile's smem fully consumed
  for (int i = threadIdx.x; i < kTB + 2; i += kTB) {
    const int t = t0 - 1 + i;
#pragma unroll
    for (int c = 0; c < C; ++c) { s_a[i * C + c] = 0.f; s_dy[i * C + c] = 0.f; }
    if (t >= 0 && t < a.T) {
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const float xh = (__bfloat162float(xb[static_cast<size_t>(t) * C + c]) - s_mean[c]) * s_rstd[c];
        s_a[i * C + c] = silu_f(xh * s_ga[c] + s_be[c]);
        s_dy[i * C + c] = __bfloat162float(dyb[static_cast<size_t>(t) * C + c]);
      }
    }
  }
  __syncthreads();
  // (1) data gradient, one thread per position
  const int t = t0 + threadIdx.x;
  float r_dg[C], r_db[C], r_s1[C], r_s2[C];
#pragma unroll
  for (int c = 0; c < C; ++c) { r_dg[c] = 0.f; r_db[c] = 0.f; r_s1[c] = 0.f; r_s2[c] = 0.f; }
  if (t < a.T) {
    float da[C];
#pragma unroll
    for (int c = 0; c < C; ++c) da[c] = 0.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float* dyr = &s_dy[(threadIdx.x + 2 - k) * C];     // dy[t - (k-1)]
#pragma unroll
      for (int co = 0; co < C; ++co) {
        const float g = dyr[co];
#pragma unroll
        for (int ci = 0; ci < C; ++ci) da[ci] += g * s_w[(k * C + co) * C + ci];
      }
    }
    float o[C], xh[C];
#pragma unroll
    for (int c = 0; c < C; ++c) {
      xh[c] = (__bfloat162float(xb[static_cast<size_t>(t) * C + c]) - s_mean[c]) * s_rstd[c];
      const float z = xh[c] * s_ga[c] + s_be[c];
      const float sg = 1.f / (1.f + __expf(-z));
      const float dz = da[c] * sg * (1.f + z * (1.f - sg));
      o[c] = dz * s_ga[c];
      r_dg[c] = dz * xh[c];
      r_db[c] = dz;
    }
    __nv_bfloat16* op = static_cast<__nv_bfloat16*>(a.dxh) + (static_cast<size_t>(b) * a.T + t) * C;
#pragma unroll
    for (int c = 0; c < C; c += 8) {
      const uint4 ov = make_uint4(pack_bf16(o[c], o[c + 1]), pack_bf16(o[c + 2], o[c + 3]),
                                  pack_bf16(o[c + 4], o[c + 5]), pack_bf16(o[c + 6], o[c + 7]));
      *reinterpret_cast<uint4*>(op + c) = ov;
      const uint32_t ou[4] = {ov.x, ov.y, ov.z, ov.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {          // sums of the ROUNDED values the second pass reads
        const float2 r = unpack_bf16(ou[j]);
        r_s1[c + 2 * j] = r.x; r_s2[c + 2 * j] = r.x * xh[c + 2 * j];
        r_s1[c + 2 * j + 1] = r.y; r_s2[c + 2 * j + 1] = r.y * xh[c + 2 * j + 1];
      }
    }
  }
  {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const float v0 = warp_sum(r_dg[c]), v1 = warp_sum(r_db[c]);
      const float v2 = warp_sum(r_s1[c]), v3 = warp_sum(r_s2[c]);
      if (lane == 0) {
        atomicAdd(&s_red[c], v0); atomicAdd(&s_red[C + c], v1);
        atomicAdd(&s_red[2 * C + c], v2); atomicAdd(&s_red[3 * C + c], v3);
      }
    }
  }
  // (2) weight gradient: thread j < 3*C*C owns dw[co][ci][k]; threads after that own dbias[co]
  // (2) weight gradient: thread = (position p of a 64-position pass, output-channel pair cg); its
  // 2 x C x 3 dw elements and 2 dbias elements live in registers across all tiles of the block
  const int nvalid = min(kTB, a.T - t0);
  {
    const int cg = threadIdx.x & 3, p = threadIdx.x >> 2;
#pragma unroll
    for (int pass = 0; pass < kTB / 64; ++pass) {
      const int i = pass * 64 + p;
      if (i < nvalid) {
        const float g0 = s_dy[(i + 1) * C + 2 * cg], g1 = s_dy[(i + 1) * C + 2 * cg + 1];
        gb[0] += g0; gb[1] += g1;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const float4* ar = reinterpret_cast<const float4*>(&s_a[(i + k) * C]);
          const float4 a0 = ar[0], a1 = ar[1];
          const float a8[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
          for (int ci = 0; ci < C; ++ci) { gwr[0][ci][k] += g0 * a8[ci]; gwr[1][ci][k] += g1 * a8[ci]; }
        }
      }
    }
  }
  }  // tiles
  {
    // lanes with the same cg (stride 4) fold, then the 8 warps through smem: one atomic per element
    __syncthreads();
    float* s_part = s_a;                        // [8 warps][4 cg][50]; the tile buffers are dead
    const int cg = threadIdx.x & 3, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    auto put = [&](int idx, float v) {
      v += __shfl_xor_sync(0xffffffffu, v, 4);
      v += __shfl_xor_sync(0xffffffffu, v, 8);
      v += __shfl_xor_sync(0xffffffffu, v, 16);
      if (lane < 4) s_part[(warp * 4 + cg) * 50 + idx] = v;
    };
#pragma unroll
    for (int c2 = 0; c2 < 2; ++c2) {
#pragma unroll
      for (int ci = 0; ci < C; ++ci)
#pragma unroll
        for (int k = 0; k < 3; ++k) put((c2 * C + ci) * 3 + k, gwr[c2][ci][k]);
      put(48 + c2, gb[c2]);
    }
    __syncthreads();
    if (threadIdx.x < 4 * 50) {
      const int cgo = threadIdx.x / 50, idx = threadIdx.x - cgo * 50;
      float tot = 0.f;
#pragma unroll
      for (int w8 = 0; w8 < 8; ++w8) tot += s_part[(w8 * 4 + cgo) * 50 + idx];
      if (idx < 48) {                                    // (c2, ci, k) -> dw[co = 2*cgo + c2][ci][k]
        const int c2 = idx / 24, r = idx - c2 * 24;
        atomicAdd(a.dw + (2 * cgo + c2) * 3 * C + r, tot);
      } else {
        atomicAdd(a.dbias + 2 * cgo + (idx - 48), tot);
      }
    }
  }
  __syncthreads();
  if (threadIdx.x < C) {
    atomicAdd(a.dgamma + threadIdx.x, s_red[threadIdx.x]);
    atomicAdd(a.dbeta + threadIdx.x, s_red[C + threadIdx.x]);
  }
  if (threadIdx.x < 2 * a.groups) {
    const int g = threadIdx.x >> 1, which = threadIdx.x & 1, gsz = C / a.groups;
    float tot = 0.f;
    for (int c = g * gsz; c < (g + 1) * gsz; ++c) tot += s_red[(2 + which) * C + c];
    atomicAdd(a.S + static_cast<size_t>(b) * 2 * a.groups + threadIdx.x, static_cast<double>(tot));
  }
}

// ------------------------------------------------------------------------- stem_out_bwd
constexpr int kSoMaxC0 = 64;
constexpr int kSoMaxCo = 4;
constexpr int kSoItems = 4;      // parameter-gradient elements per thread (co*c0*3 + ... <= 1024)
__global__ void __launch_bounds__(kTB) stem_out_bwd_kernel(const adp_stem_out_bwd_args a) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float s_dyn[];
  const int cin = a.cx + a.ca;
  const int rows_h = kTB / a.f + 2;                 // low-res rows covering t0-1 .. t0+TB
  float* s_w = s_dyn;                               // [co][3][c0]
  float* s_h = s_w + a.co * 3 * a.c0;               // [rows_h][c0]
  float* s_dy = s_h + rows_h * a.c0;                // [(TB+2)][co]  = dv * gate * gscale
  float* s_dv = s_dy + (kTB + 2) * a.co;            // [TB][co]      = dv * gscale
  float* s_xin = s_dv + kTB * a.co;                 // [TB][cin]
  const int b = blockIdx.y;
  const int Tl = a.T / a.f;
  const int ldg = a.ld_gate > 0 ? a.ld_gate : a.co;
  const float gscale = a.gscale ? a.gscale[0] : 1.f;
  for (int i = threadIdx.x; i < a.co * 3 * a.c0; i += kTB) {
    const int o = i / (3 * a.c0), r = i - o * 3 * a.c0, k = r / a.c0, c = r - k * a.c0;
    s_w[i] = a.w[(o * a.c0 + c) * 3 + k];
  }
  // persistent over tiles; each thread owns up to kSoItems parameter-gradient elements and adds
  // them to global memory once per block (see adp_narrow_conv_bwd)
  float acc_it[kSoItems];
#pragma unroll
  for (int k = 0; k < kSoItems; ++k) acc_it[k] = 0.f;
  // fast path (the shapes of every model class: c0 = 8, <= 2 output and <= 4 input channels):
  // one thread per POSITION with every parameter gradient in its own register, reduced across the
  // block once at the very end -- the generic path below gives each parameter to one thread, which
  // leaves 3/4 of the block idle in 256-step dot products (1.2 ms for this one kernel at B = 4)
  const bool fast = a.c0 == 8 && a.co <= 2 && cin <= 4;
  float fw[2][8][3], fb[2] = {0.f, 0.f}, fg[2] = {0.f, 0.f}, fad[2][4], fadb[2] = {0.f, 0.f};
#pragma unroll
  for (int o = 0; o < 2; ++o) {
#pragma unroll
    for (int c = 0; c < 8; ++c) { fw[o][c][0] = 0.f; fw[o][c][1] = 0.f; fw[o][c][2] = 0.f; }
#pragma unroll
    for (int c = 0; c < 4; ++c) fad[o][c] = 0.f;
  }
  const int n_tiles = (a.T + kTB - 1) / kTB;
  const int n_w = a.co * a.c0 * 3, n_ad = a.w_adapt ? a.co * cin : 0;
  const int n_items = n_w + a.co /*bias*/ + a.co /*gate*/ + n_ad + (a.w_adapt ? a.co : 0);
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
  const int t0 = tile * kTB;                        // multiple of f (TB % f == 0)
  const int q0 = t0 / a.f - 1;                      // first low-res row held in s_h
  __syncthreads();                                  // previous tile's smem fully consumed
  const __nv_bfloat16* hb = static_cast<const __nv_bfloat16*>(a.h) + static_cast<size_t>(b) * Tl * a.c0;
  for (int i = threadIdx.x; i < rows_h * a.c0; i += kTB) {
    const int r = i / a.c0, c = i - r * a.c0, q = q0 + r;
    s_h[i] = (q >= 0 && q < Tl) ? __bfloat162float(hb[static_cast<size_t>(q) * a.c0 + c]) : 0.f;
  }
  for (int i = threadIdx.x; i < (kTB + 2) * a.co; i += kTB) {
    const int r = i / a.co, o = i - r * a.co, t = t0 - 1 + r;
    float v = 0.f;
    if (t >= 0 && t < a.T)
      v = a.dv[(static_cast<size_t>(b) * a.co + o) * a.T + t] * gscale;
    s_dy[i] = v * a.gate[static_cast<size_t>(b) * ldg + o];
    if (r >= 1 && r <= kTB) s_dv[(r - 1) * a.co + o] = v;
  }
  float al = 1.f, be = 0.f;
  if (a.noise) { al = a.alpha[b]; be = a.beta[b]; }
  for (int i = threadIdx.x; i < kTB * cin; i += kTB) {
    const int r = i / cin, c = i - r * cin, t = t0 + r;
    float v = 0.f;
    if (t < a.T) {
      if (c < a.cx) {
        const size_t idx = (static_cast<size_t>(b) * a.cx + c) * a.T + t;
        v = a.x[idx];
        if (a.noise) v = al * v + be * a.noise[idx];
      } else {
        v = a.append[(static_cast<size_t>(b) * a.ca + (c - a.cx)) * a.T + t];
      }
    }
    s_xin[i] = v;
  }
  __syncthreads();
  const int nvalid = min(kTB, a.T - t0);
  // (1) dh: one thread per low-res row of the tile
  const int nq = kTB / a.f;
  if (threadIdx.x < nq) {
    const int q = t0 / a.f + threadIdx.x;
    if (q < Tl) {
      __nv_bfloat16* dhp = static_cast<__nv_bfloat16*>(a.dh) + (static_cast<size_t>(b) * Tl + q) * a.c0;
      for (int c8 = 0; c8 < a.c0; c8 += 8) {
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
        for (int u = q * a.f; u < q * a.f + a.f; ++u) {       // upsampled positions fed by row q
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            const int tp = u - k + 1;                          // output position using (u, k)
            if (tp < 0 || tp >= a.T) continue;
            const float* dyr = &s_dy[(tp - t0 + 1) * a.co];
            for (int o = 0; o < a.co; ++o) {
              const float g = dyr[o];
              const float* wp = &s_w[(o * 3 + k) * a.c0 + c8];
#pragma unroll
              for (int j = 0; j < 8; ++j) acc[j] += g * wp[j];
            }
          }
        }
        *reinterpret_cast<uint4*>(dhp + c8) =
            make_uint4(pack_bf16(acc[0], acc[1]), pack_bf16(acc[2], acc[3]),
                       pack_bf16(acc[4], acc[5]), pack_bf16(acc[6], acc[7]));
      }
    }
  }
  // (2) parameter gradients
  if (fast) {
    const int i = threadIdx.x;
    if (i < nvalid) {
      float dyv[2], dvv[2], yv[2];
#pragma unroll
      for (int o = 0; o < 2; ++o) {
        const bool on = o < a.co;
        dyv[o] = on ? s_dy[(i + 1) * a.co + o] : 0.f;
        dvv[o] = on ? s_dv[i * a.co + o] : 0.f;
        yv[o] = (on && a.bias) ? a.bias[o] : 0.f;
      }
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const int u = t0 + i + k - 1;
        if (u < 0 || u >= a.T) continue;
        const float4* hr = reinterpret_cast<const float4*>(&s_h[(u / a.f - q0) * 8]);
        const float4 h0 = hr[0], h1 = hr[1];
        const float h8[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
#pragma unroll
        for (int o = 0; o < 2; ++o) {
          if (o >= a.co) break;
          const float* wp = &s_w[(o * 3 + k) * 8];
#pragma unroll
          for (int c = 0; c < 8; ++c) { fw[o][c][k] += dyv[o] * h8[c]; yv[o] += h8[c] * wp[c]; }
        }
      }
#pragma unroll
      for (int o = 0; o < 2; ++o) {
        fb[o] += dyv[o];
        fg[o] += dvv[o] * yv[o];
        if (a.w_adapt) {
          fadb[o] += dvv[o];
#pragma unroll
          for (int c = 0; c < 4; ++c)
            if (c < cin) fad[o][c] += dvv[o] * s_xin[i * cin + c];
        }
      }
    }
  }
#pragma unroll
  for (int kk = 0; kk < kSoItems; ++kk) {
    const int item = threadIdx.x + kk * kTB;
    if (fast || item >= n_items) break;
    float acc = 0.f;
    if (item < n_w) {                         // dw[co][c0][k] (PyTorch layout)
      const int o = item / (a.c0 * 3), r = item - o * a.c0 * 3, c = r / 3, k = r - c * 3;
      for (int i = 0; i < nvalid; ++i) {
        const int u = t0 + i + k - 1;
        if (u < 0 || u >= a.T) continue;
        acc += s_dy[(i + 1) * a.co + o] * s_h[(u / a.f - q0) * a.c0 + c];
      }
    } else if (item < n_w + a.co) {           // dbias
      const int o = item - n_w;
      for (int i = 0; i < nvalid; ++i) acc += s_dy[(i + 1) * a.co + o];
    } else if (item < n_w + 2 * a.co) {       // dgate[b][o] = sum dv * y,  y = conv(hup) + bias
      const int o = item - n_w - a.co;
      const float bo = a.bias ? a.bias[o] : 0.f;
      for (int i = 0; i < nvalid; ++i) {
        float y = bo;
        for (int k = 0; k < 3; ++k) {
          const int u = t0 + i + k - 1;
          if (u < 0 || u >= a.T) continue;
          const float* hr = &s_h[(u / a.f - q0) * a.c0];
          const float* wp = &s_w[(o * 3 + k) * a.c0];
          for (int c = 0; c < a.c0; ++c) y += hr[c] * wp[c];
        }
        acc += s_dv[i * a.co + o] * y;
      }
    } else if (item < n_w + 2 * a.co + n_ad) {   // SkipAdapter weight [co][cin]
      const int r = item - n_w - 2 * a.co, o = r / cin, c = r - o * cin;
      for (int i = 0; i < nvalid; ++i) acc += s_dv[i * a.co + o] * s_xin[i * cin + c];
    } else {                                      // SkipAdapter bias
      const int o = item - n_w - 2 * a.co - n_ad;
      for (int i = 0; i < nvalid; ++i) acc += s_dv[i * a.co + o];
    }
    acc_it[kk] += acc;
  }
  // (3) gradient w.r.t. the net input through the skip path (v = skip(x_in) + gate*y):
  // identity skip -> dv, SkipAdapter -> W_adapt^T dv.  Plain stores: adp_stem_in_bwd adds the
  // DownsampleItem path afterwards.
  if (a.dxin != nullptr) {
    for (int i = threadIdx.x; i < kTB * cin; i += kTB) {
      const int c = i / kTB, r = i - c * kTB;
      if (r >= nvalid) continue;
      float acc = 0.f;
      if (a.w_adapt != nullptr) {
        for (int o = 0; o < a.co; ++o) acc += s_dv[r * a.co + o] * a.w_adapt[o * cin + c];
      } else if (c < a.co) {
        acc = s_dv[r * a.co + c];
      }
      a.dxin[(static_cast<size_t>(b) * cin + c) * a.T + t0 + r] = acc;
    }
  }
  }  // tiles
  if (fast) {
    // block reduction of the per-position registers: warp sums -> smem [8 warps][62] -> one atomic
    // per parameter; the item order is the generic path's (dw, dbias, dgate, dw_adapt, db_adapt)
    __syncthreads();
    float* s_red = s_dyn;                       // tile buffers are dead
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    auto put = [&](int idx, float v) {
      v = warp_sum(v);
      if (lane == 0) s_red[warp * 64 + idx] = v;
    };
#pragma unroll
    for (int o = 0; o < 2; ++o) {
#pragma unroll
      for (int c = 0; c < 8; ++c)
#pragma unroll
        for (int k = 0; k < 3; ++k) put((o * 8 + c) * 3 + k, fw[o][c][k]);       // 0..47
      put(48 + o, fb[o]);
      put(50 + o, fg[o]);
#pragma unroll
      for (int c = 0; c < 4; ++c) put(52 + o * 4 + c, fad[o][c]);
      put(60 + o, fadb[o]);
    }
    __syncthreads();
    if (threadIdx.x < 62) {
      float tot = 0.f;
#pragma unroll
      for (int w8 = 0; w8 < 8; ++w8) tot += s_red[w8 * 64 + threadIdx.x];
      const int idx = threadIdx.x;
      if (idx < 48) {
        const int o = idx / 24;
        if (o < a.co) atomicAdd(a.dw + idx, tot);              // [co][8][3] flat: same index
      } else if (idx < 50) {
        if (idx - 48 < a.co) atomicAdd(a.dbias + (idx - 48), tot);
      } else if (idx < 52) {
        if (idx - 50 < a.co) atomicAdd(a.dgate + static_cast<size_t>(b) * a.ld_dgate + (idx - 50), tot);
      } else if (idx < 60) {
        const int o = (idx - 52) >> 2, c = (idx - 52) & 3;
        if (a.w_adapt && o < a.co && c < cin) atomicAdd(a.dw_adapt + o * cin + c, tot);
      } else {
        if (a.w_adapt && idx - 60 < a.co) atomicAdd(a.db_adapt + (idx - 60), tot);
      }
    }
    return;
  }
#pragma unroll
  for (int kk = 0; kk < kSoItems; ++kk) {
    const int item = threadIdx.x + kk * kTB;
    if (item >= n_items) break;
    const float acc = acc_it[kk];
    if (item < n_w) atomicAdd(a.dw + item, acc);
    else if (item < n_w + a.co) atomicAdd(a.dbias + (item - n_w), acc);
    else if (item < n_w + 2 * a.co)
      atomicAdd(a.dgate + static_cast<size_t>(b) * a.ld_dgate + (item - n_w - a.co), acc);
    else if (item < n_w + 2 * a.co + n_ad) atomicAdd(a.dw_adapt + (item - n_w - 2 * a.co), acc);
    else atomicAdd(a.db_adapt + (item - n_w - 2 * a.co - n_ad), acc);
  }
}

// -------------------------------------------------------------------------- stem_in_bwd
constexpr int kSiItems = 9;      // c0 * (cx+ca) * f + c0 <= 64*32 + 64 parameter-gradient elements
__global__ void __launch_bounds__(kTB) stem_in_bwd_kernel(const adp_stem_in_bwd_args a) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float s_dyn[];
  const int cin = a.cx + a.ca, ci_total = cin * a.f;
  float* s_in = s_dyn;                      // [TB][ci_total]
  float* s_g = s_in + kTB * ci_total;       // [TB][c0]
  const int b = blockIdx.y;
  const int To = a.T / a.f;
  float al = 1.f, be = 0.f;
  if (a.noise) { al = a.alpha[b]; be = a.beta[b]; }
  const int n_w = a.c0 * ci_total;
  float acc_it[kSiItems];          // persistent blocks: parameter gradients flushed once per block
#pragma unroll
  for (int k = 0; k < kSiItems; ++k) acc_it[k] = 0.f;
  const int n_tiles = (To + kTB - 1) / kTB;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
  const int to0 = tile * kTB;
  __syncthreads();
  for (int i = threadIdx.x; i < kTB * ci_total; i += kTB) {
    const int r = i / ci_total, ii = i - r * ci_total, c = ii / a.f, j = ii - c * a.f, to = to0 + r;
    float v = 0.f;
    if (to < To) {
      const size_t tt = static_cast<size_t>(to) * a.f + j;
      if (c < a.cx) {
        const size_t idx = (static_cast<size_t>(b) * a.cx + c) * a.T + tt;
        v = a.x[idx];
        if (a.noise) v = al * v + be * a.noise[idx];
      } else {
        v = a.append[(static_cast<size_t>(b) * a.ca + (c - a.cx)) * a.T + tt];
      }
    }
    s_in[i] = v;
  }
  const __nv_bfloat16* gb = static_cast<const __nv_bfloat16*>(a.dout) + static_cast<size_t>(b) * To * a.c0;
  for (int i = threadIdx.x; i < kTB * a.c0; i += kTB) {
    const int r = i / a.c0, to = to0 + r;
    s_g[i] = to < To ? __bfloat162float(gb[static_cast<size_t>(to) * a.c0 + (i - r * a.c0)]) : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int kk = 0; kk < kSiItems; ++kk) {
    const int item = threadIdx.x + kk * kTB;
    if (item >= n_w + a.c0) break;
    float acc = 0.f;
    if (item < n_w) {                        // dw[c0][cin][f] flat == [c0][ci_total]
      const int o = item / ci_total, ii = item - o * ci_total;
      for (int i = 0; i < kTB; ++i) acc += s_g[i * a.c0 + o] * s_in[i * ci_total + ii];
    } else {
      const int o = item - n_w;
      for (int i = 0; i < kTB; ++i) acc += s_g[i * a.c0 + o];
    }
    acc_it[kk] += acc;
  }
  // gradient w.r.t. cat([x, append]) through the k = s = f DownsampleItem, ADDED to what
  // adp_stem_out_bwd stored: dxin[b][c][to*f + j] += sum_o dout[b][to][o] * w[o][c][j]
  if (a.dxin != nullptr) {
    for (int i = threadIdx.x; i < kTB * ci_total; i += kTB) {
      const int c = i / (kTB * a.f), rem = i - c * kTB * a.f, r = rem / a.f, j = rem - r * a.f;
      const int to = to0 + r;
      if (to >= To) continue;
      float acc = 0.f;
      const float* wp = a.w + c * a.f + j;
      for (int o = 0; o < a.c0; ++o) acc += s_g[r * a.c0 + o] * __ldg(wp + o * ci_total);
      a.dxin[(static_cast<size_t>(b) * cin + c) * a.T + static_cast<size_t>(to) * a.f + j] += acc;
    }
  }
  }  // tiles
#pragma unroll
  for (int kk = 0; kk < kSiItems; ++kk) {
    const int item = threadIdx.x + kk * kTB;
    if (item >= n_w + a.c0) break;
    if (item < n_w) atomicAdd(a.dw + item, acc_it[kk]);
    else atomicAdd(a.dbias + (item - n_w), acc_it[kk]);
  }
}

}  // namespace adp

using namespace adp;

extern "C" int adp_narrow_conv_bwd(const adp_narrow_conv_bwd_args* args, adp_stream_t stream) {
  ADP_CHECK(args && args->dy && args->x && args->stats_in && args->gamma && args->beta && args->w &&
            args->dxh && args->dgamma && args->dbeta && args->S && args->dw && args->dbias,
            "adp_narrow_conv_bwd: null pointer");
  const adp_narrow_conv_bwd_args& a = *args;
  ADP_CHECK(a.C == 8 && a.groups > 0 && a.C % a.groups == 0, "adp_narrow_conv_bwd: C=%d groups=%d", a.C, a.groups);
  dim3 grid(persistent_blocks((a.T + kTB - 1) / kTB, a.B), a.B);
  ADP_CUDA(launch_k(narrow_conv_bwd_kernel<8>, grid, dim3(kTB), (size_t)0, as_stream(stream), a));
  return 0;
}

extern "C" int adp_stem_out_bwd(const adp_stem_out_bwd_args* args, adp_stream_t stream) {
  ADP_CHECK(args && args->dv && args->h && args->x && args->w && args->gate && args->dh && args->dw &&
            args->dbias && args->dgate, "adp_stem_out_bwd: null pointer");
  const adp_stem_out_bwd_args& a = *args;
  ADP_CHECK(a.co >= 1 && a.co <= kSoMaxCo && a.c0 % 8 == 0 && a.c0 <= kSoMaxC0 && a.cx + a.ca <= 8,
            "adp_stem_out_bwd: co=%d c0=%d unsupported", a.co, a.c0);
  ADP_CHECK(a.f >= 1 && kTB % a.f == 0 && a.T % a.f == 0, "adp_stem_out_bwd: f=%d", a.f);
  ADP_CHECK(!a.w_adapt || (a.dw_adapt && a.db_adapt), "adp_stem_out_bwd: adapter grads missing");
  ADP_CHECK((a.ca == 0) == (a.append == nullptr), "adp_stem_out_bwd: append / ca mismatch");
  const int cin = a.cx + a.ca, rows_h = kTB / a.f + 2;
  const size_t smem = (static_cast<size_t>(a.co) * 3 * a.c0 + static_cast<size_t>(rows_h) * a.c0 +
                       static_cast<size_t>(kTB + 2) * a.co + static_cast<size_t>(kTB) * a.co +
                       static_cast<size_t>(kTB) * cin) * sizeof(float);
  static SmemAttrCache smem_cache;
  ADP_CUDA(ensure_dyn_smem(stem_out_bwd_kernel, smem, smem_cache));
  ADP_CHECK(a.co * a.c0 * 3 + 3 * a.co + a.co * cin <= kSoItems * kTB, "adp_stem_out_bwd: too many parameters");
  dim3 grid(persistent_blocks((a.T + kTB - 1) / kTB, a.B), a.B);
  ADP_CUDA(launch_k(stem_out_bwd_kernel, grid, dim3(kTB), smem, as_stream(stream), a));
  return 0;
}

extern "C" int adp_stem_in_bwd(const adp_stem_in_bwd_args* args, adp_stream_t stream) {
  ADP_CHECK(args && args->dout && args->x && args->dw && args->dbias, "adp_stem_in_bwd: null pointer");
  const adp_stem_in_bwd_args& a = *args;
  ADP_CHECK((a.cx + a.ca) * a.f <= 32 && a.c0 % 8 == 0 && a.c0 <= 64 && a.T % a.f == 0,
            "adp_stem_in_bwd: unsupported sizes");
  ADP_CHECK((a.ca == 0) == (a.append == nullptr), "adp_stem_in_bwd: append / ca mismatch");
  ADP_CHECK(!a.dxin || a.w, "adp_stem_in_bwd: dxin needs the conv weights");
  const size_t smem = (static_cast<size_t>(kTB) * (a.cx + a.ca) * a.f + static_cast<size_t>(kTB) * a.c0) * sizeof(float);
  static SmemAttrCache smem_cache;
  ADP_CUDA(ensure_dyn_smem(stem_in_bwd_kernel, smem, smem_cache));
  dim3 grid(persistent_blocks((a.T / a.f + kTB - 1) / kTB, a.B), a.B);
  ADP_CUDA(launch_k(stem_in_bwd_kernel, grid, dim3(kTB), smem, as_stream(stream), a));
  return 0;
}
