// Network-boundary and narrow-level kernels (CUDA cores; these levels are pure HBM streaming):
//   adp_stem_in     fp32 [B][C][T] (+append, +VDiffusion noising) -> k=s=f conv -> bf16 NWC
//   adp_stem_out    bf16 NWC -> nearest-up f + conv3 -> skip/gate -> v (+CFG, +sampler step, +loss)
//   adp_narrow_conv C == 8 ConvBlock: GN+SiLU -> conv3 (+residual) (+LayerNorm/FiLM) (+stats)
#include "stem.cuh"

namespace adp {

// Per-thread (sum, sum of squares) of an 8-channel row -> block reduction through a transposed
// smem scratch (conflict-free, 16 LDS + 10 shuffles per thread) -> fp64 GroupNorm bins.
// All NT threads of the block must call.  s_red: [16][NT] floats.
template <int NT>
__device__ __forceinline__ void block_stats8(const float (&cs)[8], const float (&cq)[8], float* s_red,
                                             double* bins, int groups) {
  const int tid = threadIdx.x;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    s_red[c * NT + tid] = cs[c];
    s_red[(8 + c) * NT + tid] = cq[c];
  }
  __syncthreads();
  const int warp = tid >> 5, lane = tid & 31;
  for (int r = warp; r < 16; r += NT / 32) {
    float v = 0.f;
#pragma unroll
    for (int i = 0; i < NT / 32; ++i) v += s_red[r * NT + i * 32 + lane];
    v = warp_sum(v);
    if (lane == 0 && v != 0.f)
      atomicAdd(bins + 2 * ((r & 7) / (8 / groups)) + (r >> 3), static_cast<double>(v));
  }
}

// ------------------------------------------------------------------------------ stem_in
// Persistent blocks over 256-position tiles of one batch element: the next tile's inputs are
// prefetched into registers before the current tile is computed (a one-tile-per-block launch
// is bound by the load -> compute -> store latency chain of each wave, not by HBM).
template <int MAXIN>
__global__ void __launch_bounds__(256) stem_in_kernel(const adp_stem_in_args a) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float s_w[];            // [c0][ci_total] then bias[c0]
  __shared__ float s_stats[2 * 64];
  __shared__ float s_red[16 * 256];
  const bool fast_stats = a.stats && a.c0 == 8 && 8 % a.groups == 0;
  const int cin = a.cx + a.ca;
  const int ci_total = cin * a.f;
  float* s_b = s_w + a.c0 * ci_total;
  for (int i = threadIdx.x; i < a.c0 * ci_total; i += blockDim.x) s_w[i] = a.w[i];
  for (int i = threadIdx.x; i < a.c0; i += blockDim.x) s_b[i] = a.bias ? a.bias[i] : 0.f;
  if (threadIdx.x < 128) s_stats[threadIdx.x] = 0.f;
  __syncthreads();

  const int b = blockIdx.y;
  const int lane = threadIdx.x & 31;
  const int To = a.T / a.f;
  float al = 1.f, be = 0.f;
  if (a.noise) { al = a.alpha[b]; be = a.beta[b]; }

  auto load_in = [&](int to, float (&in)[MAXIN]) {
#pragma unroll
    for (int i = 0; i < MAXIN; ++i) in[i] = 0.f;
    if (to >= To) return;
    // PyTorch Conv1d weight layout [c0][cin][f]: input index i = c*f + j
#pragma unroll
    for (int i = 0; i < MAXIN; ++i) {
      if (i < ci_total) {
        const int c = i / a.f, j = i - c * a.f;
        in[i] = block_input<true>(a, b, c, static_cast<size_t>(to) * a.f + j, al, be);
      }
    }
  };

  const int gsz = a.stats ? a.c0 / a.groups : 1;
  GroupStatAcc acc;
  float cs[8], cq[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { cs[j] = 0.f; cq[j] = 0.f; }
  const int stride = gridDim.x * 256;
  float in[MAXIN], nxt[MAXIN];
  load_in(blockIdx.x * 256 + threadIdx.x, in);
  for (int base = blockIdx.x * 256; base < To; base += stride) {
    const int to = base + threadIdx.x;
    const bool ok = to < To;
    if (base + stride < To) load_in(to + stride, nxt);
    __nv_bfloat16* orow =
        static_cast<__nv_bfloat16*>(a.out) + (static_cast<size_t>(b) * To + (ok ? to : 0)) * a.c0;
    for (int co = 0; co < a.c0; co += 8) {
      float v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = s_b[co + j];
#pragma unroll
      for (int i = 0; i < MAXIN; ++i) {
        if (i < ci_total) {
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] += in[i] * s_w[(co + j) * ci_total + i];
        }
      }
      uint4 o;
      o.x = pack_bf16(v[0], v[1]); o.y = pack_bf16(v[2], v[3]);
      o.z = pack_bf16(v[4], v[5]); o.w = pack_bf16(v[6], v[7]);
      if (ok) *reinterpret_cast<uint4*>(orow + co) = o;
      if (a.stats) {        // statistics of the ROUNDED values the next layer reads
        const uint32_t ou[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 r = unpack_bf16(ou[j]);
          const float r0 = ok ? r.x : 0.f, r1 = ok ? r.y : 0.f;
          if (fast_stats) {     // c0 == 8: per-channel registers, one block reduction at the end
            cs[2 * j] += r0; cq[2 * j] += r0 * r0;
            cs[2 * j + 1] += r1; cq[2 * j + 1] += r1 * r1;
          } else {
            acc.add(r0, (co + 2 * j) / gsz, s_stats, lane);
            acc.add(r1, (co + 2 * j + 1) / gsz, s_stats, lane);
          }
        }
      }
    }
#pragma unroll
    for (int i = 0; i < MAXIN; ++i) in[i] = nxt[i];
  }
  if (fast_stats) {
    block_stats8<256>(cs, cq, s_red, a.stats + static_cast<size_t>(b) * 2 * a.groups, a.groups);
  } else if (a.stats) {
    acc.flush(s_stats, lane);
    __syncthreads();
    flush_group_stats(s_stats, a.stats, b, a.groups);
  }
}

// ----------------------------------------------------------------------------- stem_out
// conv3 on the nearest-upsampled h for one output position; w in smem as [co][k][c0]
__device__ __forceinline__ void stem_out_conv(const __nv_bfloat16* __restrict__ hb, int T, int f,
                                              int c0, int co_n, int t, const float* s_w,
                                              float (&y)[kStemOutNarrowCo]) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int idx = t + k - 1;
    if (idx < 0 || idx >= T) continue;       // zero padding of the upsampled signal
    const int q = f == 1 ? idx : idx / f;    // nearest-neighbour source row
    const uint4* row = reinterpret_cast<const uint4*>(hb + static_cast<size_t>(q) * c0);
    for (int c8 = 0; c8 < c0; c8 += 8) {
      const uint4 u = __ldg(row + (c8 >> 3));
      const uint32_t uu[4] = {u.x, u.y, u.z, u.w};
      float hv[8];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f2 = unpack_bf16(uu[j]);
        hv[2 * j] = f2.x; hv[2 * j + 1] = f2.y;
      }
#pragma unroll
      for (int o = 0; o < kStemOutNarrowCo; ++o) {
        if (o < co_n) {
          // two 16-byte broadcast reads (c0 % 8 == 0 keeps them aligned) instead of eight scalar
          const float4 w0 = *reinterpret_cast<const float4*>(s_w + (o * 3 + k) * c0 + c8);
          const float4 w1 = *reinterpret_cast<const float4*>(s_w + (o * 3 + k) * c0 + c8 + 4);
          y[o] += (hv[0] * w0.x + hv[1] * w0.y) + (hv[2] * w0.z + hv[3] * w0.w) +
                  (hv[4] * w1.x + hv[5] * w1.y) + (hv[6] * w1.z + hv[7] * w1.w);
        }
      }
    }
  }
}

__global__ void __launch_bounds__(256, 3) stem_out_kernel(const adp_stem_out_args a) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ __align__(16) float s_w[];   // conv w [co][3][c0], bias[co], adapt w [co][cin], adapt b[co]
  const int cin = a.cx + a.ca;
  float* s_b = s_w + a.co * 3 * a.c0;
  float* s_wa = s_b + a.co;
  float* s_ba = s_wa + a.co * cin;
  for (int i = threadIdx.x; i < a.co * 3 * a.c0; i += blockDim.x) {
    // PyTorch layout [co][c0][3] -> [co][3][c0]
    const int o = i / (3 * a.c0), r = i - o * 3 * a.c0, k = r / a.c0, c = r - k * a.c0;
    s_w[i] = a.w[(o * a.c0 + c) * 3 + k];
  }
  for (int i = threadIdx.x; i < a.co; i += blockDim.x) {
    s_b[i] = a.bias ? a.bias[i] : 0.f;
    s_ba[i] = a.b_adapt ? a.b_adapt[i] : 0.f;
  }
  if (a.w_adapt)
    for (int i = threadIdx.x; i < a.co * cin; i += blockDim.x) s_wa[i] = a.w_adapt[i];
  __syncthreads();

  const int b = blockIdx.y;
  const int Tl = a.T / a.f;
  double lsum = 0.0;
  float al = 1.f, be = 0.f;
  if (a.noise) { al = a.alpha[b]; be = a.beta[b]; }
  // persistent blocks (grid-stride over positions): the smem weight prologue is paid once and
  // several independent positions per thread are in flight
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < a.T; t += gridDim.x * blockDim.x) {
    float xin[kStemOutNarrowCin];        // block input at this position (the U-Net skip)
#pragma unroll
    for (int c = 0; c < kStemOutNarrowCin; ++c) xin[c] = c < cin ? block_input(a, b, c, t, al, be) : 0.f;
    float y[kStemOutNarrowCo], ym[kStemOutNarrowCo];
#pragma unroll
    for (int o = 0; o < kStemOutNarrowCo; ++o) { y[o] = o < a.co ? s_b[o] : 0.f; ym[o] = y[o]; }
    const __nv_bfloat16* h = static_cast<const __nv_bfloat16*>(a.h);
    stem_out_conv(h + static_cast<size_t>(b) * Tl * a.c0, a.T, a.f, a.c0, a.co, t, s_w, y);
    if (a.cfg)
      stem_out_conv(h + static_cast<size_t>(b + a.B) * Tl * a.c0, a.T, a.f, a.c0, a.co, t, s_w, ym);
#pragma unroll
    for (int o = 0; o < kStemOutNarrowCo; ++o) {
      if (o < a.co) {
        float skip;
        if (a.w_adapt) {                       // SkipAdapter 1x1 conv (in != out channels)
          skip = s_ba[o];
#pragma unroll
          for (int c = 0; c < kStemOutNarrowCin; ++c)
            if (c < cin) skip += xin[c] * s_wa[o * cin + c];
        } else {
          skip = xin[o];
        }
        stem_out_finish(a, b, o, t, skip, y[o], ym[o], xin[o], al, be, lsum);
      }
    }
  }
  if (a.loss_sum) block_loss_flush(lsum, a.loss_sum);
}

// -------------------------------------------------------------------------- narrow_conv
// C == 8 ConvBlock on the warp-level tensor cores.  A C=8 conv3 is a [T x 24] x [24 x 8] GEMM:
// far too thin for a wgmma tile (M=64 x N>=16 x K=16 with 32-byte TMA rows), but it fits
// mma.sync m16n8k16 exactly: K = tap*8 + ci (24, padded to 32 with zero weights), N = 8.
//   * GroupNorm+SiLU is applied while staging rows into smem as bf16 (16 bytes per row), so
//     the A fragment of rows [r, r+16) x taps {0,1} is ONE ldmatrix.x4 over overlapping row
//     windows (row t of tap k is smem row t+k), tap 2 one ldmatrix.x2; B fragments (weights)
//     live in registers for the whole kernel.
//   * Blocks are persistent over 256-row tiles of one batch element: the per-block prologue
//     (weights, fp64 statistics -> coefficients) is paid once, the next tile's rows are
//     prefetched into registers before the current tile is computed, and smem is double
//     buffered (one __syncthreads per tile).
//   * Epilogue in the accumulator layout (a quad owns one row): bias, residual, LayerNorm+FiLM
//     via two quad shuffles, 128-byte coalesced stores, per-channel statistics in registers.
template <int C>
__global__ void __launch_bounds__(256) narrow_conv_kernel(const adp_narrow_conv_args a) {
  static_assert(C == 8, "narrow_conv is written for 8 channels (one 16-byte row)");
  pdl_launch_dependents();
  pdl_wait();
  constexpr int TB = 256;
  __shared__ __align__(128) uint4 s_rows[2][TB + 2];     // bf16 activated rows t0-1 .. t0+TB
  __shared__ float s_a[C], s_d[C];
  __shared__ float s_part[TB / 32][2 * C];               // (sum, sumsq) per channel, one row per warp
  const int b = blockIdx.y;
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, q = lane & 3;
  if (tid < C) {
    const int c = tid;
    const int gsz = C / a.groups, gi = c / gsz;
    const double inv_n = 1.0 / (static_cast<double>(gsz) * a.T);
    const double sm = a.stats_in[(static_cast<size_t>(b) * a.groups + gi) * 2];
    const double sq = a.stats_in[(static_cast<size_t>(b) * a.groups + gi) * 2 + 1];
    const double mean = sm * inv_n;
    double var = sq * inv_n - mean * mean;
    var = var < 0.0 ? 0.0 : var;
    const float rstd = static_cast<float>(1.0 / sqrt(var + static_cast<double>(a.gn_eps)));
    const float ga = a.gamma[c] * rstd;
    s_a[c] = ga;
    s_d[c] = a.beta[c] - static_cast<float>(mean) * ga;
  }
  // B fragments: W[n = co][k = tap*8 + ci] = w[co][ci][tap] (PyTorch layout); this thread holds
  // n = g, k = 2q, 2q+1 (+8) of each 16-wide k block.  k >= 24 is zero padding.
  uint32_t bw[3];
  {
    const float* wr = a.w + static_cast<size_t>(g) * C * 3;
#pragma unroll
    for (int tap = 0; tap < 3; ++tap)
      bw[tap] = pack_bf16(wr[(2 * q) * 3 + tap], wr[(2 * q + 1) * 3 + tap]);
  }
  const float bias0 = a.bias ? a.bias[2 * q] : 0.f, bias1 = a.bias ? a.bias[2 * q + 1] : 0.f;
  float sc0 = 1.f, sc1 = 1.f, sh0 = 0.f, sh1 = 0.f;
  if (a.scale_shift) {
    const float* ss = a.scale_shift + static_cast<size_t>(b) * a.ss_stride;
    sc0 = 1.f + ss[2 * q]; sc1 = 1.f + ss[2 * q + 1];
    sh0 = ss[C + 2 * q]; sh1 = ss[C + 2 * q + 1];
  }
  __syncthreads();
  float ga[C], de[C];
#pragma unroll
  for (int c = 0; c < C; ++c) { ga[c] = s_a[c]; de[c] = s_d[c]; }

  const __nv_bfloat16* xb = static_cast<const __nv_bfloat16*>(a.x) + static_cast<size_t>(b) * a.T * C;
  const __nv_bfloat16* rb = a.residual
      ? static_cast<const __nv_bfloat16*>(a.residual) + static_cast<size_t>(b) * a.T * C : nullptr;
  __nv_bfloat16* yb = static_cast<__nv_bfloat16*>(a.y) + static_cast<size_t>(b) * a.T * C;
  const int n_tiles = (a.T + TB - 1) / TB;

  // rows of a tile -> registers: row t0 + tid by every thread, halo rows t0-1 / t0+TB by 0 / 1
  auto load_rows = [&](int tile, uint4& mine, uint4& halo) {
    const int t0 = tile * TB;
    const int t = t0 + tid;
    mine = make_uint4(0, 0, 0, 0);
    halo = make_uint4(0, 0, 0, 0);
    if (t < a.T) mine = __ldg(reinterpret_cast<const uint4*>(xb + static_cast<size_t>(t) * C));
    if (tid < 2) {
      const int th = tid == 0 ? t0 - 1 : t0 + TB;
      if (th >= 0 && th < a.T) halo = __ldg(reinterpret_cast<const uint4*>(xb + static_cast<size_t>(th) * C));
    }
  };
  auto activate = [&](const uint4& u, bool valid) {     // GroupNorm + SiLU -> bf16 row
    if (!valid) return make_uint4(0, 0, 0, 0);          // conv zero padding
    const uint32_t uu[4] = {u.x, u.y, u.z, u.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f2 = unpack_bf16(uu[j]);
      o[j] = pack_bf16(silu_fast(f2.x * ga[2 * j] + de[2 * j]), silu_fast(f2.y * ga[2 * j + 1] + de[2 * j + 1]));
    }
    return make_uint4(o[0], o[1], o[2], o[3]);
  };

  // residual values of this lane's accumulator elements (rows g, g+8 of both m16 blocks)
  auto load_res = [&](int tile, uint32_t (&r)[4]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int t = tile * TB + warp * 32 + (i >> 1) * 16 + g + (i & 1) * 8;
      r[i] = (rb && t < a.T)
          ? __ldg(reinterpret_cast<const uint32_t*>(rb + static_cast<size_t>(t) * C + 2 * q)) : 0u;
    }
  };

  float cs0 = 0.f, cs1 = 0.f, cq0 = 0.f, cq1 = 0.f;     // statistics of channels 2q, 2q+1
  int tile = blockIdx.x;
  uint4 mine, halo;
  uint32_t rcur[4] = {0u, 0u, 0u, 0u}, rnxt[4] = {0u, 0u, 0u, 0u};
  if (tile < n_tiles) { load_rows(tile, mine, halo); load_res(tile, rcur); }
  int buf = 0;
  for (; tile < n_tiles; tile += gridDim.x, buf ^= 1) {
    const int t0 = tile * TB;
    s_rows[buf][tid + 1] = activate(mine, t0 + tid < a.T);
    if (tid < 2) {
      const int th = tid == 0 ? t0 - 1 : t0 + TB;
      s_rows[buf][tid == 0 ? 0 : TB + 1] = activate(halo, th >= 0 && th < a.T);
    }
    if (tile + gridDim.x < n_tiles) {                                           // prefetch
      load_rows(tile + gridDim.x, mine, halo);
      load_res(tile + gridDim.x, rnxt);
    }
    __syncthreads();
    const uint32_t base = smem_u32(&s_rows[buf][0]);
#pragma unroll
    for (int mb = 0; mb < 2; ++mb) {
      const int r0 = warp * 32 + mb * 16;               // tile-local first row of this m16 block
      uint32_t af[4], a2[2];
      // matrices: (rows 0-7, tap0) (rows 8-15, tap0) (rows 0-7, tap1) (rows 8-15, tap1)
      ldmatrix_x4(base + static_cast<uint32_t>(r0 + (lane & 7) + ((lane >> 3) & 1) * 8 + (lane >> 4)) * 16, af);
      ldmatrix_x2(base + static_cast<uint32_t>(r0 + (lane & 7) + ((lane >> 3) & 1) * 8 + 2) * 16, a2);
      float d[4] = {bias0, bias1, bias0, bias1};
      const uint32_t at2[4] = {a2[0], a2[1], 0u, 0u};   // tap 2: k 16..23, 24..31 zero
      mma_16816(d, af, bw[0], bw[1]);
      mma_16816(d, at2, bw[2], 0u);
#pragma unroll
      for (int h = 0; h < 2; ++h) {                     // rows g and g + 8 of the block
        const int t = t0 + r0 + g + h * 8;
        const bool ok = t < a.T;
        float y0 = d[2 * h], y1 = d[2 * h + 1];
        if (rb) {
          const float2 r2 = unpack_bf16(rcur[mb * 2 + h]);
          y0 += r2.x; y1 += r2.y;
        }
        if (a.scale_shift) {   // following ModulationItem: LayerNorm over C (no affine) + FiLM
          float m = y0 + y1;
          m += __shfl_xor_sync(0xffffffffu, m, 1);
          m += __shfl_xor_sync(0xffffffffu, m, 2);
          m *= (1.f / C);
          const float e0 = y0 - m, e1 = y1 - m;
          float v = e0 * e0 + e1 * e1;
          v += __shfl_xor_sync(0xffffffffu, v, 1);
          v += __shfl_xor_sync(0xffffffffu, v, 2);
          const float rstd = rsqrtf(v * (1.f / C) + a.ln_eps);
          y0 = e0 * rstd * sc0 + sh0;
          y1 = e1 * rstd * sc1 + sh1;
        }
        const uint32_t o = pack_bf16(y0, y1);
        if (ok) {
          *reinterpret_cast<uint32_t*>(yb + static_cast<size_t>(t) * C + 2 * q) = o;
          const float2 r = unpack_bf16(o);      // statistics of the ROUNDED values
          cs0 += r.x; cq0 += r.x * r.x;
          cs1 += r.y; cq1 += r.y * r.y;
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) rcur[i] = rnxt[i];
  }
  if (a.stats_out) {
#pragma unroll
    for (int o = 4; o < 32; o <<= 1) {
      cs0 += __shfl_xor_sync(0xffffffffu, cs0, o); cq0 += __shfl_xor_sync(0xffffffffu, cq0, o);
      cs1 += __shfl_xor_sync(0xffffffffu, cs1, o); cq1 += __shfl_xor_sync(0xffffffffu, cq1, o);
    }
    if (lane < 4) {            // lane == q: channels 2q, 2q+1, into the warp's own row
      s_part[warp][2 * (2 * q)] = cs0;     s_part[warp][2 * (2 * q) + 1] = cq0;
      s_part[warp][2 * (2 * q + 1)] = cs1; s_part[warp][2 * (2 * q + 1) + 1] = cq1;
    }
    __syncthreads();
    // warps and channels summed in a fixed order (fp64): the block's contribution does not
    // depend on the order the warps finish in, so a run repeats itself up to the fp64 atomics
    if (tid < 2 * a.groups) {  // tid = 2*group + {sum, sumsq}
      const int gi = tid >> 1, gsz = C / a.groups;
      double tot = 0.0;
      for (int w = 0; w < TB / 32; ++w)
        for (int c = gi * gsz; c < (gi + 1) * gsz; ++c) tot += s_part[w][2 * c + (tid & 1)];
      if (tot != 0.0) atomicAdd(a.stats_out + (static_cast<size_t>(b) * a.groups + gi) * 2 + (tid & 1), tot);
    }
  }
}

// ------------------------------------------------------------------ wide boundary (stem_in)
// Every size of the envelope the register-array kernel above does not take: (cx+ca)*f up to 128
// inputs per output position.  Weights live in smem transposed to [ci][c0] (256 x 128 fp32 = 128 KiB at the corner),
// the input tile [ci][kWideTP] is staged through smem with coalesced NCW reads, and each thread
// computes 8 output channels of one position per pass (the warp shares the channel chunk: the
// weight reads are 16-byte broadcasts).
constexpr int kWideTP = 64;          // low-rate positions per stem_in tile

__global__ void __launch_bounds__(256) stem_in_wide_kernel(const adp_stem_in_args a) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ __align__(16) float s_dyn[];
  __shared__ float s_stats[2 * 64];
  const int cin = a.cx + a.ca, ci_total = cin * a.f;
  float* s_w = s_dyn;                                   // [ci_total][c0]
  float* s_b = s_w + ci_total * a.c0;                   // [c0]
  float* s_in = s_b + a.c0;                             // [ci_total][kWideTP + 1]
  constexpr int LD = kWideTP + 1;
  for (int i = threadIdx.x; i < a.c0 * ci_total; i += blockDim.x) {
    const int o = i / ci_total, ii = i - o * ci_total;
    s_w[ii * a.c0 + o] = a.w[i];
  }
  for (int i = threadIdx.x; i < a.c0; i += blockDim.x) s_b[i] = a.bias ? a.bias[i] : 0.f;
  if (threadIdx.x < 128) s_stats[threadIdx.x] = 0.f;

  const int b = blockIdx.y;
  const int lane = threadIdx.x & 31;
  const int p = threadIdx.x % kWideTP, cg = threadIdx.x / kWideTP;
  const int To = a.T / a.f;
  const float al = a.noise ? a.alpha[b] : 1.f, be = a.noise ? a.beta[b] : 0.f;
  const int gsz = a.stats ? a.c0 / a.groups : 1;
  GroupStatAcc acc;
  const int n_tiles = (To + kWideTP - 1) / kWideTP;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int to0 = tile * kWideTP;
    __syncthreads();                                    // weights staged / previous tile consumed
    // (c, tt) with tt contiguous in memory -> s_in[(c*f + j)][p], tt = p*f + j
    const int span = kWideTP * a.f;
    for (int i = threadIdx.x; i < cin * span; i += blockDim.x) {
      const int c = i / span, r = i - c * span, pp = r / a.f, j = r - pp * a.f;
      const size_t tt = static_cast<size_t>(to0) * a.f + r;
      float v = 0.f;
      if (to0 + pp < To) v = block_input<true>(a, b, c, tt, al, be);
      s_in[(c * a.f + j) * LD + pp] = v;
    }
    __syncthreads();
    const int to = to0 + p;
    const bool ok = to < To;
    __nv_bfloat16* orow =
        static_cast<__nv_bfloat16*>(a.out) + (static_cast<size_t>(b) * To + (ok ? to : 0)) * a.c0;
    for (int ch = cg; ch < a.c0 / 8; ch += 256 / kWideTP) {
      float v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = s_b[ch * 8 + j];
      for (int ii = 0; ii < ci_total; ++ii) {
        const float xv = s_in[ii * LD + p];
        const float4 w0 = *reinterpret_cast<const float4*>(s_w + ii * a.c0 + ch * 8);
        const float4 w1 = *reinterpret_cast<const float4*>(s_w + ii * a.c0 + ch * 8 + 4);
        v[0] += xv * w0.x; v[1] += xv * w0.y; v[2] += xv * w0.z; v[3] += xv * w0.w;
        v[4] += xv * w1.x; v[5] += xv * w1.y; v[6] += xv * w1.z; v[7] += xv * w1.w;
      }
      uint4 o;
      o.x = pack_bf16(v[0], v[1]); o.y = pack_bf16(v[2], v[3]);
      o.z = pack_bf16(v[4], v[5]); o.w = pack_bf16(v[6], v[7]);
      if (ok) *reinterpret_cast<uint4*>(orow + ch * 8) = o;
      if (a.stats) {        // statistics of the ROUNDED values the next layer reads
        const uint32_t ou[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 r = unpack_bf16(ou[j]);
          acc.add(ok ? r.x : 0.f, (ch * 8 + 2 * j) / gsz, s_stats, lane);
          acc.add(ok ? r.y : 0.f, (ch * 8 + 2 * j + 1) / gsz, s_stats, lane);
        }
      }
    }
  }
  if (a.stats) {
    acc.flush(s_stats, lane);
    __syncthreads();
    flush_group_stats(s_stats, a.stats, b, a.groups);
  }
}

// ----------------------------------------------------------------- wide boundary (stem_out)
// Up to 64 outputs and 64 block-input channels.  A tile is kWideOP output positions; the conv3 on
// the nearest-upsampled h runs over c0 in chunks of kWideCK channels (h rows and the [co][3][ck]
// weight slice staged in smem, 192 KiB of weights at co = 64, c0 = 256 never resident at once).
// Thread = (position, output parity): up to 32 outputs per thread accumulate in registers, the
// warp shares its outputs (broadcast weight reads).  The block input cat([x(_noisy), append]) of
// the whole tile is staged before any store, so x_next may alias x.
constexpr int kWideOP = 128;
constexpr int kWideCK = 32;
constexpr int kWideHL = kWideCK + 4;     // padded h row (16-byte aligned)
constexpr int kWideOPT = kStemMaxCo / 2; // outputs per thread

__device__ __forceinline__ void stem_out_wide_conv(const adp_stem_out_args& a, const __nv_bfloat16* hb,
                                                   float* s_h, const float* s_wc, int t0, int q_base,
                                                   int rows, int c_base, int p, int og,
                                                   float (&y)[kWideOPT]) {
  const int Tl = a.T / a.f;
  const int nck = min(kWideCK, a.c0 - c_base);
  __syncthreads();                                 // s_h free
  for (int i = threadIdx.x; i < rows * (kWideCK / 8); i += blockDim.x) {
    const int r = i / (kWideCK / 8), c8 = (i - r * (kWideCK / 8)) * 8, q = q_base + r;
    float4 lo = make_float4(0.f, 0.f, 0.f, 0.f), hi = lo;
    if (q >= 0 && q < Tl && c8 < nck) {
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(hb + static_cast<size_t>(q) * a.c0 + c_base + c8));
      const float2 f0 = unpack_bf16(u.x), f1 = unpack_bf16(u.y), f2 = unpack_bf16(u.z), f3 = unpack_bf16(u.w);
      lo = make_float4(f0.x, f0.y, f1.x, f1.y);
      hi = make_float4(f2.x, f2.y, f3.x, f3.y);
    }
    *reinterpret_cast<float4*>(s_h + r * kWideHL + c8) = lo;
    *reinterpret_cast<float4*>(s_h + r * kWideHL + c8 + 4) = hi;
  }
  __syncthreads();
  const int t = t0 + p;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int u = t + k - 1;
    if (u < 0 || u >= a.T) continue;               // zero padding of the upsampled signal
    const float* hr = s_h + (u / a.f - q_base) * kWideHL;
    for (int c4 = 0; c4 < nck; c4 += 4) {
      const float4 hv = *reinterpret_cast<const float4*>(hr + c4);
#pragma unroll
      for (int m = 0; m < kWideOPT; ++m) {
        const int o = og + 2 * m;
        if (o < a.co) {
          const float4 w = *reinterpret_cast<const float4*>(s_wc + (o * 3 + k) * kWideCK + c4);
          y[m] += (hv.x * w.x + hv.y * w.y) + (hv.z * w.z + hv.w * w.w);
        }
      }
    }
  }
}

__global__ void __launch_bounds__(256) stem_out_wide_kernel(const adp_stem_out_args a) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ __align__(16) float s_dyn[];
  const int cin = a.cx + a.ca;
  const int rows = (kWideOP + 1) / a.f + 2;        // low-rate rows feeding positions t0-1 .. t0+OP
  float* s_wc = s_dyn;                             // [co][3][CK] weight slice of one c0 chunk
  float* s_h = s_wc + a.co * 3 * kWideCK;          // [rows][HL]
  float* s_xin = s_h + rows * kWideHL;             // [cin][OP]
  float* s_wa = s_xin + cin * kWideOP;             // [co][cin]
  float* s_ba = s_wa + a.co * cin;                 // [co]
  if (a.w_adapt)
    for (int i = threadIdx.x; i < a.co * cin; i += blockDim.x) s_wa[i] = a.w_adapt[i];
  for (int i = threadIdx.x; i < a.co; i += blockDim.x) s_ba[i] = a.b_adapt ? a.b_adapt[i] : 0.f;

  const int b = blockIdx.y;
  const int p = threadIdx.x % kWideOP, og = threadIdx.x / kWideOP;
  const int Tl = a.T / a.f;
  const float al = a.noise ? a.alpha[b] : 1.f, be = a.noise ? a.beta[b] : 0.f;
  const __nv_bfloat16* h = static_cast<const __nv_bfloat16*>(a.h);
  double lsum = 0.0;
  const int n_tiles = (a.T + kWideOP - 1) / kWideOP;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int t0 = tile * kWideOP;
    const int q_base = t0 == 0 ? -1 : (t0 - 1) / a.f;
    const int t = t0 + p;
    const bool ok = t < a.T;
    __syncthreads();                               // previous tile's s_xin consumed
    for (int i = threadIdx.x; i < cin * kWideOP; i += blockDim.x) {
      const int c = i / kWideOP, r = i - c * kWideOP, tt = t0 + r;
      s_xin[i] = tt < a.T ? block_input(a, b, c, tt, al, be) : 0.f;
    }
    float y[kWideOPT], ym[kWideOPT];
#pragma unroll
    for (int m = 0; m < kWideOPT; ++m) {
      const int o = og + 2 * m;
      y[m] = (o < a.co && a.bias) ? a.bias[o] : 0.f;
      ym[m] = y[m];
    }
    for (int c_base = 0; c_base < a.c0; c_base += kWideCK) {
      const int nck = min(kWideCK, a.c0 - c_base);
      __syncthreads();                             // s_wc free
      for (int i = threadIdx.x; i < a.co * 3 * kWideCK; i += blockDim.x) {
        // PyTorch layout [co][c0][3] -> [co][3][CK], zero beyond the chunk
        const int o = i / (3 * kWideCK), r = i - o * 3 * kWideCK, k = r / kWideCK, c = r - k * kWideCK;
        s_wc[i] = c < nck ? a.w[(static_cast<size_t>(o) * a.c0 + c_base + c) * 3 + k] : 0.f;
      }
      stem_out_wide_conv(a, h + static_cast<size_t>(b) * Tl * a.c0, s_h, s_wc, t0, q_base, rows, c_base,
                         p, og, y);
      if (a.cfg)
        stem_out_wide_conv(a, h + static_cast<size_t>(b + a.B) * Tl * a.c0, s_h, s_wc, t0, q_base, rows,
                           c_base, p, og, ym);
    }
    if (!ok) continue;
#pragma unroll
    for (int m = 0; m < kWideOPT; ++m) {
      const int o = og + 2 * m;
      if (o >= a.co) continue;
      float skip;
      if (a.w_adapt) {                             // SkipAdapter 1x1 conv (in != out channels)
        skip = s_ba[o];
        for (int c = 0; c < cin; ++c) skip += s_xin[c * kWideOP + p] * s_wa[o * cin + c];
      } else {
        skip = s_xin[o * kWideOP + p];
      }
      stem_out_finish(a, b, o, t, skip, y[m], ym[m], s_xin[o * kWideOP + p], al, be, lsum);
    }
  }
  if (a.loss_sum) block_loss_flush(lsum, a.loss_sum);
}

int mid_conv(const adp_narrow_conv_args& a, cudaStream_t stream);   // mid_conv.cu

}  // namespace adp

using namespace adp;

extern "C" int adp_stem_in(const adp_stem_in_args* args, adp_stream_t stream) {
  ADP_CHECK(args && args->x && args->w && args->out, "adp_stem_in: null pointer");
  const adp_stem_in_args& a = *args;
  if (int e = check_stem_envelope("adp_stem_in", a.cx, a.ca, a.c0, a.f, a.T, 1)) return e;
  ADP_CHECK((a.ca == 0) == (a.append == nullptr), "adp_stem_in: append / ca mismatch");
  ADP_CHECK(!a.noise || (a.alpha && a.beta), "adp_stem_in: noise needs alpha/beta");
  if (a.stats) ADP_CHECK(a.groups > 0 && a.groups <= 64 && a.c0 % a.groups == 0, "adp_stem_in: groups");
  const int ci_total = (a.cx + a.ca) * a.f;
  if (stem_in_narrow(a)) {
    const size_t smem = (static_cast<size_t>(a.c0) * ci_total + a.c0) * sizeof(float);
    auto kernel = ci_total <= 4 ? stem_in_kernel<4> : stem_in_kernel<kStemInNarrowIn>;
    // with its 16.5 KiB of static shared memory the weights pass the 48 KiB default from
    // c0 (ci_total + 1) > 7808 (c0 = 256 at 30 to 32 inputs per position)
    static SmemAttrCache smem_cache4, smem_cache;
    ADP_CUDA(ensure_dyn_smem(kernel, smem, ci_total <= 4 ? smem_cache4 : smem_cache));
    dim3 grid(one_wave_gx(kernel, 256, smem, a.B, (a.T / a.f + 255) / 256), a.B);
    ADP_CUDA(launch_k(kernel, grid, dim3(256), smem, as_stream(stream), a));
  } else {
    const size_t smem = (static_cast<size_t>(ci_total) * (a.c0 + kWideTP + 1) + a.c0) * sizeof(float);
    static SmemAttrCache smem_cache;
    ADP_CUDA(ensure_dyn_smem(stem_in_wide_kernel, smem, smem_cache));
    dim3 grid(one_wave_gx(stem_in_wide_kernel, 256, smem, a.B, (a.T / a.f + kWideTP - 1) / kWideTP), a.B);
    ADP_CUDA(launch_k(stem_in_wide_kernel, grid, dim3(256), smem, as_stream(stream), a));
  }
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_stem_out(const adp_stem_out_args* args, adp_stream_t stream) {
  ADP_CHECK(args && args->h && args->x && args->w && args->gate, "adp_stem_out: null pointer");
  const adp_stem_out_args& a = *args;
  if (int e = check_stem_envelope("adp_stem_out", a.cx, a.ca, a.c0, a.f, a.T, a.co)) return e;
  const int cin = a.cx + a.ca;
  ADP_CHECK(a.w_adapt || cin == a.co, "adp_stem_out: identity skip needs cx+ca == co");
  ADP_CHECK((a.ca == 0) == (a.append == nullptr), "adp_stem_out: append / ca mismatch");
  ADP_CHECK(!a.x_next || a.ab, "adp_stem_out: x_next needs ab");
  ADP_CHECK(!a.loss_sum || (a.noise && a.alpha && a.beta), "adp_stem_out: loss needs noise/alpha/beta");
  ADP_CHECK(!a.loss_sum || !a.x_next, "adp_stem_out: the loss excludes the sampler fusion");
  if (stem_out_narrow(a)) {
    const size_t smem = (static_cast<size_t>(a.co) * 3 * a.c0 + 2 * a.co + a.co * cin) * sizeof(float);
    dim3 grid(one_wave_gx(stem_out_kernel, 256, smem, a.B, (a.T + 255) / 256), a.B);
    ADP_CUDA(launch_k(stem_out_kernel, grid, dim3(256), smem, as_stream(stream), a));
  } else {
    const int rows = (kWideOP + 1) / a.f + 2;
    const size_t smem = (static_cast<size_t>(a.co) * 3 * kWideCK + static_cast<size_t>(rows) * kWideHL +
                         static_cast<size_t>(cin) * kWideOP + a.co * cin + a.co) * sizeof(float);
    static SmemAttrCache smem_cache;
    ADP_CUDA(ensure_dyn_smem(stem_out_wide_kernel, smem, smem_cache));
    dim3 grid(one_wave_gx(stem_out_wide_kernel, 256, smem, a.B, (a.T + kWideOP - 1) / kWideOP), a.B);
    ADP_CUDA(launch_k(stem_out_wide_kernel, grid, dim3(256), smem, as_stream(stream), a));
  }
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_narrow_conv(const adp_narrow_conv_args* args, adp_stream_t stream) {
  ADP_CHECK(args && args->x && args->y && args->stats_in && args->gamma && args->beta && args->w,
            "adp_narrow_conv: null pointer");
  const adp_narrow_conv_args& a = *args;
  ADP_CHECK(a.C == 8 || a.C == 32 || a.C == 64,
            "adp_narrow_conv: C=%d is not built (8, 32, 64); wider levels use adp_conv_gemm", a.C);
  ADP_CHECK(a.groups > 0 && a.C % a.groups == 0 && a.groups <= 64, "adp_narrow_conv: groups=%d", a.groups);
  if (a.C != 8) {
    ADP_CHECK(!a.stats_out || (a.C / a.groups) % 4 == 0,
              "adp_narrow_conv: group size %d must be a multiple of 4 (fused statistics)", a.C / a.groups);
    if (int e = mid_conv(a, as_stream(stream))) return e;
    ADP_LAUNCH_CHECK();
    return 0;
  }
  // persistent blocks: one wave of resident blocks shares the tiles of each batch element
  dim3 grid(one_wave_gx(narrow_conv_kernel<8>, 256, 0, a.B, (a.T + 255) / 256), a.B);
  ADP_CUDA(launch_k(narrow_conv_kernel<8>, grid, dim3(256), (size_t)0, as_stream(stream), a));
  ADP_LAUNCH_CHECK();
  return 0;
}
