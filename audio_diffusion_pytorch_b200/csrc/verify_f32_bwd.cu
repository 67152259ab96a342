// fp32 VERIFICATION MODE, training half: the backward launch kinds of the training program
// (training.build_train_plan) with fp32 activations and activation gradients, in the style of
// verify_f32.cu -- one thread per output, no tiling, exact transcendentals, fixed-order sums.
// Atomics remain only where several threads of one launch add to one element (a parameter gradient
// summed over the batch, a GroupNorm group summed over its channels), as in the bf16 kernels.
// Entry points take the arguments of the bf16 entry point they shadow, every activation pointer
// fp32.  Not a performance path.
#include "stem.cuh"

namespace adp {
namespace {

__device__ __forceinline__ float sigmoid_exact(float z) { return 1.f / (1.f + expf(-z)); }

// a load ptxas may not hoist out of a loop (keeps a thread's own row out of its registers)
__device__ __forceinline__ float ld_nc_once(const float* p) {
  float v;
  asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}

// GroupNorm coefficients of (b, channel c) exactly as f32_gn_silu_kernel computes them
struct GnCoef { float mean, rstd; };
__device__ __forceinline__ GnCoef gn_coef(const double* stats, int b, int c, int T, int C, int groups,
                                          float eps) {
  const int gsz = C / groups;
  const double inv_n = 1.0 / (static_cast<double>(gsz) * T);
  const double* st = stats + (static_cast<int64_t>(b) * groups + c / gsz) * 2;
  const double mean = st[0] * inv_n;
  const double var = fmax(st[1] * inv_n - mean * mean, 0.0);
  return {static_cast<float>(mean), static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)))};
}

#define F32B_GRID_STRIDE(i, total)                                                     \
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < (total); \
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)

// ------------------------------------------------------------------------------ wgrad
// dw[tap][n][k] += sum_{b,t} g[b,t,g_col0+n] * x[b,t+off+tap,x_col0+k]; one thread per element
__global__ void __launch_bounds__(256) f32_wgrad_kernel(const adp_wgrad_args a) {
  pdl_launch_dependents();
  pdl_wait();
  const float* G = static_cast<const float*>(a.g);
  const float* X = static_cast<const float*>(a.x);
  const int taps = a.ntaps == 3 ? 3 : 1;
  const int64_t nk = static_cast<int64_t>(a.n) * a.k;
  F32B_GRID_STRIDE(i, taps * nk) {
    const int tap = static_cast<int>(i / nk);
    const int r = static_cast<int>(i - tap * nk);
    const int n = r / a.k, k = r - n * a.k;
    const int off = a.off + tap;
    const int t_lo = off < 0 ? -off : 0, t_hi = off > 0 ? a.T - off : a.T;
    float acc = 0.f;
    for (int b = 0; b < a.B; ++b) {
      const float* gb = G + static_cast<int64_t>(b) * a.T * a.ldg + a.g_col0 + n;
      const float* xb = X + static_cast<int64_t>(b) * a.T * a.ldx + a.x_col0 + k;
      for (int t = t_lo; t < t_hi; ++t)
        acc = fmaf(gb[static_cast<int64_t>(t) * a.ldg], xb[static_cast<int64_t>(t + off) * a.ldx], acc);
    }
    a.dw[tap * a.tap_stride + static_cast<int64_t>(n) * a.ldw + k] += acc;
  }
}

// ------------------------------------------------------------------ GroupNorm + SiLU backward
// pass 1, one thread per (b, c): dz = da * silu'(z); dxh = dz*gamma; dgamma += sum dz*xhat,
// dbeta += sum dz, S[b][g] += (sum dxh, sum dxh*xhat)
__global__ void __launch_bounds__(256)
f32_gn_silu_bwd_kernel(const float* __restrict__ da, const float* __restrict__ x, const double* __restrict__ stats,
                       const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ dxh,
                       float* __restrict__ dgamma, float* __restrict__ dbeta, double* __restrict__ S, int B, int T,
                       int C, int groups, float eps) {
  pdl_launch_dependents();
  pdl_wait();
  F32B_GRID_STRIDE(i, static_cast<int64_t>(B) * C) {
    const int b = static_cast<int>(i / C), c = static_cast<int>(i % C);
    const GnCoef k = gn_coef(stats, b, c, T, C, groups, eps);
    const float g = gamma[c], be = beta[c];
    float dg = 0.f, db = 0.f, s1 = 0.f, s2 = 0.f;
    for (int t = 0; t < T; ++t) {
      const int64_t idx = (static_cast<int64_t>(b) * T + t) * C + c;
      const float xh = (x[idx] - k.mean) * k.rstd;
      const float z = xh * g + be;
      const float sg = sigmoid_exact(z);
      const float dz = da[idx] * sg * (1.f + z * (1.f - sg));
      const float o = dz * g;
      dxh[idx] = o;
      dg += dz * xh; db += dz; s1 += o; s2 += o * xh;
    }
    atomicAdd(dgamma + c, dg);
    atomicAdd(dbeta + c, db);
    double* sb = S + (static_cast<int64_t>(b) * groups + c / (C / groups)) * 2;
    atomicAdd(sb, static_cast<double>(s1));
    atomicAdd(sb + 1, static_cast<double>(s2));
  }
}

// pass 2, one thread per (b, c): dx = rstd*(dxh - S1/n - xhat*S2/n) [+ dres]; colsum[c] += sum dx
__global__ void __launch_bounds__(256)
f32_gn_bwd_apply_kernel(const float* __restrict__ dxh, const float* __restrict__ x, const double* __restrict__ stats,
                        const double* __restrict__ S, const float* __restrict__ dres, float* __restrict__ dx,
                        float* __restrict__ colsum, int B, int T, int C, int groups, float eps) {
  pdl_launch_dependents();
  pdl_wait();
  const int gsz = C / groups;
  const double inv_n = 1.0 / (static_cast<double>(gsz) * T);
  F32B_GRID_STRIDE(i, static_cast<int64_t>(B) * C) {
    const int b = static_cast<int>(i / C), c = static_cast<int>(i % C);
    const GnCoef k = gn_coef(stats, b, c, T, C, groups, eps);
    const double* sb = S + (static_cast<int64_t>(b) * groups + c / gsz) * 2;
    const float c1 = static_cast<float>(sb[0] * inv_n), c2 = static_cast<float>(sb[1] * inv_n);
    float cs = 0.f;
    for (int t = 0; t < T; ++t) {
      const int64_t idx = (static_cast<int64_t>(b) * T + t) * C + c;
      const float xh = (x[idx] - k.mean) * k.rstd;
      float o = k.rstd * (dxh[idx] - c1 - xh * c2);
      if (dres) o += dres[idx];
      dx[idx] = o;
      cs += o;
    }
    if (colsum) atomicAdd(colsum + c, cs);
  }
}

// ---------------------------------------------------------------------- LayerNorm-FiLM backward
// y = xhat*(1+s) + t per row (f32_ln_film_kernel).  One warp per (b, 32-channel chunk), walking
// the rows of b in order: the warp recomputes the row statistics, then each lane owns one channel:
// dx = rstd*(g - mean(g) - xhat*mean(g*xhat)) [+ dres], g = dy*(1+s); dss[b][c] += sum_t dy*xhat,
// dss[b][C+c] += sum_t dy; colsum[c] += sum dx.
__global__ void __launch_bounds__(256)
f32_ln_film_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ ss,
                       int ss_stride, float* __restrict__ dx, float* __restrict__ dss, int dss_stride,
                       float* __restrict__ colsum, const float* __restrict__ dres, int B, int T, int C, float eps) {
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int chunks = (C + 31) / 32;
  const int64_t warps = static_cast<int64_t>(B) * chunks;
  for (int64_t w = static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5); w < warps;
       w += static_cast<int64_t>(gridDim.x) * 8) {
    const int b = static_cast<int>(w / chunks);
    const int c = static_cast<int>(w % chunks) * 32 + lane;
    const bool own = c < C;
    const float* sc = ss ? ss + static_cast<int64_t>(b) * ss_stride : nullptr;
    float ads = 0.f, adt = 0.f, acs = 0.f;
    for (int t = 0; t < T; ++t) {
      const int64_t r = static_cast<int64_t>(b) * T + t;
      const float* xr = x + r * C;
      const float* dr = dy + r * C;
      float m = 0.f;
      for (int cc = lane; cc < C; cc += 32) m += xr[cc];
      m = warp_sum(m) / C;
      float v = 0.f;
      for (int cc = lane; cc < C; cc += 32) { const float d = xr[cc] - m; v += d * d; }
      const float rstd = rsqrtf(warp_sum(v) / C + eps);
      float m1 = 0.f, m2 = 0.f;
      for (int cc = lane; cc < C; cc += 32) {
        const float g = dr[cc] * (sc ? 1.f + sc[cc] : 1.f);
        m1 += g; m2 += g * ((xr[cc] - m) * rstd);
      }
      m1 = warp_sum(m1) / C;
      m2 = warp_sum(m2) / C;
      if (own) {
        const float xh = (xr[c] - m) * rstd;
        const float d = dr[c];
        float o = rstd * (d * (sc ? 1.f + sc[c] : 1.f) - m1 - xh * m2);
        if (dres) o += dres[r * C + c];
        dx[r * C + c] = o;
        ads += d * xh; adt += d; acs += o;
      }
    }
    if (own) {
      if (dss) {                         // this warp is the only writer of (b, c) and (b, C + c)
        dss[static_cast<int64_t>(b) * dss_stride + c] += ads;
        dss[static_cast<int64_t>(b) * dss_stride + C + c] += adt;
      }
      if (colsum) atomicAdd(colsum + c, acs);
    }
  }
}

// ----------------------------------------------------------------------------- colsum
// out[c] += sum_b gate[b][c] * sum_t x[b][t][c]  (gate == NULL: 1); one thread per channel
__global__ void __launch_bounds__(256)
f32_colsum_kernel(const float* __restrict__ x, const float* __restrict__ gate, int ld_gate, float* __restrict__ out,
                  int B, int T, int C) {
  pdl_launch_dependents();
  pdl_wait();
  F32B_GRID_STRIDE(c, C) {
    float acc = 0.f;
    for (int b = 0; b < B; ++b) {
      float s = 0.f;
      for (int t = 0; t < T; ++t) s += x[(static_cast<int64_t>(b) * T + t) * C + c];
      acc += gate ? s * gate[static_cast<int64_t>(b) * ld_gate + c] : s;
    }
    out[c] += acc;
  }
}

// --------------------------------------------------------------------------- skip_gate
// out = skip + gate[b][c] * y (the GroupNorm statistics of out are a separate adp_f32_gn_stats pass)
__global__ void __launch_bounds__(256)
f32_skip_gate_kernel(const float* __restrict__ y, const float* __restrict__ skip, const float* __restrict__ gate,
                     int ld_gate, float* __restrict__ out, int B, int T, int C) {
  pdl_launch_dependents();
  pdl_wait();
  F32B_GRID_STRIDE(i, static_cast<int64_t>(B) * T * C) {
    const int c = static_cast<int>(i % C);
    const int b = static_cast<int>(i / (static_cast<int64_t>(T) * C));
    out[i] = skip[i] + gate[static_cast<int64_t>(b) * ld_gate + c] * y[i];
  }
}

// dys = gate*dout; dgate[b][c] += sum_t dout*y.  One thread per (b, c)
__global__ void __launch_bounds__(256)
f32_skip_gate_bwd_kernel(const float* __restrict__ dout, const float* __restrict__ y, const float* __restrict__ gate,
                         int ld_gate, float* __restrict__ dys, float* __restrict__ dgate, int ld_dgate, int B, int T,
                         int C) {
  pdl_launch_dependents();
  pdl_wait();
  F32B_GRID_STRIDE(i, static_cast<int64_t>(B) * C) {
    const int b = static_cast<int>(i / C), c = static_cast<int>(i % C);
    const float g = gate[static_cast<int64_t>(b) * ld_gate + c];
    float acc = 0.f;
    for (int t = 0; t < T; ++t) {
      const int64_t idx = (static_cast<int64_t>(b) * T + t) * C + c;
      dys[idx] = g * dout[idx];
      acc += dout[idx] * y[idx];
    }
    dgate[static_cast<int64_t>(b) * ld_dgate + c] += acc;
  }
}

// ---------------------------------------------------------------------------- cond_bwd
// ss[b][n] = sum_k cond[b][k] W[n][k] + bias[n]:  dW[n][k] = sum_b dss[b][n] cond[b][k] and
// dbias[n] = sum_b dss[b][n] (stored, as adp_cond_bwd does); dcond[b][k] += sum_n dss[b][n] W[n][k]
__global__ void __launch_bounds__(256)
f32_cond_bwd_w_kernel(const float* __restrict__ dss, int ld_dss, const float* __restrict__ cond,
                      float* __restrict__ dw, float* __restrict__ dbias, int B, int N, int K) {
  pdl_launch_dependents();
  pdl_wait();
  F32B_GRID_STRIDE(i, static_cast<int64_t>(N) * K) {
    const int n = static_cast<int>(i / K), k = static_cast<int>(i % K);
    float acc = 0.f, accb = 0.f;
    for (int b = 0; b < B; ++b) {
      const float d = dss[static_cast<int64_t>(b) * ld_dss + n];
      acc = fmaf(d, cond[static_cast<int64_t>(b) * K + k], acc);
      accb += d;
    }
    dw[i] = acc;
    if (k == 0) dbias[n] = accb;
  }
}

__global__ void __launch_bounds__(256)
f32_cond_bwd_x_kernel(const float* __restrict__ dss, int ld_dss, const float* __restrict__ w,
                      float* __restrict__ dcond, int B, int N, int K) {
  pdl_launch_dependents();
  pdl_wait();
  F32B_GRID_STRIDE(i, static_cast<int64_t>(B) * K) {
    const int b = static_cast<int>(i / K), k = static_cast<int>(i % K);
    float acc = 0.f;
    for (int n = 0; n < N; ++n)
      acc = fmaf(dss[static_cast<int64_t>(b) * ld_dss + n], w[static_cast<int64_t>(n) * K + k], acc);
    dcond[i] += acc;
  }
}

// ------------------------------------------------------------------------ stem_out backward
// forward (f32_stem_out_kernel): v[b,o,t] = skip(xin)[o] + gate[b][o] * y[b,o,t],
// y = bias[o] + sum_{k,c} h[b, (t+k-1)/f, c] w[o][c][k].  dvs = dv * gscale, dy = dvs * gate.
__device__ __forceinline__ float so_dvs(const adp_stem_out_bwd_args& a, int b, int o, int t) {
  return a.dv[(static_cast<int64_t>(b) * a.co + o) * a.T + t] * (a.gscale ? a.gscale[0] : 1.f);
}
__device__ __forceinline__ float so_dy(const adp_stem_out_bwd_args& a, int b, int o, int t) {
  const int ldg = a.ld_gate > 0 ? a.ld_gate : a.co;
  return so_dvs(a, b, o, t) * a.gate[static_cast<int64_t>(b) * ldg + o];
}

// dh[b][q][c] = sum over the upsampled positions u fed by row q and taps k of dy[t = u-k+1] w[o][c][k]
__global__ void __launch_bounds__(256) f32_stem_out_bwd_dh_kernel(const adp_stem_out_bwd_args a) {
  pdl_launch_dependents();
  pdl_wait();
  const int Tl = a.T / a.f;
  float* dh = static_cast<float*>(a.dh);
  F32B_GRID_STRIDE(i, static_cast<int64_t>(a.B) * Tl * a.c0) {
    const int c = static_cast<int>(i % a.c0);
    const int q = static_cast<int>((i / a.c0) % Tl);
    const int b = static_cast<int>(i / (static_cast<int64_t>(a.c0) * Tl));
    float acc = 0.f;
    for (int u = q * a.f; u < q * a.f + a.f; ++u)
      for (int k = 0; k < 3; ++k) {
        const int tp = u - k + 1;
        if (tp < 0 || tp >= a.T) continue;
        for (int o = 0; o < a.co; ++o) acc = fmaf(so_dy(a, b, o, tp), a.w[(o * a.c0 + c) * 3 + k], acc);
      }
    dh[i] = acc;
  }
}

// one thread per parameter-gradient element: dw [co][c0][3], dbias [co], dgate [B][co],
// dw_adapt [co][cin], db_adapt [co]
__global__ void __launch_bounds__(256) f32_stem_out_bwd_param_kernel(const adp_stem_out_bwd_args a) {
  pdl_launch_dependents();
  pdl_wait();
  const int cin = a.cx + a.ca, Tl = a.T / a.f;
  const float* h = static_cast<const float*>(a.h);
  const int n_w = a.co * a.c0 * 3, n_g = a.B * a.co, n_ad = a.w_adapt ? a.co * cin : 0;
  const int n_items = n_w + a.co + n_g + (a.w_adapt ? n_ad + a.co : 0);
  F32B_GRID_STRIDE(item64, n_items) {
    const int item = static_cast<int>(item64);
    float acc = 0.f;
    if (item < n_w) {                                   // dw[o][c][k]
      const int o = item / (a.c0 * 3), r = item - o * a.c0 * 3, c = r / 3, k = r - c * 3;
      for (int b = 0; b < a.B; ++b)
        for (int t = 0; t < a.T; ++t) {
          const int u = t + k - 1;
          if (u < 0 || u >= a.T) continue;
          acc = fmaf(so_dy(a, b, o, t), h[(static_cast<int64_t>(b) * Tl + u / a.f) * a.c0 + c], acc);
        }
      a.dw[item] += acc;
    } else if (item < n_w + a.co) {                     // dbias[o]
      const int o = item - n_w;
      for (int b = 0; b < a.B; ++b)
        for (int t = 0; t < a.T; ++t) acc += so_dy(a, b, o, t);
      a.dbias[o] += acc;
    } else if (item < n_w + a.co + n_g) {               // dgate[b][o] = sum_t dvs * y
      const int r = item - n_w - a.co, b = r / a.co, o = r - b * a.co;
      const float* hb = h + static_cast<int64_t>(b) * Tl * a.c0;
      for (int t = 0; t < a.T; ++t) {
        float y = a.bias ? a.bias[o] : 0.f;
        for (int k = 0; k < 3; ++k) {
          const int u = t + k - 1;
          if (u < 0 || u >= a.T) continue;
          const float* row = hb + static_cast<int64_t>(u / a.f) * a.c0;
          for (int c = 0; c < a.c0; ++c) y = fmaf(row[c], a.w[(o * a.c0 + c) * 3 + k], y);
        }
        acc = fmaf(so_dvs(a, b, o, t), y, acc);
      }
      a.dgate[static_cast<int64_t>(b) * a.ld_dgate + o] += acc;
    } else if (item < n_w + a.co + n_g + n_ad) {        // dw_adapt[o][c]
      const int r = item - n_w - a.co - n_g, o = r / cin, c = r - o * cin;
      for (int b = 0; b < a.B; ++b) {
        const float al = a.noise ? a.alpha[b] : 1.f, be = a.noise ? a.beta[b] : 0.f;
        for (int t = 0; t < a.T; ++t) acc = fmaf(so_dvs(a, b, o, t), block_input(a, b, c, t, al, be), acc);
      }
      a.dw_adapt[r] += acc;
    } else {                                            // db_adapt[o]
      const int o = item - n_w - a.co - n_g - n_ad;
      for (int b = 0; b < a.B; ++b)
        for (int t = 0; t < a.T; ++t) acc += so_dvs(a, b, o, t);
      a.db_adapt[o] += acc;
    }
  }
}

// dxin[b][c][t] = (W_adapt^T dvs)[c] or dvs[c] (identity skip), STORED
__global__ void __launch_bounds__(256) f32_stem_out_bwd_dxin_kernel(const adp_stem_out_bwd_args a) {
  pdl_launch_dependents();
  pdl_wait();
  const int cin = a.cx + a.ca;
  F32B_GRID_STRIDE(i, static_cast<int64_t>(a.B) * cin * a.T) {
    const int t = static_cast<int>(i % a.T);
    const int c = static_cast<int>((i / a.T) % cin);
    const int b = static_cast<int>(i / (static_cast<int64_t>(a.T) * cin));
    float acc = 0.f;
    if (a.w_adapt) {
      for (int o = 0; o < a.co; ++o) acc = fmaf(so_dvs(a, b, o, t), a.w_adapt[o * cin + c], acc);
    } else if (c < a.co) {
      acc = so_dvs(a, b, c, t);
    }
    a.dxin[i] = acc;
  }
}

// ------------------------------------------------------------------------- stem_in backward
// forward (f32_stem_in_kernel): out[b,to,o] = bias[o] + sum_{c,j} w[o][c][j] xin[b,c,to*f+j]
__global__ void __launch_bounds__(256) f32_stem_in_bwd_param_kernel(const adp_stem_in_bwd_args a) {
  pdl_launch_dependents();
  pdl_wait();
  const int cin = a.cx + a.ca, ci_total = cin * a.f, To = a.T / a.f;
  const float* g = static_cast<const float*>(a.dout);
  const int n_w = a.c0 * ci_total;
  F32B_GRID_STRIDE(item64, n_w + a.c0) {
    const int item = static_cast<int>(item64);
    float acc = 0.f;
    if (item < n_w) {                                   // dw[o][c][j]
      const int o = item / ci_total, r = item - o * ci_total, c = r / a.f, j = r - c * a.f;
      for (int b = 0; b < a.B; ++b) {
        const float al = a.noise ? a.alpha[b] : 1.f, be = a.noise ? a.beta[b] : 0.f;
        for (int to = 0; to < To; ++to)
          acc = fmaf(g[(static_cast<int64_t>(b) * To + to) * a.c0 + o],
                     block_input(a, b, c, static_cast<size_t>(to) * a.f + j, al, be), acc);
      }
      a.dw[item] += acc;
    } else {
      const int o = item - n_w;
      for (int b = 0; b < a.B; ++b)
        for (int to = 0; to < To; ++to) acc += g[(static_cast<int64_t>(b) * To + to) * a.c0 + o];
      a.dbias[o] += acc;
    }
  }
}

// dxin[b][c][t] += sum_o dout[b][t/f][o] w[o][c][t%f]  (after adp_f32_stem_out_bwd stored its part)
__global__ void __launch_bounds__(256) f32_stem_in_bwd_dxin_kernel(const adp_stem_in_bwd_args a) {
  pdl_launch_dependents();
  pdl_wait();
  const int cin = a.cx + a.ca, To = a.T / a.f;
  const float* g = static_cast<const float*>(a.dout);
  F32B_GRID_STRIDE(i, static_cast<int64_t>(a.B) * cin * a.T) {
    const int t = static_cast<int>(i % a.T);
    const int c = static_cast<int>((i / a.T) % cin);
    const int b = static_cast<int>(i / (static_cast<int64_t>(a.T) * cin));
    const int to = t / a.f, j = t - to * a.f;
    float acc = 0.f;
    for (int o = 0; o < a.c0; ++o)
      acc = fmaf(g[(static_cast<int64_t>(b) * To + to) * a.c0 + o], a.w[(o * cin + c) * a.f + j], acc);
    a.dxin[i] += acc;
  }
}

// ------------------------------------------------------------------------ attention backward
// forward (f32_attention_kernel): s_ij = sum_d (q_i[d]*scale) k_j[d], P = exp(s - lse_i).
//   delta_i = sum_d dO_i o_i;  dS_ij = P_ij (dO_i.v_j - delta_i)
//   dq_i = scale sum_j dS_ij k_j;  dk_j = scale sum_i dS_ij q_i;  dv_j = sum_i P_ij dO_i
// One thread per query row (delta, dq) or key row (dk, dv); the output columns are produced 32 at a
// time, each pass recomputing the scores (the thread's own rows are re-read, not held).
constexpr int kAttCols = 32;

__global__ void __launch_bounds__(256) f32_attention_delta_kernel(const adp_attention_bwd_args a, int D) {
  pdl_launch_dependents();
  pdl_wait();
  const float* O = static_cast<const float*>(a.o);
  const float* dO = static_cast<const float*>(a.d_o);
  F32B_GRID_STRIDE(i, static_cast<int64_t>(a.B) * a.H * a.Tq) {
    const int tq = static_cast<int>(i % a.Tq);
    const int h = static_cast<int>((i / a.Tq) % a.H);
    const int b = static_cast<int>(i / (static_cast<int64_t>(a.Tq) * a.H));
    const float* orow = O + (static_cast<int64_t>(b) * a.Tq + tq) * a.ldo + h * D;
    const float* drow = dO + (static_cast<int64_t>(b) * a.Tq + tq) * a.lddo + h * D;
    float acc = 0.f;
    for (int d = 0; d < D; ++d) acc = fmaf(drow[d], orow[d], acc);
    a.delta[i] = acc;      // [B][H][Tq] is the loop order
  }
}

template <int D>
__global__ void __launch_bounds__(128) f32_attention_dq_kernel(const adp_attention_bwd_args a) {
  pdl_launch_dependents();
  pdl_wait();
  const float* Q = static_cast<const float*>(a.q);
  const float* K = static_cast<const float*>(a.k);
  const float* V = static_cast<const float*>(a.v);
  const float* dO = static_cast<const float*>(a.d_o);
  float* dQ = static_cast<float*>(a.dq);
  F32B_GRID_STRIDE(i, static_cast<int64_t>(a.B) * a.H * a.Tq) {
    const int tq = static_cast<int>(i % a.Tq);
    const int h = static_cast<int>((i / a.Tq) % a.H);
    const int b = static_cast<int>(i / (static_cast<int64_t>(a.Tq) * a.H));
    const float* qr = Q + (static_cast<int64_t>(b) * a.Tq + tq) * a.ldq + h * D;
    const float* dor = dO + (static_cast<int64_t>(b) * a.Tq + tq) * a.lddo + h * D;
    const float lse = a.lse[i], dl = a.delta[i];
    for (int c0 = 0; c0 < D; c0 += kAttCols) {
      float acc[kAttCols];
#pragma unroll
      for (int d = 0; d < kAttCols; ++d) acc[d] = 0.f;
      for (int j = 0; j < a.Tk; ++j) {
        const float* kr = K + (static_cast<int64_t>(b) * a.Tk + j) * a.ldk + h * D;
        const float* vr = V + (static_cast<int64_t>(b) * a.Tk + j) * a.ldv + h * D;
        float s = 0.f, dp = 0.f;
#pragma unroll 8
        for (int d = 0; d < D; ++d) {
          s = fmaf(ld_nc_once(qr + d) * a.scale, kr[d], s);
          dp = fmaf(ld_nc_once(dor + d), vr[d], dp);
        }
        const float ds = expf(s - lse) * (dp - dl);
#pragma unroll
        for (int d = 0; d < kAttCols; ++d) acc[d] = fmaf(ds, kr[c0 + d], acc[d]);
      }
      float* out = dQ + (static_cast<int64_t>(b) * a.Tq + tq) * a.lddq + h * D + c0;
#pragma unroll
      for (int d = 0; d < kAttCols; ++d) out[d] = acc[d] * a.scale;
    }
  }
}

template <int D>
__global__ void __launch_bounds__(128) f32_attention_dkdv_kernel(const adp_attention_bwd_args a) {
  pdl_launch_dependents();
  pdl_wait();
  const float* Q = static_cast<const float*>(a.q);
  const float* K = static_cast<const float*>(a.k);
  const float* V = static_cast<const float*>(a.v);
  const float* dO = static_cast<const float*>(a.d_o);
  float* dK = static_cast<float*>(a.dk);
  float* dV = static_cast<float*>(a.dv);
  F32B_GRID_STRIDE(i, static_cast<int64_t>(a.B) * a.H * a.Tk) {
    const int tk = static_cast<int>(i % a.Tk);
    const int h = static_cast<int>((i / a.Tk) % a.H);
    const int b = static_cast<int>(i / (static_cast<int64_t>(a.Tk) * a.H));
    const float* kr = K + (static_cast<int64_t>(b) * a.Tk + tk) * a.ldk + h * D;
    const float* vr = V + (static_cast<int64_t>(b) * a.Tk + tk) * a.ldv + h * D;
    const int64_t row0 = (static_cast<int64_t>(b) * a.H + h) * a.Tq;
    for (int c0 = 0; c0 < D; c0 += kAttCols) {
      float adk[kAttCols], adv[kAttCols];
#pragma unroll
      for (int d = 0; d < kAttCols; ++d) { adk[d] = 0.f; adv[d] = 0.f; }
      for (int tq = 0; tq < a.Tq; ++tq) {
        const float* qr = Q + (static_cast<int64_t>(b) * a.Tq + tq) * a.ldq + h * D;
        const float* dor = dO + (static_cast<int64_t>(b) * a.Tq + tq) * a.lddo + h * D;
        float s = 0.f, dp = 0.f;
#pragma unroll 8
        for (int d = 0; d < D; ++d) {
          s = fmaf(qr[d] * a.scale, ld_nc_once(kr + d), s);
          dp = fmaf(dor[d], ld_nc_once(vr + d), dp);
        }
        const float p = expf(s - a.lse[row0 + tq]);
        const float ds = p * (dp - a.delta[row0 + tq]);
#pragma unroll
        for (int d = 0; d < kAttCols; ++d) {
          adv[d] = fmaf(p, dor[c0 + d], adv[d]);
          adk[d] = fmaf(ds, qr[c0 + d], adk[d]);
        }
      }
      float* ok = dK + (static_cast<int64_t>(b) * a.Tk + tk) * a.lddk + h * D + c0;
      float* ov = dV + (static_cast<int64_t>(b) * a.Tk + tk) * a.lddv + h * D + c0;
#pragma unroll
      for (int d = 0; d < kAttCols; ++d) { ok[d] = adk[d] * a.scale; ov[d] = adv[d]; }
    }
  }
}

}  // namespace
}  // namespace adp

using namespace adp;

extern "C" int adp_f32_wgrad(const adp_wgrad_args* args, adp_stream_t stream) {
  ADP_CHECK(args && args->g && args->x && args->dw, "adp_f32_wgrad: null pointer");
  const adp_wgrad_args& a = *args;
  ADP_CHECK(a.B > 0 && a.T > 0 && a.n > 0 && a.k > 0, "adp_f32_wgrad: bad sizes");
  ADP_CHECK(a.g_col0 >= 0 && a.x_col0 >= 0 && a.g_col0 + a.n <= a.g_cols && a.x_col0 + a.k <= a.x_cols &&
            a.g_cols <= a.ldg && a.x_cols <= a.ldx && a.k <= a.ldw, "adp_f32_wgrad: columns out of range");
  ADP_CHECK(a.ntaps == 0 || a.ntaps == 1 || a.ntaps == 3, "adp_f32_wgrad: ntaps must be 1 or 3");
  ADP_CHECK(a.ntaps != 3 || a.tap_stride >= (long long)a.n * a.ldw, "adp_f32_wgrad: tap_stride smaller than one dW slab");
  const int64_t n = static_cast<int64_t>(a.ntaps == 3 ? 3 : 1) * a.n * a.k;
  ADP_CUDA(launch_k(f32_wgrad_kernel, dim3(capped_grid(n, 256)), dim3(256), (size_t)0, as_stream(stream), a));
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_f32_gn_silu_bwd(const float* da, const float* x, const double* stats, const float* gamma,
                                   const float* beta, float* dxh, float* dgamma, float* dbeta, double* S, int B,
                                   int T, int C, int groups, float eps, adp_stream_t stream) {
  ADP_CHECK(da && x && stats && gamma && beta && dxh && dgamma && dbeta && S, "adp_f32_gn_silu_bwd: null");
  ADP_CHECK(B > 0 && T > 0 && C > 0 && groups > 0 && C % groups == 0, "adp_f32_gn_silu_bwd: C=%d groups=%d",
            C, groups);
  ADP_CUDA(launch_k(f32_gn_silu_bwd_kernel, dim3(capped_grid(static_cast<int64_t>(B) * C, 256)), dim3(256),
                    (size_t)0, as_stream(stream), da, x, stats, gamma, beta, dxh, dgamma, dbeta, S, B, T, C,
                    groups, eps));
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_f32_gn_bwd_apply(const float* dxh, const float* x, const double* stats, const double* S,
                                    const float* dres, float* dx, float* colsum, int B, int T, int C, int groups,
                                    float eps, adp_stream_t stream) {
  ADP_CHECK(dxh && x && stats && S && dx, "adp_f32_gn_bwd_apply: null");
  ADP_CHECK(B > 0 && T > 0 && C > 0 && groups > 0 && C % groups == 0, "adp_f32_gn_bwd_apply: C=%d groups=%d",
            C, groups);
  ADP_CUDA(launch_k(f32_gn_bwd_apply_kernel, dim3(capped_grid(static_cast<int64_t>(B) * C, 256)), dim3(256),
                    (size_t)0, as_stream(stream), dxh, x, stats, S, dres, dx, colsum, B, T, C, groups, eps));
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_f32_ln_film_bwd(const float* dy, const float* x, const float* scale_shift, int ss_stride,
                                   float* dx, float* dss, int dss_stride, float* colsum, const float* dres, int B,
                                   int T, int C, float eps, adp_stream_t stream) {
  ADP_CHECK(dy && x && dx, "adp_f32_ln_film_bwd: null");
  ADP_CHECK(B > 0 && T > 0 && C > 0, "adp_f32_ln_film_bwd: bad sizes");
  ADP_CHECK(!scale_shift || ss_stride >= 2 * C, "adp_f32_ln_film_bwd: ss_stride %d < 2C", ss_stride);
  ADP_CHECK(!dss || dss_stride >= 2 * C, "adp_f32_ln_film_bwd: dss_stride %d < 2C", dss_stride);
  const int64_t warps = static_cast<int64_t>(B) * ((C + 31) / 32);
  ADP_CUDA(launch_k(f32_ln_film_bwd_kernel, dim3(capped_grid(warps * 32, 256)), dim3(256), (size_t)0,
                    as_stream(stream), dy, x, scale_shift, ss_stride, dx, dss, dss_stride, colsum, dres, B, T, C,
                    eps));
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_f32_colsum(const float* x, const float* gate, int ld_gate, float* out, int B, int T, int C,
                              adp_stream_t stream) {
  ADP_CHECK(x && out && B > 0 && T > 0 && C > 0, "adp_f32_colsum: bad args");
  ADP_CHECK(!gate || ld_gate >= C, "adp_f32_colsum: ld_gate %d < C", ld_gate);
  ADP_CUDA(launch_k(f32_colsum_kernel, dim3(capped_grid(C, 256)), dim3(256), (size_t)0, as_stream(stream), x, gate,
                    ld_gate, out, B, T, C));
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_f32_skip_gate(const float* y, const float* skip, const float* gate, int ld_gate, float* out,
                                 double* stats, int B, int T, int C, int groups, adp_stream_t stream) {
  (void)groups;
  ADP_CHECK(y && skip && gate && out && B > 0 && T > 0 && C > 0 && ld_gate >= C, "adp_f32_skip_gate: bad args");
  ADP_CHECK(!stats, "adp_f32_skip_gate: statistics are a separate adp_f32_gn_stats pass");
  ADP_CUDA(launch_k(f32_skip_gate_kernel, dim3(capped_grid(static_cast<int64_t>(B) * T * C, 256)), dim3(256),
                    (size_t)0, as_stream(stream), y, skip, gate, ld_gate, out, B, T, C));
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_f32_skip_gate_bwd(const float* dout, const float* y, const float* gate, int ld_gate, float* dys,
                                     float* dgate, int ld_dgate, int B, int T, int C, adp_stream_t stream) {
  ADP_CHECK(dout && y && gate && dys && dgate && B > 0 && T > 0 && C > 0 && ld_gate >= C && ld_dgate >= C,
            "adp_f32_skip_gate_bwd: bad args");
  ADP_CUDA(launch_k(f32_skip_gate_bwd_kernel, dim3(capped_grid(static_cast<int64_t>(B) * C, 256)), dim3(256),
                    (size_t)0, as_stream(stream), dout, y, gate, ld_gate, dys, dgate, ld_dgate, B, T, C));
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_f32_cond_bwd(const float* dss, int ld_dss, const float* cond, const float* w, float* dw,
                                float* dbias, float* dcond, int B, int N, int K, adp_stream_t stream) {
  ADP_CHECK(dss && cond && w && dw && dbias, "adp_f32_cond_bwd: null");   // dcond may be NULL
  ADP_CHECK(B >= 1 && N >= 1 && K >= 1 && ld_dss >= N, "adp_f32_cond_bwd: B=%d N=%d K=%d", B, N, K);
  cudaStream_t s = as_stream(stream);
  ADP_CUDA(launch_k(f32_cond_bwd_w_kernel, dim3(capped_grid(static_cast<int64_t>(N) * K, 256)), dim3(256), (size_t)0,
                    s, dss, ld_dss, cond, dw, dbias, B, N, K));
  if (dcond)
    ADP_CUDA(launch_k(f32_cond_bwd_x_kernel, dim3(capped_grid(static_cast<int64_t>(B) * K, 256)), dim3(256),
                      (size_t)0, s, dss, ld_dss, w, dcond, B, N, K));
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_f32_stem_out_bwd(const adp_stem_out_bwd_args* args, adp_stream_t stream) {
  ADP_CHECK(args && args->dv && args->h && args->x && args->w && args->gate && args->dh && args->dw &&
            args->dbias && args->dgate, "adp_f32_stem_out_bwd: null pointer");
  const adp_stem_out_bwd_args& a = *args;
  ADP_CHECK(a.B > 0 && a.T > 0 && a.co >= 1 && a.c0 >= 1 && a.cx >= 1 && a.ca >= 0 && a.f >= 1 && a.T % a.f == 0,
            "adp_f32_stem_out_bwd: bad sizes");
  ADP_CHECK(!a.w_adapt || (a.dw_adapt && a.db_adapt), "adp_f32_stem_out_bwd: adapter grads missing");
  ADP_CHECK(a.w_adapt || a.cx + a.ca == a.co, "adp_f32_stem_out_bwd: identity skip needs cx+ca == co");
  ADP_CHECK((a.ca == 0) == (a.append == nullptr), "adp_f32_stem_out_bwd: append / ca mismatch");
  ADP_CHECK(!a.noise || (a.alpha && a.beta), "adp_f32_stem_out_bwd: noise needs alpha/beta");
  ADP_CHECK(a.ld_dgate >= a.co && (a.ld_gate == 0 || a.ld_gate >= a.co), "adp_f32_stem_out_bwd: gate pitches");
  cudaStream_t s = as_stream(stream);
  const int cin = a.cx + a.ca;
  const int n_items = a.co * a.c0 * 3 + a.co + a.B * a.co + (a.w_adapt ? a.co * cin + a.co : 0);
  ADP_CUDA(launch_k(f32_stem_out_bwd_dh_kernel, dim3(capped_grid(static_cast<int64_t>(a.B) * (a.T / a.f) * a.c0, 256)),
                    dim3(256), (size_t)0, s, a));
  ADP_CUDA(launch_k(f32_stem_out_bwd_param_kernel, dim3(capped_grid(n_items, 256)), dim3(256), (size_t)0, s, a));
  if (a.dxin)
    ADP_CUDA(launch_k(f32_stem_out_bwd_dxin_kernel, dim3(capped_grid(static_cast<int64_t>(a.B) * cin * a.T, 256)),
                      dim3(256), (size_t)0, s, a));
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_f32_stem_in_bwd(const adp_stem_in_bwd_args* args, adp_stream_t stream) {
  ADP_CHECK(args && args->dout && args->x && args->dw && args->dbias, "adp_f32_stem_in_bwd: null pointer");
  const adp_stem_in_bwd_args& a = *args;
  ADP_CHECK(a.B > 0 && a.T > 0 && a.cx >= 1 && a.ca >= 0 && a.c0 >= 1 && a.f >= 1 && a.T % a.f == 0,
            "adp_f32_stem_in_bwd: bad sizes");
  ADP_CHECK((a.ca == 0) == (a.append == nullptr), "adp_f32_stem_in_bwd: append / ca mismatch");
  ADP_CHECK(!a.noise || (a.alpha && a.beta), "adp_f32_stem_in_bwd: noise needs alpha/beta");
  ADP_CHECK(!a.dxin || a.w, "adp_f32_stem_in_bwd: dxin needs the conv weights");
  cudaStream_t s = as_stream(stream);
  const int cin = a.cx + a.ca;
  ADP_CUDA(launch_k(f32_stem_in_bwd_param_kernel, dim3(capped_grid(a.c0 * cin * a.f + a.c0, 256)), dim3(256),
                    (size_t)0, s, a));
  if (a.dxin)
    ADP_CUDA(launch_k(f32_stem_in_bwd_dxin_kernel, dim3(capped_grid(static_cast<int64_t>(a.B) * cin * a.T, 256)),
                      dim3(256), (size_t)0, s, a));
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_f32_attention_bwd(const adp_attention_bwd_args* args, int head_dim, adp_stream_t stream) {
  ADP_CHECK(head_dim == 32 || head_dim == 64 || head_dim == 128,
            "adp_f32_attention_bwd: head_dim %d not supported (32, 64 or 128)", head_dim);
  ADP_CHECK(args != nullptr, "adp_f32_attention_bwd: null args");
  const adp_attention_bwd_args& a = *args;
  ADP_CHECK(a.q && a.k && a.v && a.o && a.d_o && a.lse && a.delta && a.dq && a.dk && a.dv,
            "adp_f32_attention_bwd: null pointer");
  ADP_CHECK(a.B > 0 && a.H > 0 && a.Tq > 0 && a.Tk > 0 && a.scale > 0.f, "adp_f32_attention_bwd: bad sizes");
  const int64_t w = static_cast<int64_t>(a.H) * head_dim;
  ADP_CHECK(a.ldq >= w && a.ldk >= w && a.ldv >= w && a.ldo >= w && a.lddo >= w && a.lddq >= w && a.lddk >= w &&
            a.lddv >= w, "adp_f32_attention_bwd: row pitches must be >= heads*head_dim (%d*%d)", a.H, head_dim);
  cudaStream_t s = as_stream(stream);
  const int64_t nq = static_cast<int64_t>(a.B) * a.H * a.Tq, nk = static_cast<int64_t>(a.B) * a.H * a.Tk;
  ADP_CUDA(launch_k(f32_attention_delta_kernel, dim3(capped_grid(nq, 256)), dim3(256), (size_t)0, s, a, head_dim));
  auto dq = head_dim == 32 ? f32_attention_dq_kernel<32>
            : head_dim == 128 ? f32_attention_dq_kernel<128> : f32_attention_dq_kernel<64>;
  auto dkdv = head_dim == 32 ? f32_attention_dkdv_kernel<32>
              : head_dim == 128 ? f32_attention_dkdv_kernel<128> : f32_attention_dkdv_kernel<64>;
  ADP_CUDA(launch_k(dq, dim3(capped_grid(nq, 128)), dim3(128), (size_t)0, s, a));
  ADP_CUDA(launch_k(dkdv, dim3(capped_grid(nk, 128)), dim3(128), (size_t)0, s, a));
  ADP_LAUNCH_CHECK();
  return 0;
}
