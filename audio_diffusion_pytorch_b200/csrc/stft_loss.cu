// Multi-resolution STFT loss (losses.MultiResolutionSTFTLoss), fp32 on CUDA cores, one resolution
// (n_fft N, hop, Hann window of length W centred in N) per call:
//   adp_stft_loss_fwd   frames of x and y (reflect pad N/2) through the mixed-radix FFT (fft.cuh),
//                       fp64 partial sums per (row, frame group), then a one-CTA fixed-order
//                       reduction to the per-row norms and the resolution's loss term
//   adp_stft_loss_bwd   recompute both spectra, form dL/dX, run the adjoint of the one-sided
//                       transform (one more FFT per frame), window, store the frame gradients;
//                       then gather them onto dx (overlap-add + reflect-pad fold)
// No atomics: the loss and dx are bitwise reproducible.
#include <cuda_bf16.h>

#include "common.cuh"
#include "fft.cuh"
#include "ptx.cuh"

namespace adp {

constexpr int kLossFrames = 8;        // frames per CTA (forward and backward)
constexpr int kLossThreads = 256;

__device__ __forceinline__ float ld(const float* p, size_t i) { return p[i]; }
__device__ __forceinline__ float ld(const __nv_bfloat16* p, size_t i) { return __bfloat162float(p[i]); }

__device__ __forceinline__ float sgn(float v) { return static_cast<float>((v > 0.f) - (v < 0.f)); }

// Frame f of row s, windowed, as a complex signal with zero imaginary part in buf (N points; the
// window is zero outside its W taps, so those samples are not read).  x and y go through separate
// transforms: sharing one (z = x + i y) would give X an absolute error on the scale of |Y|, which
// the log-magnitude gradient's 1 / Xmag amplifies at the small bins of nearly silent frames.
template <typename T>
__device__ __forceinline__ void load_frame(float2* buf, const T* __restrict__ s, const float* __restrict__ window,
                                           int f, int N, int hop, int pad, int t) {
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    const float w = window[n];
    float v = 0.f;
    if (w != 0.f) v = w * ld(s, reflect_index(f * hop + n - pad, t));
    buf[n] = make_float2(v, 0.f);
  }
}

// ------------------------------------------------------------------------------ forward
// One CTA per (row, group of kLossFrames frames).  Shared memory: two [N] complex buffers, the [N]
// twiddles and the frame's X [N/2 + 1] while Y is transformed (28 N + 8 bytes: 229,384 at
// N = 8192) plus the block reduction.  Each thread accumulates its bins in fp64;
// the CTA writes partials[row][group] = {sum (Xmag - Ymag)^2, sum Ymag^2, sum |log Xmag - log Ymag|,
// sum |Xmag - Ymag|}, reduced in a fixed order.
template <typename T>
__global__ void __launch_bounds__(kLossThreads)
stft_loss_fwd_kernel(const T* __restrict__ x, const T* __restrict__ y, const float* __restrict__ window,
                     double* __restrict__ partials, int t, int N, unsigned long long plan, int hop,
                     int frames, float eps) {
  extern __shared__ __align__(16) float smem[];
  float2* buf0 = reinterpret_cast<float2*>(smem);
  float2* buf1 = buf0 + N;
  float2* tw = buf1 + N;
  float2* xs = tw + N;                                        // [N/2 + 1] X of the frame
  double* red = reinterpret_cast<double*>(xs + N / 2 + 2);    // [warps][4]
  pdl_launch_dependents();
  fft_twiddles(tw, N);
  const float2* z = (fft_stages(plan) & 1) ? buf1 : buf0;
  pdl_wait();
  const int row = blockIdx.y, f0 = blockIdx.x * kLossFrames, bins = N / 2 + 1, pad = N / 2;
  const T* xr = x + static_cast<size_t>(row) * t;
  const T* yr = y + static_cast<size_t>(row) * t;
  double s_d2 = 0.0, s_y2 = 0.0, s_log = 0.0, s_lin = 0.0;
  const int f_end = min(f0 + kLossFrames, frames);
  for (int f = f0; f < f_end; ++f) {
    __syncthreads();
    load_frame(buf0, xr, window, f, N, hop, pad, t);
    __syncthreads();
    fft_forward(buf0, buf1, tw, N, plan);
    for (int k = threadIdx.x; k < bins; k += blockDim.x) xs[k] = z[k];
    __syncthreads();
    load_frame(buf0, yr, window, f, N, hop, pad, t);
    __syncthreads();
    fft_forward(buf0, buf1, tw, N, plan);
    for (int k = threadIdx.x; k < bins; k += blockDim.x) {
      const float2 X = xs[k], Y = z[k];
      const float xm = sqrtf(fmaxf(X.x * X.x + X.y * X.y, eps));
      const float ym = sqrtf(fmaxf(Y.x * Y.x + Y.y * Y.y, eps));
      const float d = xm - ym;
      s_d2 += static_cast<double>(d) * d;
      s_y2 += static_cast<double>(ym) * ym;
      s_log += fabsf(logf(xm) - logf(ym));
      s_lin += fabsf(d);
    }
  }
  double v[4] = {s_d2, s_y2, s_log, s_lin};
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[q] += __shfl_down_sync(0xffffffffu, v[q], o);
  }
  if (lane == 0) {
#pragma unroll
    for (int q = 0; q < 4; ++q) red[warp * 4 + q] = v[q];
  }
  __syncthreads();
  if (threadIdx.x < 4) {
    double s = 0.0;
    for (int w = 0; w < kLossThreads / 32; ++w) s += red[w * 4 + threadIdx.x];
    partials[(static_cast<size_t>(row) * gridDim.x + blockIdx.x) * 4 + threadIdx.x] = s;
  }
}

// One CTA: per row, the groups' partials in order -> row_stats[row] = {||Y - X||, ||Y||}; then
// sc = mean_rows ||Y - X|| / ||Y||, log and lin means, and acc = (accumulate ? acc : 0) +
// scale * (w_sc sc + w_log log_mag + w_lin lin_mag), loss = (float) acc.
__global__ void __launch_bounds__(kLossThreads)
stft_loss_reduce_kernel(const double* __restrict__ partials, double* __restrict__ row_stats,
                        double* __restrict__ acc, float* __restrict__ loss, int rows, int groups,
                        double inv_count, float w_sc, float w_log, float w_lin, float scale, int accumulate) {
  __shared__ double red[kLossThreads / 32][3];
  pdl_launch_dependents();
  pdl_wait();
  double v[3] = {0.0, 0.0, 0.0};
  for (int r = threadIdx.x; r < rows; r += blockDim.x) {
    double s[4] = {0.0, 0.0, 0.0, 0.0};
    const double* p = partials + static_cast<size_t>(r) * groups * 4;
    for (int g = 0; g < groups; ++g) {
#pragma unroll
      for (int q = 0; q < 4; ++q) s[q] += p[g * 4 + q];
    }
    const double dn = sqrt(s[0]), yn = sqrt(s[1]);
    row_stats[2 * r] = dn;
    row_stats[2 * r + 1] = yn;
    v[0] += dn / yn;
    v[1] += s[2];
    v[2] += s[3];
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int q = 0; q < 3; ++q) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[q] += __shfl_down_sync(0xffffffffu, v[q], o);
  }
  if (lane == 0) {
#pragma unroll
    for (int q = 0; q < 3; ++q) red[warp][q] = v[q];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double s[3] = {0.0, 0.0, 0.0};
    for (int w = 0; w < kLossThreads / 32; ++w) {
#pragma unroll
      for (int q = 0; q < 3; ++q) s[q] += red[w][q];
    }
    const double l = static_cast<double>(w_sc) * s[0] / rows + static_cast<double>(w_log) * s[1] * inv_count +
                     static_cast<double>(w_lin) * s[2] * inv_count;
    const double total = (accumulate ? acc[0] : 0.0) + static_cast<double>(scale) * l;
    acc[0] = total;
    loss[0] = static_cast<float>(total);
  }
}

// ----------------------------------------------------------------------------- backward
// One CTA per (row, group of kLossFrames frames), two frames at a time.  For each frame the
// spectra X, Y are recomputed as in the forward, and
//   g = gout (a_sc (Xmag - Ymag) + c_log sign(log Xmag - log Ymag) / Xmag + c_lin sign(Xmag - Ymag)),
//   G = g X / Xmag where |X|^2 >= eps, else 0 (the clamp's gradient mask),
// with a_sc = c_sc / (||Y - X|| ||Y||) of the row (0 when ||Y - X|| = 0).  The frame gradient
// Re sum_(k <= N/2) G_k exp(+2 pi i k n / N) is the inverse transform of the Hermitian extension
// H (H_0 = Re G_0, H_(N/2) = Re G_(N/2), H_k = G_k / 2, H_(N-k) = conj(G_k) / 2), taken through the
// forward FFT of conj(H), whose result is real.  The windowed gradients of the W window taps go to
// frame_grad[row][frame][W].  Shared memory as in the forward: 28 N + 8 bytes.
template <typename T>
__global__ void __launch_bounds__(kLossThreads)
stft_loss_bwd_kernel(const T* __restrict__ x, const T* __restrict__ y, const float* __restrict__ window,
                     const double* __restrict__ row_stats, const float* __restrict__ grad_out,
                     float* __restrict__ frame_grad, int t, int N, unsigned long long plan, int hop,
                     int frames, int off, int W, float eps, float c_sc, float c_log, float c_lin) {
  extern __shared__ __align__(16) float smem[];
  float2* buf0 = reinterpret_cast<float2*>(smem);
  float2* buf1 = buf0 + N;
  float2* tw = buf1 + N;
  float2* xs = tw + N;                                        // [N/2 + 1] X of the frame
  pdl_launch_dependents();
  fft_twiddles(tw, N);
  const bool odd = fft_stages(plan) & 1;
  float2* spec = odd ? buf1 : buf0;                           // a frame's spectrum
  float2* free_buf = odd ? buf0 : buf1;                       // conj(H); its transform lands in buf1
  pdl_wait();
  const int row = blockIdx.y, f0 = blockIdx.x * kLossFrames, bins = N / 2 + 1, pad = N / 2;
  const T* xr = x + static_cast<size_t>(row) * t;
  const T* yr = y + static_cast<size_t>(row) * t;
  const double dn = row_stats[2 * row], yn = row_stats[2 * row + 1];
  const float gout = grad_out[0];
  const float a_sc = dn > 0.0 ? static_cast<float>(static_cast<double>(c_sc) / (dn * yn)) : 0.f;
  for (int f = f0; f < min(f0 + kLossFrames, frames); ++f) {
    __syncthreads();
    load_frame(buf0, xr, window, f, N, hop, pad, t);
    __syncthreads();
    fft_forward(buf0, buf1, tw, N, plan);
    for (int k = threadIdx.x; k < bins; k += blockDim.x) xs[k] = spec[k];
    __syncthreads();
    load_frame(buf0, yr, window, f, N, hop, pad, t);
    __syncthreads();
    fft_forward(buf0, buf1, tw, N, plan);
    for (int k = threadIdx.x; k < bins; k += blockDim.x) {
      const float2 X = xs[k], Y = spec[k];
      float2 h = make_float2(0.f, 0.f);
      const float p2 = X.x * X.x + X.y * X.y;
      if (p2 >= eps) {
        const float xm = sqrtf(p2);
        const float ym = sqrtf(fmaxf(Y.x * Y.x + Y.y * Y.y, eps));
        const float d = xm - ym;
        float g = a_sc * d + c_log * sgn(logf(xm) - logf(ym)) / xm + c_lin * sgn(d);
        g = g * gout / xm;
        h = (k == 0 || 2 * k == N) ? make_float2(g * X.x, 0.f) : make_float2(0.5f * g * X.x, 0.5f * g * X.y);
      }
      free_buf[k] = make_float2(h.x, -h.y);                   // conj(H_k)
      if (k != 0 && 2 * k != N) free_buf[N - k] = h;          // conj(H_(N-k)) = H_k
    }
    __syncthreads();
    fft_forward(free_buf, spec, tw, N, plan);
    float* fg = frame_grad + (static_cast<size_t>(row) * frames + f) * W;
    for (int n = threadIdx.x; n < W; n += blockDim.x) fg[n] = window[off + n] * buf1[off + n].x;
  }
}

// dx[row, j] (+)= sum over the padded positions p that reflect onto j (p = j + pad, and pad - j,
// pad + 2 (t - 1) - j where the pad mirrors j) of sum over frames f covering p of
// frame_grad[row][f][p - f hop - off], frames in increasing order.  dx_bf16 (optional) receives
// the same values rounded.
__global__ void __launch_bounds__(kLossThreads)
stft_loss_ola_kernel(const float* __restrict__ frame_grad, float* __restrict__ dx,
                     __nv_bfloat16* __restrict__ dx_bf16, int t, int frames, int hop, int off, int W,
                     int pad, int accumulate) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.y;
  const float* fg = frame_grad + static_cast<size_t>(row) * frames * W;
  auto tap = [&](int p) {
    const int q = p - off;                                     // position in the frames' W taps
    float s = 0.f;
    if (q < 0) return s;
    int f_lo = q - W + 1 <= 0 ? 0 : (q - W + hop) / hop;         // ceil((q - W + 1) / hop)
    const int f_hi = min(q / hop, frames - 1);
    for (int f = f_lo; f <= f_hi; ++f) s += fg[static_cast<size_t>(f) * W + (q - f * hop)];
    return s;
  };
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < t; j += gridDim.x * blockDim.x) {
    float s = tap(j + pad);
    if (j >= 1 && j <= pad) s += tap(pad - j);
    if (j >= t - 1 - pad && j <= t - 2) s += tap(pad + 2 * (t - 1) - j);
    const size_t i = static_cast<size_t>(row) * t + j;
    if (accumulate) s += dx[i];
    dx[i] = s;
    if (dx_bf16) dx_bf16[i] = __float2bfloat16_rn(s);
  }
}

// Shared size checks of both entry points; returns the FFT plan through *plan.
static int stft_loss_check(const char* what, int rows, int t, int n_fft, int hop, int win_length,
                           int frames, unsigned long long* plan) {
  *plan = n_fft >= 32 && n_fft <= kFftMaxN ? fft_plan(n_fft) : 0;
  ADP_CHECK(*plan != 0, "%s: fft_size=%d must have prime factors 2, 3, 5, 7 only and lie in [32, %d]", what,
            n_fft, kFftMaxN);
  ADP_CHECK(win_length >= 1 && win_length <= n_fft, "%s: win_length=%d must lie in [1, fft_size=%d]", what,
            win_length, n_fft);
  ADP_CHECK(hop >= 1, "%s: hop_size=%d must be at least 1", what, hop);
  ADP_CHECK(t > n_fft / 2, "%s: the signal (%d samples) must be longer than fft_size // 2 = %d (reflect pad)",
            what, t, n_fft / 2);
  ADP_CHECK(rows > 0 && rows <= 65535, "%s: rows=%d must lie in [1, 65535]", what, rows);
  ADP_CHECK(frames == 1 + (t + 2 * (n_fft / 2) - n_fft) / hop, "%s: frames=%d does not match the signal", what,
            frames);
  return 0;
}

}  // namespace adp

using namespace adp;

extern "C" int adp_stft_loss_fwd(const void* x, const void* y, const float* window, double* partials,
                                 double* row_stats, double* acc, float* loss, int rows, int t, int n_fft,
                                 int hop, int win_length, int frames, int in_bf16, float eps, float w_sc,
                                 float w_log_mag, float w_lin_mag, float scale, int accumulate,
                                 adp_stream_t stream) {
  ADP_CHECK(x && y && window && partials && row_stats && acc && loss, "adp_stft_loss_fwd: null pointer");
  unsigned long long plan = 0;
  if (int rc = stft_loss_check("adp_stft_loss_fwd", rows, t, n_fft, hop, win_length, frames, &plan)) return rc;
  const int groups = (frames + kLossFrames - 1) / kLossFrames;
  const size_t smem = (static_cast<size_t>(n_fft) * 3 + n_fft / 2 + 2) * sizeof(float2) +
                      (kLossThreads / 32) * 4 * sizeof(double);
  const dim3 grid(groups, rows);
  if (in_bf16) {
    static SmemAttrCache cache;
    ADP_CUDA(ensure_dyn_smem(stft_loss_fwd_kernel<__nv_bfloat16>, smem, cache));
    ADP_CUDA(launch_k(stft_loss_fwd_kernel<__nv_bfloat16>, grid, dim3(kLossThreads), smem, as_stream(stream),
                      static_cast<const __nv_bfloat16*>(x), static_cast<const __nv_bfloat16*>(y), window,
                      partials, t, n_fft, plan, hop, frames, eps));
  } else {
    static SmemAttrCache cache;
    ADP_CUDA(ensure_dyn_smem(stft_loss_fwd_kernel<float>, smem, cache));
    ADP_CUDA(launch_k(stft_loss_fwd_kernel<float>, grid, dim3(kLossThreads), smem, as_stream(stream),
                      static_cast<const float*>(x), static_cast<const float*>(y), window, partials, t, n_fft,
                      plan, hop, frames, eps));
  }
  ADP_LAUNCH_CHECK();
  const double count = static_cast<double>(rows) * frames * (n_fft / 2 + 1);
  ADP_CUDA(launch_k(stft_loss_reduce_kernel, dim3(1), dim3(kLossThreads), (size_t)0, as_stream(stream),
                    static_cast<const double*>(partials), row_stats, acc, loss, rows, groups, 1.0 / count, w_sc,
                    w_log_mag, w_lin_mag, scale, accumulate));
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_stft_loss_bwd(const void* x, const void* y, const float* window, const double* row_stats,
                                 const float* grad_out, float* frame_grad, float* dx, void* dx_bf16, int rows,
                                 int t, int n_fft, int hop, int win_length, int frames, int in_bf16, float eps,
                                 float w_sc, float w_log_mag, float w_lin_mag, float scale, int accumulate,
                                 adp_stream_t stream) {
  ADP_CHECK(x && y && window && row_stats && grad_out && frame_grad && dx, "adp_stft_loss_bwd: null pointer");
  unsigned long long plan = 0;
  if (int rc = stft_loss_check("adp_stft_loss_bwd", rows, t, n_fft, hop, win_length, frames, &plan)) return rc;
  const int groups = (frames + kLossFrames - 1) / kLossFrames;
  const int bins = n_fft / 2 + 1, off = (n_fft - win_length) / 2;
  const double count = static_cast<double>(rows) * frames * bins;
  const float c_sc = static_cast<float>(static_cast<double>(scale) * w_sc / rows);
  const float c_log = static_cast<float>(static_cast<double>(scale) * w_log_mag / count);
  const float c_lin = static_cast<float>(static_cast<double>(scale) * w_lin_mag / count);
  const size_t smem = (static_cast<size_t>(n_fft) * 3 + bins) * sizeof(float2);
  const dim3 grid(groups, rows);
  if (in_bf16) {
    static SmemAttrCache cache;
    ADP_CUDA(ensure_dyn_smem(stft_loss_bwd_kernel<__nv_bfloat16>, smem, cache));
    ADP_CUDA(launch_k(stft_loss_bwd_kernel<__nv_bfloat16>, grid, dim3(kLossThreads), smem, as_stream(stream),
                      static_cast<const __nv_bfloat16*>(x), static_cast<const __nv_bfloat16*>(y), window,
                      row_stats, grad_out, frame_grad, t, n_fft, plan, hop, frames, off, win_length, eps, c_sc,
                      c_log, c_lin));
  } else {
    static SmemAttrCache cache;
    ADP_CUDA(ensure_dyn_smem(stft_loss_bwd_kernel<float>, smem, cache));
    ADP_CUDA(launch_k(stft_loss_bwd_kernel<float>, grid, dim3(kLossThreads), smem, as_stream(stream),
                      static_cast<const float*>(x), static_cast<const float*>(y), window, row_stats, grad_out,
                      frame_grad, t, n_fft, plan, hop, frames, off, win_length, eps, c_sc, c_log, c_lin));
  }
  ADP_LAUNCH_CHECK();
  const int gx = capped_grid(t, kLossThreads);
  ADP_CUDA(launch_k(stft_loss_ola_kernel, dim3(gx, rows), dim3(kLossThreads), (size_t)0, as_stream(stream),
                    static_cast<const float*>(frame_grad), dx, static_cast<__nv_bfloat16*>(dx_bf16), t, frames,
                    hop, off, win_length, n_fft / 2, accumulate));
  ADP_LAUNCH_CHECK();
  return 0;
}
