// Mixed-radix Stockham FFT in shared memory, shared by the mel front-end (frontend.cu) and the
// multi-resolution STFT loss (stft_loss.cu).  N = product of the plan's radices (4s, then at most
// one 2, then 3s, 5s, 7s); each stage reads one buffer in natural order and writes the other, so
// no digit reversal is needed.  The twiddle table holds exp(-2 pi i k / N) for k < N.
#pragma once
#include <cuda_runtime.h>

namespace adp {

constexpr int kFftMaxN = 8192;

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }

// cos and sin of 2 pi j / R for R in {3, 5, 7} and 1 <= j <= R / 2
__host__ __device__ constexpr float dft_cos(int R, int j) {
  return R == 3 ? -0.5f
       : R == 5 ? (j == 1 ? 0.30901699437494745f : -0.80901699437494745f)
       : (j == 1 ? 0.62348980185873353f : j == 2 ? -0.22252093395631440f : -0.90096886790241913f);
}
__host__ __device__ constexpr float dft_sin(int R, int j) {
  return R == 3 ? 0.86602540378443865f
       : R == 5 ? (j == 1 ? 0.95105651629515357f : 0.58778525229247313f)
       : (j == 1 ? 0.78183148246802981f : j == 2 ? 0.97492791218182361f : 0.43388373911755812f);
}

// In-register forward DFT of R points, X_k = sum_n v_n exp(-2 pi i k n / R).  Odd R pairs
// v_m with v_(R-m): X_k = A_k - i B_k, X_(R-k) = A_k + i B_k with A_k = v_0 + sum_m (v_m + v_(R-m))
// cos(2 pi k m / R) and B_k = sum_m (v_m - v_(R-m)) sin(2 pi k m / R).
template <int R>
__device__ __forceinline__ void dft(float2 (&v)[R]) {
  constexpr int H = R / 2;
  float2 s[H + 1], d[H + 1];
  const float2 x0 = v[0];
  float2 sum = x0;
#pragma unroll
  for (int m = 1; m <= H; ++m) {
    s[m] = cadd(v[m], v[R - m]);
    d[m] = csub(v[m], v[R - m]);
    sum = cadd(sum, s[m]);
  }
  v[0] = sum;
#pragma unroll
  for (int k = 1; k <= H; ++k) {
    float2 a = x0, b = make_float2(0.f, 0.f);
#pragma unroll
    for (int m = 1; m <= H; ++m) {
      const int j = (k * m) % R;
      const float c = j <= H ? dft_cos(R, j) : dft_cos(R, R - j);
      const float sn = j <= H ? dft_sin(R, j) : -dft_sin(R, R - j);
      a = make_float2(fmaf(s[m].x, c, a.x), fmaf(s[m].y, c, a.y));
      b = make_float2(fmaf(d[m].x, sn, b.x), fmaf(d[m].y, sn, b.y));
    }
    v[k] = make_float2(a.x + b.y, a.y - b.x);
    v[R - k] = make_float2(a.x - b.y, a.y + b.x);
  }
}
template <>
__device__ __forceinline__ void dft<2>(float2 (&v)[2]) {
  const float2 a = v[0], b = v[1];
  v[0] = cadd(a, b);
  v[1] = csub(a, b);
}
template <>
__device__ __forceinline__ void dft<4>(float2 (&v)[4]) {
  const float2 t0 = cadd(v[0], v[2]), t1 = csub(v[0], v[2]), t2 = cadd(v[1], v[3]), t3 = csub(v[1], v[3]);
  const float2 mt3 = make_float2(t3.y, -t3.x);                       // -i t3
  v[0] = cadd(t0, t2);
  v[1] = cadd(t1, mt3);
  v[2] = csub(t0, t2);
  v[3] = csub(t1, mt3);
}

// One Stockham radix-R stage after sub-transforms of length Ns: butterfly j (k = j mod Ns) reads
// src[j + r N/R], twiddles input r by exp(-2 pi i k r / (Ns R)) and writes dst[(j - k) R + k + r Ns].
template <int R>
__device__ __forceinline__ void fft_stage(const float2* __restrict__ src, float2* __restrict__ dst,
                                          const float2* __restrict__ tw, int N, int Ns) {
  const int m = N / R, step = N / (Ns * R);
  for (int j = threadIdx.x; j < m; j += blockDim.x) {
    const int k = j % Ns;
    float2 v[R];
#pragma unroll
    for (int r = 0; r < R; ++r) v[r] = src[j + r * m];
    if (Ns > 1) {
#pragma unroll
      for (int r = 1; r < R; ++r) v[r] = cmul(v[r], tw[k * r * step]);
    }
    dft<R>(v);
    float2* d = dst + (j - k) * R + k;
#pragma unroll
    for (int r = 0; r < R; ++r) d[r * Ns] = v[r];
  }
}

// The twiddle table of an N-point transform: tw[k] = exp(-2 pi i k / N), k < N.
__device__ __forceinline__ void fft_twiddles(float2* tw, int N) {
  for (int k = threadIdx.x; k < N; k += blockDim.x) {
    float s, c;
    sincospif(-2.f * static_cast<float>(k) / static_cast<float>(N), &s, &c);
    tw[k] = make_float2(c, s);
  }
}

// Number of stages of a plan; the spectrum of a transform that starts in buffer a ends in buffer b
// when it is odd.
__device__ __forceinline__ int fft_stages(unsigned long long plan) {
  int stages = 0;
  for (unsigned long long p = plan; p; p >>= 4) ++stages;
  return stages;
}

// The whole forward transform of src (N points, natural order), ping-ponging with dst; the result
// lands in src after an even number of stages and in dst after an odd one.  Ends with a barrier.
__device__ __forceinline__ void fft_forward(float2* src, float2* dst, const float2* __restrict__ tw,
                                            int N, unsigned long long plan) {
  int Ns = 1;
  for (unsigned long long p = plan; p; p >>= 4) {
    const int R = static_cast<int>(p & 15);
    switch (R) {
      case 4: fft_stage<4>(src, dst, tw, N, Ns); break;
      case 2: fft_stage<2>(src, dst, tw, N, Ns); break;
      case 3: fft_stage<3>(src, dst, tw, N, Ns); break;
      case 5: fft_stage<5>(src, dst, tw, N, Ns); break;
      default: fft_stage<7>(src, dst, tw, N, Ns); break;
    }
    __syncthreads();
    float2* tmp = src;
    src = dst;
    dst = tmp;
    Ns *= R;
  }
}

// F.pad(mode="reflect") index: the edge sample is not repeated (|j| < len assumed)
__device__ __forceinline__ int reflect_index(int j, int len) {
  return j < 0 ? -j : (j >= len ? 2 * (len - 1) - j : j);
}

// Radices of n, 4 bits per stage with the first stage lowest: 4s, at most one 2, then 3s, 5s, 7s.
// 0 when n has a prime factor above 7.
static inline unsigned long long fft_plan(int n) {
  unsigned long long plan = 0;
  int shift = 0;
  auto take = [&](int r) {
    while (n % r == 0 && n > 1 && shift < 64) {
      plan |= static_cast<unsigned long long>(r) << shift;
      shift += 4;
      n /= r;
      if (r == 2) break;
    }
  };
  take(4);
  take(2);
  take(3);
  take(5);
  take(7);
  return n == 1 ? plan : 0;
}

}  // namespace adp
