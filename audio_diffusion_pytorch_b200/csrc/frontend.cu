// Conditioning front-ends of the model wrappers (SURVEY.md 8f-2), fp32 on CUDA cores; they run
// once per call, outside the step loop, on waveform-rate data (HBM-bound, a few MB):
//   adp_resample / _adjoint   polyphase windowed-sinc rate change (reference utils.py:82-117,
//                             DiffusionUpsampler.reupsample / .sample)
//   adp_mel_spectrogram       reflect-pad framing (+ stft's center pad) + window + mixed-radix
//                             FFT in shared memory + magnitude + triangular mel filters (+ log),
//                             reference components.py:188-236 (DiffusionVocoder.forward)
//   adp_to_flat / _bwd        ConvTranspose1d(mel -> 1 channel, bias-free), reference
//                             models.py:194-201, with the gradients of its weight and input
#include "common.cuh"
#include "fft.cuh"
#include "ptx.cuh"

namespace adp {

// --------------------------------------------------------------------------- resample
// y[r, i*fo + p] = sum_k xpad[r, i*fi + k] * bank[p, k],  xpad[j] = x[j - half] (0 outside [0, t)).
// One thread per output sample; the bank (fo x taps floats, <= a few KB) sits in shared memory.
__global__ void __launch_bounds__(256)
resample_kernel(const float* __restrict__ x, const float* __restrict__ bank, float* __restrict__ y,
                int t, int t_out, int fi, int fo, int taps, int half) {
  extern __shared__ float s_bank[];
  pdl_launch_dependents();
  for (int i = threadIdx.x; i < fo * taps; i += blockDim.x) s_bank[i] = bank[i];
  pdl_wait();
  __syncthreads();
  const float* xr = x + static_cast<size_t>(blockIdx.y) * t;
  float* yr = y + static_cast<size_t>(blockIdx.y) * t_out;
  for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < t_out; o += gridDim.x * blockDim.x) {
    const int frame = o / fo, p = o - frame * fo;
    const int j0 = frame * fi - half;
    const float* bk = s_bank + p * taps;
    float acc = 0.f;
    for (int k = 0; k < taps; ++k) {
      const int j = j0 + k;
      if (j >= 0 && j < t) acc = fmaf(xr[j], bk[k], acc);
    }
    yr[o] = acc;
  }
}

// dx[r, j] = sum over (frame, p, k) with frame*fi + k - half == j of dy[r, frame*fo + p] * bank[p, k]
__global__ void __launch_bounds__(256)
resample_adjoint_kernel(const float* __restrict__ dy, const float* __restrict__ bank,
                        float* __restrict__ dx, int t, int t_out, int fi, int fo, int taps, int half) {
  extern __shared__ float s_bank[];
  pdl_launch_dependents();
  for (int i = threadIdx.x; i < fo * taps; i += blockDim.x) s_bank[i] = bank[i];
  pdl_wait();
  __syncthreads();
  const float* dyr = dy + static_cast<size_t>(blockIdx.y) * t_out;
  float* dxr = dx + static_cast<size_t>(blockIdx.y) * t;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < t; j += gridDim.x * blockDim.x) {
    float acc = 0.f;
    // k = j + half - frame*fi in [0, taps)
    const int num = j + half;
    int f_lo = (num - taps + fi) / fi;        // smallest frame with k <= taps-1  (ceil((num-taps+1)/fi))
    if (num - taps + 1 <= 0) f_lo = 0;
    const int f_hi = num / fi;                // largest frame with k >= 0
    for (int frame = f_lo; frame <= f_hi; ++frame) {
      const int k = num - frame * fi;
      if (k < 0 || k >= taps) continue;
      for (int p = 0; p < fo; ++p) {
        const int o = frame * fo + p;
        if (o < t_out) acc = fmaf(dyr[o], s_bank[p * taps + k], acc);
      }
    }
    dxr[j] = acc;
  }
}

// --------------------------------------------------------------------------- mel spectrogram
// One CTA (256 threads) per (row, group of kMelFrames frames).  Two real frames ride through one
// complex FFT (z = a + i b; A[k] = (Z[k] + conj Z[N-k]) / 2, B[k] = (Z[k] - conj Z[N-k]) / 2i,
// N-k taken mod N).  The FFT is a mixed-radix Stockham transform in shared memory: N = product
// of the plan's radices (4s, then at most one 2, then 3s, 5s, 7s), each stage reads one buffer in
// natural order and writes the other, so no digit reversal is needed; the twiddle table holds
// exp(-2 pi i k / N) for k < N.  Shared memory: two [N] complex buffers, the [N] twiddles and the
// [n_mels][kMelFrames] accumulators (24 N + 32 n_mels bytes: 208 KB at N = 8192 and 512 mels);
// the magnitudes [2][N/2 + 1] reuse the buffer the last stage read.  Each mel filter is a
// triangle over a contiguous bin range [lo, hi) (host-computed from the filterbank's non-zeros):
// a thread owns one (mel, frame) output.
constexpr int kMelFrames = 8;
constexpr int kMelMaxN = kFftMaxN;

__global__ void __launch_bounds__(256)
mel_spectrogram_kernel(const float* __restrict__ wave, const float* __restrict__ window,
                       const float* __restrict__ fb, const int* __restrict__ band,
                       float* __restrict__ mel, int t, int n_fft, unsigned long long plan, int hop,
                       int pad, int center_pad, int frames, int n_mels, int apply_log) {
  extern __shared__ __align__(16) float smem[];
  const int N = n_fft, bins = N / 2 + 1;
  float2* buf0 = reinterpret_cast<float2*>(smem);              // [N] frames in, even stages' input
  float2* buf1 = buf0 + N;                                     // [N]
  float2* tw = buf1 + N;                                       // [N]
  float* acc = reinterpret_cast<float*>(tw + N);               // [n_mels][kMelFrames]
  pdl_launch_dependents();
  for (int k = threadIdx.x; k < N; k += blockDim.x) {
    float s, c;
    sincospif(-2.f * static_cast<float>(k) / static_cast<float>(N), &s, &c);
    tw[k] = make_float2(c, s);
  }
  int stages = 0;
  for (unsigned long long p = plan; p; p >>= 4) ++stages;
  const float2* z = (stages & 1) ? buf1 : buf0;                // the spectrum after the last stage
  float* mag = reinterpret_cast<float*>((stages & 1) ? buf0 : buf1);   // [2][bins]
  pdl_wait();
  const int row = blockIdx.y;
  const int f0 = blockIdx.x * kMelFrames;
  const int t_pad = t + 2 * pad;
  const float* wr = wave + static_cast<size_t>(row) * t;
  for (int pair = 0; pair < kMelFrames / 2; ++pair) {
    const int fa = f0 + 2 * pair, fbm = fa + 1;
    __syncthreads();
    // windowed frames of the row reflect-padded by pad, then the result reflect-padded by
    // center_pad (torch.stft's center=True after the module's own pad)
    for (int n = threadIdx.x; n < N; n += blockDim.x) {
      float va = 0.f, vb = 0.f;
      const float w = window[n];
      if (fa < frames) va = wr[reflect_index(reflect_index(fa * hop + n - center_pad, t_pad) - pad, t)] * w;
      if (fbm < frames) vb = wr[reflect_index(reflect_index(fbm * hop + n - center_pad, t_pad) - pad, t)] * w;
      buf0[n] = make_float2(va, vb);
    }
    __syncthreads();
    float2 *src = buf0, *dst = buf1;
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
    for (int k = threadIdx.x; k < bins; k += blockDim.x) {
      const float2 p = z[k], q = z[k == 0 ? 0 : N - k];
      const float ar = 0.5f * (p.x + q.x), ai = 0.5f * (p.y - q.y);     // frame a
      const float br = 0.5f * (p.y + q.y), bi = -0.5f * (p.x - q.x);    // frame b
      mag[k] = sqrtf(ar * ar + ai * ai);
      mag[bins + k] = sqrtf(br * br + bi * bi);
    }
    __syncthreads();
    for (int o = threadIdx.x; o < 2 * n_mels; o += blockDim.x) {
      const int m = o >> 1, which = o & 1;
      const int lo = band[2 * m], hi = band[2 * m + 1];
      const float* mg = mag + which * bins;
      float a = 0.f;
      for (int k = lo; k < hi; ++k) a = fmaf(mg[k], fb[static_cast<size_t>(k) * n_mels + m], a);
      acc[m * kMelFrames + 2 * pair + which] = a;
    }
  }
  __syncthreads();
  float* out = mel + static_cast<size_t>(row) * n_mels * frames;
  for (int o = threadIdx.x; o < n_mels * kMelFrames; o += blockDim.x) {
    const int m = o / kMelFrames, f = f0 + (o - m * kMelFrames);
    if (f < frames) {
      float v = acc[o];
      if (apply_log) v = logf(fmaxf(v, 1e-5f));
      out[static_cast<size_t>(m) * frames + f] = v;
    }
  }
}

// --------------------------------------------------------------------------- to_flat
// ConvTranspose1d(C -> 1, kernel win, stride hop, padding pad, no bias):
//   out[b, t] = sum_c sum_j spec[b, c, j] * w[c, t + pad - j*hop]   (0 <= t + pad - j*hop < win)
__global__ void __launch_bounds__(256)
to_flat_kernel(const float* __restrict__ spec, const float* __restrict__ w, float* __restrict__ out,
               int C, int frames, int win, int hop, int pad, int t_out) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y;
  const float* sb = spec + static_cast<size_t>(b) * C * frames;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < t_out; t += gridDim.x * blockDim.x) {
    const int q = t + pad;
    int j_lo = (q - win + hop) / hop;                 // ceil((q - win + 1) / hop)
    if (q - win + 1 <= 0) j_lo = 0;
    int j_hi = q / hop;
    if (j_hi > frames - 1) j_hi = frames - 1;
    float acc = 0.f;
    for (int j = j_lo; j <= j_hi; ++j) {
      const int k = q - j * hop;
      for (int c = 0; c < C; ++c)
        acc = fmaf(sb[static_cast<size_t>(c) * frames + j], w[static_cast<size_t>(c) * win + k], acc);
    }
    out[static_cast<size_t>(b) * t_out + t] = acc;
  }
}

// dspec[b, c, j] = sum_k w[c, k] * dout[b, j*hop + k - pad]: one CTA per (b, j) stages the dout
// window in shared memory, a warp per channel (strided) reduces over k.
__global__ void __launch_bounds__(256)
to_flat_dspec_kernel(const float* __restrict__ dout, const float* __restrict__ w,
                     float* __restrict__ dspec, int C, int frames, int win, int hop, int pad,
                     int t_out) {
  extern __shared__ float s_d[];
  pdl_launch_dependents();
  pdl_wait();
  const int j = blockIdx.x, b = blockIdx.y;
  const float* db = dout + static_cast<size_t>(b) * t_out;
  for (int k = threadIdx.x; k < win; k += blockDim.x) {
    const int t = j * hop + k - pad;
    s_d[k] = (t >= 0 && t < t_out) ? db[t] : 0.f;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int c = warp; c < C; c += 8) {
    const float* wc = w + static_cast<size_t>(c) * win;
    float acc = 0.f;
    for (int k = lane; k < win; k += 32) acc = fmaf(wc[k], s_d[k], acc);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) dspec[(static_cast<size_t>(b) * C + c) * frames + j] = acc;
  }
}

// dw[c, k] += sum_b sum_j spec[b, c, j] * dout[b, j*hop + k - pad]; grid (k tiles, c, b): a thread
// owns one k of one channel for one batch row, one atomicAdd at the end (dw zeroed by the caller).
__global__ void __launch_bounds__(256)
to_flat_dw_kernel(const float* __restrict__ spec, const float* __restrict__ dout,
                  float* __restrict__ dw, int C, int frames, int win, int hop, int pad, int t_out) {
  pdl_launch_dependents();
  pdl_wait();
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const int c = blockIdx.y, b = blockIdx.z;
  if (k >= win) return;
  const float* sp = spec + (static_cast<size_t>(b) * C + c) * frames;
  const float* db = dout + static_cast<size_t>(b) * t_out;
  float acc = 0.f;
  for (int j = 0; j < frames; ++j) {
    const int t = j * hop + k - pad;
    if (t >= 0 && t < t_out) acc = fmaf(sp[j], db[t], acc);
  }
  atomicAdd(dw + static_cast<size_t>(c) * win + k, acc);
}

static int grid_1d(int64_t n, int per_block, int cap) {
  int64_t g = (n + per_block - 1) / per_block;
  if (g < 1) g = 1;
  if (g > cap) g = cap;
  return static_cast<int>(g);
}

}  // namespace adp

using namespace adp;

extern "C" int adp_resample(const float* x, const float* bank, float* y, int rows, int t, int t_out,
                            int factor_in, int factor_out, int taps, int half, adp_stream_t stream) {
  ADP_CHECK(x && bank && y, "adp_resample: null pointer");
  ADP_CHECK(rows > 0 && rows <= 65535 && t > 0 && t_out > 0 && factor_in > 0 && factor_out > 0 &&
                taps > 0 && half >= 0, "adp_resample: bad sizes");
  const size_t smem = static_cast<size_t>(factor_out) * taps * sizeof(float);
  ADP_CHECK(smem <= 48 * 1024, "adp_resample: filter bank of %zu bytes exceeds 48 KB", smem);
  ADP_CUDA(launch_k(resample_kernel, dim3(grid_1d(t_out, 256, num_sms() * 8), rows), dim3(256), smem,
                    as_stream(stream), x, bank, y, t, t_out, factor_in, factor_out, taps, half));
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_resample_adjoint(const float* dy, const float* bank, float* dx, int rows, int t,
                                    int t_out, int factor_in, int factor_out, int taps, int half,
                                    adp_stream_t stream) {
  ADP_CHECK(dy && bank && dx, "adp_resample_adjoint: null pointer");
  ADP_CHECK(rows > 0 && rows <= 65535 && t > 0 && t_out > 0 && factor_in > 0 && factor_out > 0 &&
                taps > 0 && half >= 0, "adp_resample_adjoint: bad sizes");
  const size_t smem = static_cast<size_t>(factor_out) * taps * sizeof(float);
  ADP_CHECK(smem <= 48 * 1024, "adp_resample_adjoint: filter bank of %zu bytes exceeds 48 KB", smem);
  ADP_CUDA(launch_k(resample_adjoint_kernel, dim3(grid_1d(t, 256, num_sms() * 8), rows), dim3(256), smem,
                    as_stream(stream), dy, bank, dx, t, t_out, factor_in, factor_out, taps, half));
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_mel_spectrogram(const float* wave, const float* window, const float* fb,
                                   const int32_t* band, float* mel, int rows, int t, int n_fft,
                                   int hop, int pad, int center_pad, int frames, int n_mels,
                                   int apply_log, adp_stream_t stream) {
  ADP_CHECK(wave && window && fb && band && mel, "adp_mel_spectrogram: null pointer");
  const unsigned long long plan = n_fft >= 32 && n_fft <= kMelMaxN ? fft_plan(n_fft) : 0;
  ADP_CHECK(plan != 0, "adp_mel_spectrogram: n_fft=%d must have prime factors 2, 3, 5, 7 only and lie in [32, %d]",
            n_fft, kMelMaxN);
  ADP_CHECK(rows > 0 && rows <= 65535 && hop > 0 && frames > 0 && n_mels > 0 && n_mels <= 512,
            "adp_mel_spectrogram: bad sizes");
  ADP_CHECK(pad >= 0 && pad < t && center_pad >= 0 && center_pad < t + 2 * pad,
            "adp_mel_spectrogram: each reflect pad must be shorter than the signal it mirrors "
            "(t=%d, pad=%d, center_pad=%d)", t, pad, center_pad);
  ADP_CHECK(static_cast<int64_t>(frames - 1) * hop + n_fft <= static_cast<int64_t>(t) + 2 * pad + 2 * center_pad,
            "adp_mel_spectrogram: frames do not fit the reflect-padded signal");
  const size_t smem = (static_cast<size_t>(n_fft) * 6 + static_cast<size_t>(n_mels) * kMelFrames) * sizeof(float);
  static SmemAttrCache cache;
  ADP_CUDA(ensure_dyn_smem(mel_spectrogram_kernel, smem, cache));
  ADP_CUDA(launch_k(mel_spectrogram_kernel, dim3((frames + kMelFrames - 1) / kMelFrames, rows), dim3(256),
                    smem, as_stream(stream), wave, window, fb, band, mel, t, n_fft, plan, hop, pad,
                    center_pad, frames, n_mels, apply_log));
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_to_flat(const float* spec, const float* w, float* out, int B, int C, int frames,
                           int win, int hop, int pad, int t_out, adp_stream_t stream) {
  ADP_CHECK(spec && w && out, "adp_to_flat: null pointer");
  ADP_CHECK(B > 0 && B <= 65535 && C > 0 && frames > 0 && win > 0 && hop > 0 && pad >= 0 &&
                t_out == (frames - 1) * hop - 2 * pad + win, "adp_to_flat: bad sizes");
  ADP_CUDA(launch_k(to_flat_kernel, dim3(grid_1d(t_out, 256, num_sms() * 8), B), dim3(256), (size_t)0,
                    as_stream(stream), spec, w, out, C, frames, win, hop, pad, t_out));
  ADP_LAUNCH_CHECK();
  return 0;
}

extern "C" int adp_to_flat_bwd(const float* spec, const float* w, const float* dout, float* dspec,
                               float* dw, int B, int C, int frames, int win, int hop, int pad,
                               int t_out, adp_stream_t stream) {
  ADP_CHECK(spec && w && dout, "adp_to_flat_bwd: null pointer");
  ADP_CHECK(B > 0 && B <= 65535 && C > 0 && C <= 65535 && frames > 0 && win > 0 && hop > 0 && pad >= 0 &&
                t_out == (frames - 1) * hop - 2 * pad + win, "adp_to_flat_bwd: bad sizes");
  if (dspec) {
    const size_t smem = static_cast<size_t>(win) * sizeof(float);
    ADP_CHECK(smem <= 48 * 1024, "adp_to_flat_bwd: window of %d samples exceeds 48 KB", win);
    ADP_CUDA(launch_k(to_flat_dspec_kernel, dim3(frames, B), dim3(256), smem, as_stream(stream), dout, w,
                      dspec, C, frames, win, hop, pad, t_out));
    ADP_LAUNCH_CHECK();
  }
  if (dw) {      // accumulates: the caller zeroes dw
    ADP_CUDA(launch_k(to_flat_dw_kernel, dim3((win + 255) / 256, C, B), dim3(256), (size_t)0,
                      as_stream(stream), spec, dout, dw, C, frames, win, hop, pad, t_out));
    ADP_LAUNCH_CHECK();
  }
  return 0;
}
