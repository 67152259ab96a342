// adp_attention_bwd: backward of o = softmax(q k^T * scale) v (a_unet AttentionBase), head dim
// D in {32, 64, 128}.
//
// Flash-attention style: the probabilities are never stored; each kernel recomputes
// P = exp(S*scale - lse) from q, k and the log-sum-exp rows saved by adp_attention.
//   dV = P^T dO          dP = dO V^T          dS = P o (dP - delta) * scale,  delta = rowsum(dO o O)
//   dQ = dS K            dK = dS^T Q
// Three launches, no atomics (every output element has exactly one writer):
//   attn_delta_kernel   delta[b,h,t] = sum_d dO*O
//   attn_dkv_kernel     one CTA per (BT keys, head, batch), loops over the query tiles
//   attn_dq_kernel      one CTA per (BT queries, head, batch), loops over the key tiles
// BT = 64 rows (4 warps of 16) for D <= 64; at D = 128 the per-warp dK / dV accumulators double
// (128 registers) and the four padded tiles would exceed 48 KB of static shared memory, so the
// tiles shrink to BT = 32 rows (2 warps).
// Tensor cores through mma.sync.m16n8k16 (bf16 in, fp32 accumulate): the backward of attention
// is < 2 % of a training step of the networks this library runs (N <= 1024 tokens), so this
// kernel is written for exactness and simplicity; the forward is the wgmma kernel.
#include "common.cuh"
#include "ptx.cuh"

namespace adp {

template <int D>
struct BwdShape {
  static constexpr int kBT = D > 64 ? 32 : 64;   // tile rows (queries or keys)
  static constexpr int kThreads = kBT * 2;       // one warp per 16 rows
  static constexpr int kLd = D + 8;              // padded smem row (bf16 elements): ldmatrix conflict-free
};
constexpr float kLog2e = 1.4426950408889634f;

struct AttnBwdParams {
  const __nv_bfloat16 *q, *k, *v, *o, *d_o;
  const float* lse;      // [B][H][Tq] natural-log units
  float* delta;          // [B][H][Tq]
  __nv_bfloat16 *dq, *dk, *dv;
  int B, H, Tq, Tk;
  int ldq, ldk, ldv, ldo, lddo, lddq, lddk, lddv;
  float scale, scale_log2;
};

__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// BT x D bf16 tile (rows row0.., D columns from `src`, row pitch ld) -> padded smem; rows
// >= limit are zero.  16-byte chunks.
template <int D>
__device__ __forceinline__ void load_tile(__nv_bfloat16* dst, const __nv_bfloat16* src, int ld, int row0,
                                          int limit) {
  constexpr int kCh = D / 8, kLd = BwdShape<D>::kLd;
  for (int i = threadIdx.x; i < BwdShape<D>::kBT * kCh; i += blockDim.x) {
    const int r = i / kCh, c = (i % kCh) * 8;
    uint4 u = make_uint4(0, 0, 0, 0);
    if (row0 + r < limit)
      u = __ldg(reinterpret_cast<const uint4*>(src + static_cast<size_t>(row0 + r) * ld + c));
    *reinterpret_cast<uint4*>(dst + r * kLd + c) = u;
  }
}

// A fragment (16 rows r0.., k columns kc..kc+15) of a row-major padded tile
template <int LD>
__device__ __forceinline__ void frag_a(const __nv_bfloat16* tile, int r0, int kc, int lane, uint32_t (&a)[4]) {
  const int row = r0 + (lane & 7) + ((lane >> 3) & 1) * 8, col = kc + (lane >> 4) * 8;
  ldmatrix_x4(smem_u32(tile + row * LD + col), a);
}
// B fragments of TWO n-tiles (n0..n0+15) x k (kc..kc+15) from a tile stored [n][k] (k contiguous):
// r[0],r[1] = (b0,b1) of n-tile n0, r[2],r[3] = n-tile n0+8
template <int LD>
__device__ __forceinline__ void frag_b_nk(const __nv_bfloat16* tile, int n0, int kc, int lane, uint32_t (&r)[4]) {
  const int row = n0 + (lane & 7) + (lane >> 4) * 8, col = kc + ((lane >> 3) & 1) * 8;
  ldmatrix_x4(smem_u32(tile + row * LD + col), r);
}
// same, from a tile stored [k][n] (n contiguous): transposing load
template <int LD>
__device__ __forceinline__ void frag_b_kn(const __nv_bfloat16* tile, int n0, int kc, int lane, uint32_t (&r)[4]) {
  const int row = kc + (lane & 7) + ((lane >> 3) & 1) * 8, col = n0 + (lane >> 4) * 8;
  ldmatrix_x4_trans(smem_u32(tile + row * LD + col), r);
}

// ------------------------------------------------------------------------------- delta
template <int D>
__global__ void __launch_bounds__(256)
attn_delta_kernel(const AttnBwdParams p) {
  pdl_launch_dependents();
  pdl_wait();
  // one 16-byte chunk per thread, kTpr = D / 8 consecutive threads = one (row, head)
  constexpr int kTpr = D / 8;
  const size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t total = static_cast<size_t>(p.B) * p.Tq * p.H * kTpr;
  float acc = 0.f;
  size_t rh = idx / kTpr;
  const bool ok = idx < total;
  if (ok) {
    const int h = static_cast<int>(rh % p.H);
    const size_t row = rh / p.H;                 // b*Tq + t
    const int c = h * D + static_cast<int>(idx % kTpr) * 8;
    const uint4 uo = __ldg(reinterpret_cast<const uint4*>(p.o + row * p.ldo + c));
    const uint4 ud = __ldg(reinterpret_cast<const uint4*>(p.d_o + row * p.lddo + c));
    const uint32_t ao[4] = {uo.x, uo.y, uo.z, uo.w}, ad[4] = {ud.x, ud.y, ud.z, ud.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 fo = unpack_bf16(ao[j]), fd = unpack_bf16(ad[j]);
      acc += fo.x * fd.x + fo.y * fd.y;
    }
  }
#pragma unroll
  for (int m = 1; m < kTpr; m <<= 1) acc += __shfl_xor_sync(0xffffffffu, acc, m);
  if (ok && idx % kTpr == 0) {
    const int h = static_cast<int>(rh % p.H);
    const size_t row = rh / p.H;
    const size_t b = row / p.Tq, t = row - b * p.Tq;
    p.delta[(b * p.H + h) * p.Tq + t] = acc;
  }
}

// --------------------------------------------------------------------------------- dK, dV
template <int D>
__global__ void __launch_bounds__(BwdShape<D>::kThreads)
attn_dkv_kernel(const AttnBwdParams p) {
  constexpr int kBT = BwdShape<D>::kBT, kLd = BwdShape<D>::kLd;
  constexpr int kNQ = kBT / 8;     // 8-query n-tiles of S^T / dP^T
  constexpr int kND = D / 8;       // 8-column n-tiles of dK / dV
  pdl_launch_dependents();
  pdl_wait();
  __shared__ __align__(16) __nv_bfloat16 k_s[kBT * kLd], v_s[kBT * kLd], q_s[kBT * kLd], do_s[kBT * kLd];
  __shared__ float lse_s[kBT], dl_s[kBT];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int key0 = blockIdx.x * kBT, h = blockIdx.y, b = blockIdx.z;
  const __nv_bfloat16* qb = p.q + static_cast<size_t>(b) * p.Tq * p.ldq + h * D;
  const __nv_bfloat16* kb = p.k + static_cast<size_t>(b) * p.Tk * p.ldk + h * D;
  const __nv_bfloat16* vb = p.v + static_cast<size_t>(b) * p.Tk * p.ldv + h * D;
  const __nv_bfloat16* dob = p.d_o + static_cast<size_t>(b) * p.Tq * p.lddo + h * D;
  const float* lse_b = p.lse + (static_cast<size_t>(b) * p.H + h) * p.Tq;
  const float* dl_b = p.delta + (static_cast<size_t>(b) * p.H + h) * p.Tq;
  load_tile<D>(k_s, kb, p.ldk, key0, p.Tk);
  load_tile<D>(v_s, vb, p.ldv, key0, p.Tk);
  float dv[kND][4], dk[kND][4];
#pragma unroll
  for (int i = 0; i < kND; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) { dv[i][j] = 0.f; dk[i][j] = 0.f; }
  const int r0 = warp * 16;                      // this warp's 16 keys inside the tile
  const int n_qt = (p.Tq + kBT - 1) / kBT;
  for (int qt = 0; qt < n_qt; ++qt) {
    __syncthreads();                             // previous tile fully consumed (and K/V visible)
    load_tile<D>(q_s, qb, p.ldq, qt * kBT, p.Tq);
    load_tile<D>(do_s, dob, p.lddo, qt * kBT, p.Tq);
    if (threadIdx.x < kBT) {
      const int t = qt * kBT + threadIdx.x;
      // invalid queries: lse = +inf -> P = 0
      lse_s[threadIdx.x] = t < p.Tq ? lse_b[t] * kLog2e : INFINITY;
      dl_s[threadIdx.x] = t < p.Tq ? dl_b[t] : 0.f;
    }
    __syncthreads();
    // S^T = K Q^T and dP^T = V dO^T : [16 keys] x [kBT queries]
    float s[kNQ][4], dp[kNQ][4];
#pragma unroll
    for (int i = 0; i < kNQ; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) { s[i][j] = 0.f; dp[i][j] = 0.f; }
#pragma unroll
    for (int ks = 0; ks < D / 16; ++ks) {
      uint32_t ka[4], va[4];
      frag_a<kLd>(k_s, r0, ks * 16, lane, ka);
      frag_a<kLd>(v_s, r0, ks * 16, lane, va);
#pragma unroll
      for (int n2 = 0; n2 < kBT / 16; ++n2) {
        uint32_t bq[4], bd[4];
        frag_b_nk<kLd>(q_s, n2 * 16, ks * 16, lane, bq);
        frag_b_nk<kLd>(do_s, n2 * 16, ks * 16, lane, bd);
        mma_16816(s[2 * n2], ka, bq[0], bq[1]);
        mma_16816(s[2 * n2 + 1], ka, bq[2], bq[3]);
        mma_16816(dp[2 * n2], va, bd[0], bd[1]);
        mma_16816(dp[2 * n2 + 1], va, bd[2], bd[3]);
      }
    }
    // P^T and dS^T as bf16 A fragments (k = queries)
    uint32_t pa[kBT / 16][4], dsa[kBT / 16][4];
#pragma unroll
    for (int nt = 0; nt < kNQ; ++nt) {
      const int qc = nt * 8 + (lane & 3) * 2;
      const float l0 = lse_s[qc], l1 = lse_s[qc + 1], d0 = dl_s[qc], d1 = dl_s[qc + 1];
      const float p0 = ex2f(s[nt][0] * p.scale_log2 - l0), p1 = ex2f(s[nt][1] * p.scale_log2 - l1);
      const float p2 = ex2f(s[nt][2] * p.scale_log2 - l0), p3 = ex2f(s[nt][3] * p.scale_log2 - l1);
      const float e0 = p0 * (dp[nt][0] - d0) * p.scale, e1 = p1 * (dp[nt][1] - d1) * p.scale;
      const float e2 = p2 * (dp[nt][2] - d0) * p.scale, e3 = p3 * (dp[nt][3] - d1) * p.scale;
      const int ks = nt >> 1, hi = (nt & 1) * 2;
      pa[ks][hi] = pack_bf16(p0, p1);      // rows lane/4
      pa[ks][hi + 1] = pack_bf16(p2, p3);  // rows lane/4 + 8
      dsa[ks][hi] = pack_bf16(e0, e1);
      dsa[ks][hi + 1] = pack_bf16(e2, e3);
    }
    // dV += P^T dO ; dK += dS^T Q   (B operands stored [k = query][n = d])
#pragma unroll
    for (int ks = 0; ks < kBT / 16; ++ks) {
#pragma unroll
      for (int n2 = 0; n2 < D / 16; ++n2) {
        uint32_t bd[4], bq[4];
        frag_b_kn<kLd>(do_s, n2 * 16, ks * 16, lane, bd);
        frag_b_kn<kLd>(q_s, n2 * 16, ks * 16, lane, bq);
        mma_16816(dv[2 * n2], pa[ks], bd[0], bd[1]);
        mma_16816(dv[2 * n2 + 1], pa[ks], bd[2], bd[3]);
        mma_16816(dk[2 * n2], dsa[ks], bq[0], bq[1]);
        mma_16816(dk[2 * n2 + 1], dsa[ks], bq[2], bq[3]);
      }
    }
  }
  // store
  const int ra = key0 + r0 + (lane >> 2), rb = ra + 8;
  __nv_bfloat16* dkb = p.dk + static_cast<size_t>(b) * p.Tk * p.lddk + h * D;
  __nv_bfloat16* dvb = p.dv + static_cast<size_t>(b) * p.Tk * p.lddv + h * D;
#pragma unroll
  for (int nt = 0; nt < kND; ++nt) {
    const int c = nt * 8 + (lane & 3) * 2;
    if (ra < p.Tk) {
      *reinterpret_cast<uint32_t*>(dkb + static_cast<size_t>(ra) * p.lddk + c) = pack_bf16(dk[nt][0], dk[nt][1]);
      *reinterpret_cast<uint32_t*>(dvb + static_cast<size_t>(ra) * p.lddv + c) = pack_bf16(dv[nt][0], dv[nt][1]);
    }
    if (rb < p.Tk) {
      *reinterpret_cast<uint32_t*>(dkb + static_cast<size_t>(rb) * p.lddk + c) = pack_bf16(dk[nt][2], dk[nt][3]);
      *reinterpret_cast<uint32_t*>(dvb + static_cast<size_t>(rb) * p.lddv + c) = pack_bf16(dv[nt][2], dv[nt][3]);
    }
  }
}

// ------------------------------------------------------------------------------------- dQ
template <int D>
__global__ void __launch_bounds__(BwdShape<D>::kThreads)
attn_dq_kernel(const AttnBwdParams p) {
  constexpr int kBT = BwdShape<D>::kBT, kLd = BwdShape<D>::kLd;
  constexpr int kNK = kBT / 8;     // 8-key n-tiles of S / dP
  constexpr int kND = D / 8;       // 8-column n-tiles of dQ
  pdl_launch_dependents();
  pdl_wait();
  __shared__ __align__(16) __nv_bfloat16 k_s[kBT * kLd], v_s[kBT * kLd], q_s[kBT * kLd], do_s[kBT * kLd];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t0 = blockIdx.x * kBT, h = blockIdx.y, b = blockIdx.z;
  const __nv_bfloat16* qb = p.q + static_cast<size_t>(b) * p.Tq * p.ldq + h * D;
  const __nv_bfloat16* kb = p.k + static_cast<size_t>(b) * p.Tk * p.ldk + h * D;
  const __nv_bfloat16* vb = p.v + static_cast<size_t>(b) * p.Tk * p.ldv + h * D;
  const __nv_bfloat16* dob = p.d_o + static_cast<size_t>(b) * p.Tq * p.lddo + h * D;
  load_tile<D>(q_s, qb, p.ldq, t0, p.Tq);
  load_tile<D>(do_s, dob, p.lddo, t0, p.Tq);
  const int r0 = warp * 16;
  const int ta = t0 + r0 + (lane >> 2), tb = ta + 8;
  const size_t rowbase = (static_cast<size_t>(b) * p.H + h) * p.Tq;
  const float lse_a = ta < p.Tq ? p.lse[rowbase + ta] * kLog2e : INFINITY;
  const float lse_b = tb < p.Tq ? p.lse[rowbase + tb] * kLog2e : INFINITY;
  const float dl_a = ta < p.Tq ? p.delta[rowbase + ta] : 0.f;
  const float dl_b = tb < p.Tq ? p.delta[rowbase + tb] : 0.f;
  float dq[kND][4];
#pragma unroll
  for (int i = 0; i < kND; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) dq[i][j] = 0.f;
  const int n_kt = (p.Tk + kBT - 1) / kBT;
  for (int kt = 0; kt < n_kt; ++kt) {
    __syncthreads();
    load_tile<D>(k_s, kb, p.ldk, kt * kBT, p.Tk);
    load_tile<D>(v_s, vb, p.ldv, kt * kBT, p.Tk);
    __syncthreads();
    float s[kNK][4], dp[kNK][4];
#pragma unroll
    for (int i = 0; i < kNK; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) { s[i][j] = 0.f; dp[i][j] = 0.f; }
#pragma unroll
    for (int ks = 0; ks < D / 16; ++ks) {
      uint32_t qa[4], da[4];
      frag_a<kLd>(q_s, r0, ks * 16, lane, qa);
      frag_a<kLd>(do_s, r0, ks * 16, lane, da);
#pragma unroll
      for (int n2 = 0; n2 < kBT / 16; ++n2) {
        uint32_t bk[4], bv[4];
        frag_b_nk<kLd>(k_s, n2 * 16, ks * 16, lane, bk);
        frag_b_nk<kLd>(v_s, n2 * 16, ks * 16, lane, bv);
        mma_16816(s[2 * n2], qa, bk[0], bk[1]);
        mma_16816(s[2 * n2 + 1], qa, bk[2], bk[3]);
        mma_16816(dp[2 * n2], da, bv[0], bv[1]);
        mma_16816(dp[2 * n2 + 1], da, bv[2], bv[3]);
      }
    }
    uint32_t dsa[kBT / 16][4];
#pragma unroll
    for (int nt = 0; nt < kNK; ++nt) {
      const int key = kt * kBT + nt * 8 + (lane & 3) * 2;
      const bool ok0 = key < p.Tk, ok1 = key + 1 < p.Tk;
      const float p0 = ok0 ? ex2f(s[nt][0] * p.scale_log2 - lse_a) : 0.f;
      const float p1 = ok1 ? ex2f(s[nt][1] * p.scale_log2 - lse_a) : 0.f;
      const float p2 = ok0 ? ex2f(s[nt][2] * p.scale_log2 - lse_b) : 0.f;
      const float p3 = ok1 ? ex2f(s[nt][3] * p.scale_log2 - lse_b) : 0.f;
      const int ks = nt >> 1, hi = (nt & 1) * 2;
      dsa[ks][hi] = pack_bf16(p0 * (dp[nt][0] - dl_a) * p.scale, p1 * (dp[nt][1] - dl_a) * p.scale);
      dsa[ks][hi + 1] = pack_bf16(p2 * (dp[nt][2] - dl_b) * p.scale, p3 * (dp[nt][3] - dl_b) * p.scale);
    }
    // dQ += dS K   (K stored [k = key][n = d])
#pragma unroll
    for (int ks = 0; ks < kBT / 16; ++ks) {
#pragma unroll
      for (int n2 = 0; n2 < D / 16; ++n2) {
        uint32_t bk[4];
        frag_b_kn<kLd>(k_s, n2 * 16, ks * 16, lane, bk);
        mma_16816(dq[2 * n2], dsa[ks], bk[0], bk[1]);
        mma_16816(dq[2 * n2 + 1], dsa[ks], bk[2], bk[3]);
      }
    }
  }
  __nv_bfloat16* dqb = p.dq + static_cast<size_t>(b) * p.Tq * p.lddq + h * D;
#pragma unroll
  for (int nt = 0; nt < kND; ++nt) {
    const int c = nt * 8 + (lane & 3) * 2;
    if (ta < p.Tq)
      *reinterpret_cast<uint32_t*>(dqb + static_cast<size_t>(ta) * p.lddq + c) = pack_bf16(dq[nt][0], dq[nt][1]);
    if (tb < p.Tq)
      *reinterpret_cast<uint32_t*>(dqb + static_cast<size_t>(tb) * p.lddq + c) = pack_bf16(dq[nt][2], dq[nt][3]);
  }
}

// --------------------------------------------------------------------- LayerNorm-fold backward
// The attention projections run with the LayerNorm affine folded in: Wf = W*diag(g), bf = W b.
// Given dWf [N][ldwf] and dbf [N]:  dW = dWf*g + dbf (x) b ;  dg += colsum(dWf o W) ;
// db += W^T dbf.   grid (ceil(C/128), ceil(N/64)), 128 threads: thread = one column.
__global__ void __launch_bounds__(128)
ln_fold_bwd_kernel(const float* __restrict__ w, const float* __restrict__ g, const float* __restrict__ bvec,
                   const float* __restrict__ dwf, int ldwf, const float* __restrict__ dbf,
                   float* __restrict__ dw, float* __restrict__ dg, float* __restrict__ db, int N, int C) {
  pdl_launch_dependents();
  pdl_wait();
  const int c = blockIdx.x * 128 + threadIdx.x;
  const int n0 = blockIdx.y * 64, n1 = min(n0 + 64, N);
  if (c >= C) return;
  const float gc = g[c], bc = bvec[c];
  float ag = 0.f, ab = 0.f;
  for (int n = n0; n < n1; ++n) {
    const float wv = w[static_cast<size_t>(n) * C + c];
    const float dv = dwf[static_cast<size_t>(n) * ldwf + c];
    const float dbn = dbf[n];
    dw[static_cast<size_t>(n) * C + c] = dv * gc + dbn * bc;
    ag += dv * wv;
    ab += wv * dbn;
  }
  atomicAdd(dg + c, ag);
  atomicAdd(db + c, ab);
}

}  // namespace adp

using namespace adp;

namespace {

template <int D>
int attention_bwd_launch(const AttnBwdParams& p, cudaStream_t s) {
  constexpr int kBT = BwdShape<D>::kBT, kThreads = BwdShape<D>::kThreads;
  const size_t chunks = static_cast<size_t>(p.B) * p.Tq * p.H * (D / 8);
  ADP_CUDA(launch_k(attn_delta_kernel<D>, dim3(static_cast<unsigned>((chunks + 255) / 256)), dim3(256),
                    (size_t)0, s, p));
  ADP_CUDA(launch_k(attn_dkv_kernel<D>, dim3((p.Tk + kBT - 1) / kBT, p.H, p.B), dim3(kThreads), (size_t)0, s, p));
  ADP_CUDA(launch_k(attn_dq_kernel<D>, dim3((p.Tq + kBT - 1) / kBT, p.H, p.B), dim3(kThreads), (size_t)0, s, p));
  ADP_LAUNCH_CHECK();
  return 0;
}

}  // namespace

extern "C" int adp_attention_bwd_hd(const adp_attention_bwd_args* args, int32_t head_dim,
                                    adp_stream_t stream) {
  ADP_CHECK(head_dim == 32 || head_dim == 64 || head_dim == 128,
            "adp_attention_bwd: head_dim %d not supported (32, 64 or 128)", head_dim);
  ADP_CHECK(args != nullptr, "adp_attention_bwd: null args");
  const adp_attention_bwd_args& a = *args;
  ADP_CHECK(a.q && a.k && a.v && a.o && a.d_o && a.lse && a.delta && a.dq && a.dk && a.dv,
            "adp_attention_bwd: null pointer");
  ADP_CHECK(a.B > 0 && a.H > 0 && a.Tq > 0 && a.Tk > 0 && a.scale > 0.f, "adp_attention_bwd: bad sizes");
  const int lds[8] = {a.ldq, a.ldk, a.ldv, a.ldo, a.lddo, a.lddq, a.lddk, a.lddv};
  for (int i = 0; i < 8; ++i)
    ADP_CHECK(lds[i] % 8 == 0 && lds[i] >= static_cast<int64_t>(a.H) * head_dim,
              "adp_attention_bwd: row pitch %d must be a multiple of 8 and >= heads*head_dim (%d*%d)",
              lds[i], a.H, head_dim);
  AttnBwdParams p;
  p.q = static_cast<const __nv_bfloat16*>(a.q);
  p.k = static_cast<const __nv_bfloat16*>(a.k);
  p.v = static_cast<const __nv_bfloat16*>(a.v);
  p.o = static_cast<const __nv_bfloat16*>(a.o);
  p.d_o = static_cast<const __nv_bfloat16*>(a.d_o);
  p.lse = a.lse;
  p.delta = a.delta;
  p.dq = static_cast<__nv_bfloat16*>(a.dq);
  p.dk = static_cast<__nv_bfloat16*>(a.dk);
  p.dv = static_cast<__nv_bfloat16*>(a.dv);
  p.B = a.B; p.H = a.H; p.Tq = a.Tq; p.Tk = a.Tk;
  p.ldq = a.ldq; p.ldk = a.ldk; p.ldv = a.ldv; p.ldo = a.ldo; p.lddo = a.lddo;
  p.lddq = a.lddq; p.lddk = a.lddk; p.lddv = a.lddv;
  p.scale = a.scale;
  p.scale_log2 = a.scale * kLog2e;
  cudaStream_t s = as_stream(stream);
  if (head_dim == 32) return attention_bwd_launch<32>(p, s);
  if (head_dim == 128) return attention_bwd_launch<128>(p, s);
  return attention_bwd_launch<64>(p, s);
}

extern "C" int adp_attention_bwd(const adp_attention_bwd_args* args, adp_stream_t stream) {
  return adp_attention_bwd_hd(args, 64, stream);
}

extern "C" int adp_ln_fold_bwd(const float* w, const float* g, const float* b, const float* dwf,
                               int32_t ldwf, const float* dbf, float* dw, float* dg, float* db,
                               int32_t N, int32_t C, adp_stream_t stream) {
  ADP_CHECK(w && g && b && dwf && dbf && dw && dg && db, "adp_ln_fold_bwd: null pointer");
  ADP_CHECK(N > 0 && C > 0 && ldwf >= C, "adp_ln_fold_bwd: bad sizes");
  dim3 grid((C + 127) / 128, (N + 63) / 64);
  ADP_CUDA(launch_k(ln_fold_bwd_kernel, grid, dim3(128), (size_t)0, as_stream(stream), w, g, b, dwf,
                    (int)ldwf, dbf, dw, dg, db, (int)N, (int)C));
  return 0;
}
