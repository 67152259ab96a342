// adp_attention: softmax(q k^T * scale) v, head dim D in {32, 64, 128}, on wgmma (a_unet
// AttentionBase).
//
// One CTA = one (batch, head, 128-query tile).  Two consumer warpgroups own 64 query rows each:
// S = Q K_j^T (64 x 128 keys) accumulates in registers, the online softmax runs on the
// accumulator fragments (a row is spread over the four lanes of a quad: two shuffles per
// reduction), and P is converted to bf16 in registers and fed straight back as the A operand
// of O += P V_j (the fp32 accumulator layout of a 64 x 16 slice is the bf16 A-fragment layout).
//   warps 0-7: consumers   S = Q K^T -> max -> ex2 -> P (registers) -> O += P V
//   warp 8   : TMA producer  Q once; K and V double-buffered
// K is the K-major B operand of the first GEMM (keys x d); V is used in place as the
// MN-major B operand of the second (d contiguous per key), so no transpose is materialised.
//
// Head dims: a tile row is split into swizzle-wide column chunks, each its own TMA box and
// stored [128 rows][kSW bytes] one after the other.  D = 64 is one 128-byte chunk; D = 128 is
// two (the QK^T loop steps the K-major descriptors into the second chunk after four k-steps,
// and the MN-major V descriptor reaches it through LBO); D = 32 is one 64-byte chunk with
// 64-byte swizzle.
#include "common.cuh"
#include "ptx.cuh"

namespace adp {

constexpr int kQT = 128;       // query rows per CTA
constexpr int kKT = 128;       // keys per tile
constexpr int kAttnThreads = 288;

template <int D>
struct AttnShape {
  static constexpr int kSW = D * 2 < 128 ? D * 2 : 128;   // swizzle / chunk width (bytes)
  static constexpr int kChunks = D * 2 / kSW;               // column chunks per row
  static constexpr int kQBytes = kQT * D * 2;               // 16 KB at D = 64
  static constexpr int kKVBytes = kKT * D * 2;              // 16 KB at D = 64
  static constexpr int kSmem = kQBytes + 4 * kKVBytes + 1024;   // Q + 2 x (K, V): 81 KB at D = 64
};

struct AttnParams {
  __nv_bfloat16* o;
  float* lse;         // optional [B][H][Tq]: log-sum-exp of the scaled scores (training forward)
  int Tq, Tk, ldo;
  float scale_log2;   // scale * log2(e)
};

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// descriptor offset (16-byte units) of k-step kk (16 columns) in a chunked K-major tile of
// `rows` rows: chunk kk / (kSW / 32), then 32 bytes per k-step inside the chunk
template <int SW>
__device__ __forceinline__ uint32_t kstep_off(int kk, int rows) {
  constexpr int kPerChunk = SW / 32;
  return static_cast<uint32_t>((kk / kPerChunk) * rows * SW + (kk % kPerChunk) * 32) >> 4;
}

template <int D>
__device__ __forceinline__ uint64_t v_desc_mnmajor(uint32_t addr) {
  if constexpr (D == 32) return gmma_desc_mnmajor_sw64(addr, kKT * 64);
  else return gmma_desc_mnmajor_sw128(addr, D == 64 ? 1024 : kKT * 128);
}

// LSE: the training forward, which also writes the log-sum-exp rows (p.lse); the inference
// instantiation keeps no second row sum.
template <int D, bool LSE>
__global__ void __launch_bounds__(kAttnThreads, 1)
attention_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                 const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
  using S = AttnShape<D>;
  constexpr int kSW = S::kSW, kQBytes = S::kQBytes, kKVBytes = S::kKVBytes;
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t q_full, kv_full[2], kv_empty[2];

  pdl_launch_dependents();
  const int warp = warp_id_uniform();
  const int lane = threadIdx.x & 31;
  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* base = smem_raw + ((1024u - (raw & 1023u)) & 1023u);
  uint8_t* q_s = base;
  uint8_t* k_s = q_s + kQBytes;            // [2][kKVBytes]
  uint8_t* v_s = k_s + 2 * kKVBytes;       // [2][kKVBytes]

  const int t0 = blockIdx.x * kQT;
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  const int n_tiles = (p.Tk + kKT - 1) / kKT;

  if (warp == 8 && lane == 0) {
    mbar_init(&q_full, 1);
    for (int s = 0; s < 2; ++s) { mbar_init(&kv_full[s], 1); mbar_init(&kv_empty[s], 8); }
    fence_mbar_init();
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
  }
  __syncthreads();
  pdl_wait();

  if (warp == 8) {
    // whole warp runs the loop (uniform control flow), one elected lane issues: see ptx.cuh
    if (elect_one()) {
      mbar_arrive_expect_tx(&q_full, kQBytes);
#pragma unroll
      for (int c = 0; c < S::kChunks; ++c)
        tma_load_3d(q_s + c * kQT * kSW, &tmQ, &q_full, h * D + c * (kSW / 2), t0, b);
    }
    __syncwarp();
    for (int j = 0; j < n_tiles; ++j) {
      const int s = j & 1;
      mbar_wait(&kv_empty[s], ((j >> 1) & 1) ^ 1);
      if (elect_one()) {
        mbar_arrive_expect_tx(&kv_full[s], 2 * kKVBytes);
#pragma unroll
        for (int c = 0; c < S::kChunks; ++c) {
          tma_load_3d(k_s + s * kKVBytes + c * kKT * kSW, &tmK, &kv_full[s], h * D + c * (kSW / 2), j * kKT, b);
          tma_load_3d(v_s + s * kKVBytes + c * kKT * kSW, &tmV, &kv_full[s], h * D + c * (kSW / 2), j * kKT, b);
        }
      }
      __syncwarp();
    }
    return;
  }

  // ------------------------------------------------------------------ consumers (softmax)
  const int wg = threadIdx.x >> 7;
  const int row_lo = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // fragment rows row_lo, row_lo + 8
  const int cq = 2 * (lane & 3);
  const uint64_t q_desc = gmma_desc_kmajor<kSW>(smem_u32(q_s) + wg * 64 * kSW);
  // l_run: row sum of P as rounded to bf16 for the P V GEMM (it normalises o, so o is consistent
  // with what the tensor cores saw); e_run: the same sum before that rounding (lse).  When the
  // terms of a row round the same way (near-equal scores) the two differ by up to 2^-8.
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f}, e_run[2] = {0.f, 0.f};
  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  mbar_wait(&q_full, 0);
  for (int j = 0; j < n_tiles; ++j) {
    const int s = j & 1;
    mbar_wait(&kv_full[s], (j >> 1) & 1);
    float sc[kKT / 2];
    const uint64_t k_desc = gmma_desc_kmajor<kSW>(smem_u32(k_s + s * kKVBytes));
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk)
      Wgmma<kKT>::ss<0, 0>(sc, q_desc + kstep_off<kSW>(kk, kQT), k_desc + kstep_off<kSW>(kk, kKT), kk != 0);
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(sc);

    const int key0 = j * kKT;
    if (key0 + kKT > p.Tk) {
#pragma unroll
      for (int i = 0; i < kKT / 2; ++i)
        if (key0 + 8 * (i >> 2) + cq + (i & 1) >= p.Tk) sc[i] = -INFINITY;   // key outside the sequence
    }
    float m_loc[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < kKT / 2; ++i) m_loc[(i >> 1) & 1] = fmaxf(m_loc[(i >> 1) & 1], sc[i]);
    float alpha[2], m_scaled[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      m_loc[r] = fmaxf(m_loc[r], __shfl_xor_sync(0xffffffffu, m_loc[r], 1));
      m_loc[r] = fmaxf(m_loc[r], __shfl_xor_sync(0xffffffffu, m_loc[r], 2));
      const float m_new = fmaxf(m_run[r], m_loc[r]);
      alpha[r] = ex2_approx((m_run[r] - m_new) * p.scale_log2);   // 0 on the first tile
      m_scaled[r] = m_new * p.scale_log2;
      m_run[r] = m_new;
    }
    if (j > 0) {
#pragma unroll
      for (int i = 0; i < D / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
    }
    // p = 2^(s*c - m*c) -> bf16 A fragments of P V (16 keys per fragment)
    uint32_t pa[kKT / 16][4];
    float l_tile[2] = {0.f, 0.f}, e_tile[2] = {0.f, 0.f};
#pragma unroll
    for (int kk = 0; kk < kKT / 16; ++kk) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int i = 8 * kk + 2 * q;
        const int r = q & 1;
        const float p0 = ex2_approx(sc[i] * p.scale_log2 - m_scaled[r]);
        const float p1 = ex2_approx(sc[i + 1] * p.scale_log2 - m_scaled[r]);
        pa[kk][q] = pack_bf16(p0, p1);
        const float2 pr = unpack_bf16(pa[kk][q]);   // sum what the MMA will actually see
        l_tile[r] += pr.x + pr.y;
        if constexpr (LSE) e_tile[r] += p0 + p1;
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      l_run[r] = l_run[r] * alpha[r] + l_tile[r];
      if constexpr (LSE) e_run[r] = e_run[r] * alpha[r] + e_tile[r];
    }

    const uint64_t v_desc = v_desc_mnmajor<D>(smem_u32(v_s + s * kKVBytes));
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kKT / 16; ++kk)
      Wgmma<D>::template rs<1>(o, pa[kk], v_desc + ((kk * 16 * kSW) >> 4), 1);
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[s]);
  }

#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
    if constexpr (LSE) {
      e_run[r] += __shfl_xor_sync(0xffffffffu, e_run[r], 1);
      e_run[r] += __shfl_xor_sync(0xffffffffu, e_run[r], 2);
    }
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int t = t0 + row_lo + 8 * r;
    if (t >= p.Tq) continue;
    const float inv_l = 1.f / l_run[r];
    if (LSE && (lane & 3) == 0)                  // natural-log units (adp_attention_bwd)
      p.lse[(static_cast<size_t>(b) * gridDim.y + h) * p.Tq + t] =
          (m_run[r] * p.scale_log2 + log2f(e_run[r])) * 0.6931471805599453f;
    __nv_bfloat16* orow = p.o + (static_cast<size_t>(b) * p.Tq + t) * p.ldo + h * D;
#pragma unroll
    for (int jb = 0; jb < D / 8; ++jb)
      *reinterpret_cast<uint32_t*>(orow + 8 * jb + cq) =
          pack_bf16(o[4 * jb + 2 * r] * inv_l, o[4 * jb + 2 * r + 1] * inv_l);
  }
}

}  // namespace adp

using namespace adp;

namespace {

template <int D>
int attention_launch(const void* q, const void* k, const void* v, void* o, int32_t B, int32_t H,
                     int32_t Tq, int32_t Tk, int32_t ldq, int32_t ldk, int32_t ldv, int32_t ldo,
                     float scale, float* lse, adp_stream_t stream) {
  using S = AttnShape<D>;
  CUtensorMap tmQ, tmK, tmV;
  const uint32_t box[3] = {(uint32_t)(S::kSW / 2), (uint32_t)kQT, 1};
  {
    const uint64_t dims[3] = {(uint64_t)H * D, (uint64_t)Tq, (uint64_t)B};
    const uint64_t str[2] = {(uint64_t)ldq * 2, (uint64_t)Tq * ldq * 2};
    if (int e = make_tmap_bf16(&tmQ, q, 3, dims, str, box, S::kSW)) return e;
  }
  {
    const uint64_t dims[3] = {(uint64_t)H * D, (uint64_t)Tk, (uint64_t)B};
    const uint64_t str[2] = {(uint64_t)ldk * 2, (uint64_t)Tk * ldk * 2};
    if (int e = make_tmap_bf16(&tmK, k, 3, dims, str, box, S::kSW)) return e;
  }
  {
    const uint64_t dims[3] = {(uint64_t)H * D, (uint64_t)Tk, (uint64_t)B};
    const uint64_t str[2] = {(uint64_t)ldv * 2, (uint64_t)Tk * ldv * 2};
    if (int e = make_tmap_bf16(&tmV, v, 3, dims, str, box, S::kSW)) return e;
  }
  auto kernel = lse != nullptr ? attention_kernel<D, true> : attention_kernel<D, false>;
  static SmemAttrCache smem_cache, smem_cache_lse;
  ADP_CUDA(ensure_dyn_smem(kernel, (size_t)S::kSmem, lse != nullptr ? smem_cache_lse : smem_cache));
  AttnParams p;
  p.o = static_cast<__nv_bfloat16*>(o);
  p.lse = lse;
  p.Tq = Tq;
  p.Tk = Tk;
  p.ldo = ldo;
  p.scale_log2 = scale * 1.4426950408889634f;
  dim3 grid((Tq + kQT - 1) / kQT, H, B);
  ADP_CUDA(launch_k(kernel, grid, dim3(kAttnThreads), (size_t)S::kSmem, as_stream(stream), tmQ, tmK, tmV, p));
  ADP_LAUNCH_CHECK();
  return 0;
}

}  // namespace

extern "C" int adp_attention_hd(const void* q, const void* k, const void* v, void* o, int32_t B,
                                int32_t H, int32_t head_dim, int32_t Tq, int32_t Tk, int32_t ldq,
                                int32_t ldk, int32_t ldv, int32_t ldo, float scale, float* lse,
                                adp_stream_t stream) {
  ADP_CHECK(head_dim == 32 || head_dim == 64 || head_dim == 128,
            "adp_attention: head_dim %d not supported (32, 64 or 128)", head_dim);
  ADP_CHECK(q && k && v && o, "adp_attention: null pointer");
  ADP_CHECK(B > 0 && H > 0 && Tq > 0 && Tk > 0, "adp_attention: bad sizes");
  const int64_t w = static_cast<int64_t>(H) * head_dim;
  ADP_CHECK(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0 && ldq >= w &&
                ldk >= w && ldv >= w && ldo >= w,
            "adp_attention: row pitches must be multiples of 8 and >= heads*head_dim (%d*%d)", H,
            head_dim);
  ADP_CHECK(scale > 0.f, "adp_attention: scale must be positive");
  if (head_dim == 32)
    return attention_launch<32>(q, k, v, o, B, H, Tq, Tk, ldq, ldk, ldv, ldo, scale, lse, stream);
  if (head_dim == 128)
    return attention_launch<128>(q, k, v, o, B, H, Tq, Tk, ldq, ldk, ldv, ldo, scale, lse, stream);
  return attention_launch<64>(q, k, v, o, B, H, Tq, Tk, ldq, ldk, ldv, ldo, scale, lse, stream);
}

extern "C" int adp_attention(const void* q, const void* k, const void* v, void* o, int32_t B,
                             int32_t H, int32_t Tq, int32_t Tk, int32_t ldq, int32_t ldk,
                             int32_t ldv, int32_t ldo, float scale, float* lse,
                             adp_stream_t stream) {
  return adp_attention_hd(q, k, v, o, B, H, 64, Tq, Tk, ldq, ldk, ldv, ldo, scale, lse, stream);
}
