// adp_conv_gemm: persistent shifted-tap GEMM on wgmma (see include/adp_b200.h).
//
// GEMM view (swapped w.r.t. the usual conv-as-GEMM so that one accumulator ROW is one time
// position): D[m = time position, n = output channel] = sum_{tap,k} A[m + off(tap), k] * W[n, tap, k]
//   A: channels-last activations -> K-major operand.  ONE TMA box of (128 + span) rows per
//      64-channel chunk serves all taps: tap j is the same smem tile read through a wgmma
//      descriptor whose start address is advanced by j rows (the swizzle is a function of the
//      absolute smem address, so row-shifted starts need no re-layout).  Rows outside [0,T)
//      are zero-filled by TMA = the conv's zero padding.
//   W: packed weights [N][taps*C_in] -> K-major operand.
//   A pipeline stage = KC chunks x {A box, one W box per tap} behind ONE full/empty mbarrier
//      pair, so the issue loops pay one barrier round trip per KC*taps*4 MMAs.
//   D: fp32 in registers.  Two consumer warpgroups own 64 tile rows each (m64nBNk16 per
//      warpgroup); one MMA stage stays in flight while the next is issued.
// Persistent: each CTA owns a contiguous range of tiles (n fastest).  Warp roles (288 threads):
// warps 0-7 the two consumer warpgroups (MMA issue + epilogue straight from the accumulator
// registers), warp 8 the TMA producer, which keeps filling the ring while the consumers drain
// a tile.  GroupNorm partial sums of the output are reduced per warp into per-warp shared-memory
// slots; one global reduction per batch change.
#include "common.cuh"
#include "ptx.cuh"

namespace adp {

// diagnostic switches (adp_debug_set): [2] 1 = weights are not written by the preceding kernels
// (fetch them before griddepcontrol.wait); [3] CTAs/SM override; [5] KC override; [6] PDL
int g_debug[8] = {0, 0, 0, 0, 0, 0, 0, 0};

constexpr int kBM = 128;
constexpr int kMaxStages = 8;
constexpr int kMaxGroups = 8;      // GroupNorm groups handled by the fused statistics
constexpr int kConsumers = 256;    // two warpgroups
constexpr int kGemmThreads = kConsumers + 32;
constexpr int kSmemPerSM = 228 * 1024;
constexpr int kSmemPerBlock = 227 * 1024;

struct Gemm2Params {
  __nv_bfloat16* out;
  const __nv_bfloat16* residual;
  const float* bias;
  const float* gate;
  double* stats;
  int B, T, tiles_per_batch, c_in, ldo;
  int n_pad, n_valid;
  int ntaps, tap_off0, up_factor;
  int groups, group_size, group_shift;   // group_shift >= 0: group = ch >> shift
  int out_fp32, ld_gate;
  int n_tiles_n, total_tiles, tiles_per_cta;
  int a_rows;            // rows per A box = 128 + tap span
  int kc;                // 64-channel chunks per stage
  int k_stages;          // stages per tile = (c_in / BK) / kc
  int n_stages;          // ring depth
  int a_sub_bytes, w_sub_bytes, stage_bytes, max_taps;
  int early_w;           // weights may be fetched before griddepcontrol.wait
  // optional GroupNorm-apply + SiLU on the A operand (the consumers rewrite the smem tile)
  const double* gn_stats;   // fp64 [B][gn_groups][2] of the A tensor
  const float* gn_gamma;
  const float* gn_beta;
  float gn_eps;
  int gn_groups;
};

struct TileInfo {
  int b, t0, n0, phase, ch0, ntaps, min_off;
};

__device__ __forceinline__ TileInfo tile_info(const Gemm2Params& p, int tile, int BN) {
  TileInfo ti;
  const int m_tile = tile / p.n_tiles_n;
  const int n_tile = tile - m_tile * p.n_tiles_n;
  ti.b = m_tile / p.tiles_per_batch;
  ti.t0 = (m_tile - ti.b * p.tiles_per_batch) * kBM;
  ti.n0 = n_tile * BN;
  ti.phase = ti.n0 / p.n_pad;
  ti.ch0 = ti.n0 - ti.phase * p.n_pad;
  if (p.up_factor > 1) {   // nearest-upsample + conv3: taps collapse per output phase
    if (ti.phase == 0) { ti.ntaps = 2; ti.min_off = -1; }
    else if (ti.phase == p.up_factor - 1) { ti.ntaps = 2; ti.min_off = 0; }
    else { ti.ntaps = 1; ti.min_off = 0; }
  } else {
    ti.ntaps = p.ntaps;
    ti.min_off = p.tap_off0;
  }
  return ti;
}

// SiLU with ONE special-function op per element (the A-tile transform is MUFU-bound):
// z*sigmoid(z) = 0.5*z*(1 + tanh(z/2)); tanh.approx error (2^-11) is below bf16 rounding.
__device__ __forceinline__ float silu_tanh(float z) {
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.5f * z));
  const float hz = 0.5f * z;
  return fmaf(hz, t, hz);
}

// Running per-group (sum, sumsq) of one consumer warp.  Channels arrive in increasing order and
// the group is warp-uniform: lanes accumulate privately; on a group change the warp reduces with
// shuffles and lane 0 adds into the warp's OWN shared-memory column.  Each column has a single
// writer and the columns are summed in warp order, so the statistics do not depend on the
// order in which warps finish (only the fp64 global reduction across CTAs does).
struct WarpStats {
  int cur_g = -1;
  float s = 0.f, q = 0.f;
  __device__ __forceinline__ void flush(float (*slots)[8], int w, int lane) {
    if (cur_g >= 0) {
      const float ws = warp_sum(s), wq = warp_sum(q);
      if (lane == 0) { slots[2 * cur_g][w] += ws; slots[2 * cur_g + 1][w] += wq; }
    }
    s = 0.f; q = 0.f;
  }
  __device__ __forceinline__ void add(float v, int g, float (*slots)[8], int w, int lane) {
    if (g != cur_g) { flush(slots, w, lane); cur_g = g; }
    s += v; q += v * v;
  }
};

template <int BN, int SW, bool XF>
__global__ void __launch_bounds__(kGemmThreads, BN <= 32 ? 3 : (BN <= 64 ? 2 : 1))
conv_gemm2_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
                  const Gemm2Params p) {
  constexpr int BK = SW / 2;
  constexpr int NACC = BN / 2;                    // accumulator registers per consumer thread
  constexpr uint32_t kWTapBytes = BN * SW;        // bytes one W box writes
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t full_bar[kMaxStages], empty_bar[kMaxStages];
  __shared__ float s_part[2 * kMaxGroups][8];     // (sum, sumsq) per group of the current batch, per consumer warp
  __shared__ __align__(16) float s_coef[XF ? 2 * 1024 : 4];   // (a, d) per input channel of the current batch

  pdl_launch_dependents();
  const int warp = warp_id_uniform();
  const int lane = threadIdx.x & 31;
  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* ring = smem_raw + ((1024u - (raw & 1023u)) & 1023u);

  const int tile_begin = blockIdx.x * p.tiles_per_cta;
  int tile_end = tile_begin + p.tiles_per_cta;
  if (tile_end > p.total_tiles) tile_end = p.total_tiles;

  if (threadIdx.x < 2 * kMaxGroups * 8) (&s_part[0][0])[threadIdx.x] = 0.f;
  if (warp == 8 && lane == 0) {
    for (int s = 0; s < p.n_stages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }
    fence_mbar_init();
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmW);
  }
  __syncthreads();
  // Programmatic dependent launch: this kernel may have started while its predecessor still
  // runs.  Activations / statistics / conditioning come from the predecessor, so every role
  // that reads them calls griddepcontrol.wait first.  The WEIGHTS do not (p.early_w, set by the
  // host only while it captures an inference graph): the producer puts the weight boxes of the
  // first ring stages in flight BEFORE waiting, taking the first-load latency off the
  // critical path of the many short GEMMs that follow an elementwise kernel.
  if (warp == 8) {
    // ---------------------------------------------------------------------- TMA producer
    const uint32_t a_bytes = static_cast<uint32_t>(p.a_rows) * SW;
    const int total_it = (tile_end - tile_begin) * p.k_stages;
    int early = 0;
    if (p.early_w) {
      early = total_it < p.n_stages ? total_it : p.n_stages;
      if (elect_one()) {
        int tile = tile_begin, ks = 0;
        for (int it = 0; it < early; ++it) {          // stage `it` of the (still empty) ring
          const TileInfo ti = tile_info(p, tile, BN);
          uint8_t* st = ring + it * p.stage_bytes;
          mbar_arrive_expect_tx(&full_bar[it], static_cast<uint32_t>(p.kc) * (a_bytes + ti.ntaps * kWTapBytes));
          for (int c = 0; c < p.kc; ++c) {
            const int k0 = (ks * p.kc + c) * BK;
            uint8_t* wdst = st + p.kc * p.a_sub_bytes + c * p.max_taps * p.w_sub_bytes;
            for (int tap = 0; tap < ti.ntaps; ++tap)
              tma_load_2d(wdst + tap * p.w_sub_bytes, &tmW, &full_bar[it], tap * p.c_in + k0, ti.n0);
          }
          if (++ks == p.k_stages) { ks = 0; ++tile; }
        }
      }
      __syncwarp();
    }
    pdl_wait();
    int s = 0, it = 0;
    uint32_t ph = 0;
    for (int tile = tile_begin; tile < tile_end; ++tile) {
      const TileInfo ti = tile_info(p, tile, BN);
      const uint32_t tx = static_cast<uint32_t>(p.kc) * (a_bytes + ti.ntaps * kWTapBytes);
      for (int ks = 0; ks < p.k_stages; ++ks, ++it) {
        const bool armed = it < early;                 // barrier armed + weights already issued
        if (!armed) mbar_wait(&empty_bar[s], ph ^ 1);
        uint8_t* st = ring + s * p.stage_bytes;
        if (elect_one()) {
          if (!armed) mbar_arrive_expect_tx(&full_bar[s], tx);
          for (int c = 0; c < p.kc; ++c) {
            const int k0 = (ks * p.kc + c) * BK;
            tma_load_3d(st + c * p.a_sub_bytes, &tmA, &full_bar[s], k0, ti.t0 + ti.min_off, ti.b);
            if (armed) continue;
            uint8_t* wdst = st + p.kc * p.a_sub_bytes + c * p.max_taps * p.w_sub_bytes;
            for (int tap = 0; tap < ti.ntaps; ++tap)
              tma_load_2d(wdst + tap * p.w_sub_bytes, &tmW, &full_bar[s], tap * p.c_in + k0, ti.n0);
          }
        }
        __syncwarp();
        if (++s == p.n_stages) { s = 0; ph ^= 1; }
      }
    }
    return;
  }

  // ------------------------------------------------------------------------------ consumers
  pdl_wait();
  const int tid = threadIdx.x;                 // 0..255
  const int wg = tid >> 7;                     // warpgroup: tile rows [64*wg, 64*wg + 64)
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // fragment rows r0 and r0 + 8
  const int cq = 2 * (lane & 3);               // fragment column offset inside each 8-column block
  const bool do_stats = p.stats != nullptr;
  WarpStats acc_st;
  int cur_b = -1, coef_b = -1;

  auto publish_stats = [&](int b_done) {       // all 256 consumer threads
    acc_st.flush(s_part, warp, lane);
    acc_st.cur_g = -1;
    named_bar_sync(1, kConsumers);
    if (tid < 2 * p.groups) {
      float tot = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) { tot += s_part[tid][w]; s_part[tid][w] = 0.f; }
      if (tot != 0.f) atomicAdd(p.stats + static_cast<size_t>(b_done) * 2 * p.groups + tid, static_cast<double>(tot));
    }
    named_bar_sync(1, kConsumers);
  };

  // descriptor of the ring base; byte offsets are added to the 14-bit address field
  const uint64_t desc0 = gmma_desc_kmajor<SW>(smem_u32(ring));
  const uint32_t stage_u = static_cast<uint32_t>(p.stage_bytes) >> 4;
  const uint32_t a_sub_u = static_cast<uint32_t>(p.a_sub_bytes) >> 4;
  const uint32_t w_sub_u = static_cast<uint32_t>(p.w_sub_bytes) >> 4;
  const uint32_t w_base_u = static_cast<uint32_t>(p.kc) * a_sub_u;
  const uint32_t wg_row_u = static_cast<uint32_t>(wg * 64 * SW) >> 4;
  int s = 0;
  uint32_t ph = 0;
  for (int tile = tile_begin; tile < tile_end; ++tile) {
    const TileInfo ti = tile_info(p, tile, BN);
    if constexpr (XF) {
      if (ti.b != coef_b) {     // (a, d) of every input channel for this batch element, once
        named_bar_sync(1, kConsumers);          // previous batch's coefficients no longer in use
        const int gsz = p.c_in / p.gn_groups;
        const double inv_n = 1.0 / (static_cast<double>(gsz) * p.T);
        for (int ch = tid; ch < p.c_in; ch += kConsumers) {
          const int g = ch / gsz;
          const double mean = p.gn_stats[(static_cast<size_t>(ti.b) * p.gn_groups + g) * 2] * inv_n;
          const float var = fmaxf(static_cast<float>(
              p.gn_stats[(static_cast<size_t>(ti.b) * p.gn_groups + g) * 2 + 1] * inv_n - mean * mean), 0.f);
          const float ga = __ldg(p.gn_gamma + ch) * rsqrtf(var + p.gn_eps);
          s_coef[2 * ch] = ga;
          s_coef[2 * ch + 1] = __ldg(p.gn_beta + ch) - static_cast<float>(mean) * ga;
        }
        named_bar_sync(1, kConsumers);
        coef_b = ti.b;
      }
    }
    float acc[NACC];
    uint32_t accumulate = 0;
    int prev_s = -1;
    for (int ks = 0; ks < p.k_stages; ++ks) {
      mbar_wait(&full_bar[s], ph);
      if constexpr (XF) {
        // a = silu(x*ga + de) in place, two threads per tile row.  The TMA tile is SW-byte rows
        // with the 16-byte chunks XOR-swizzled by address bits [7, 7+log2(SW/16)); zero rows
        // (conv padding) stay zero.  Rows are shared by both warpgroups (tap shifts), so all
        // consumers finish the stage before either issues its MMAs.
        constexpr int CPR = SW / 16;                 // 16-byte chunks per row
        constexpr int CPT = CPR / 2 > 0 ? CPR / 2 : 1;   // chunks per thread
        uint8_t* st = ring + s * p.stage_bytes;
        for (int c = 0; c < p.kc; ++c) {
          uint8_t* sub = st + c * p.a_sub_bytes;
          const float* cf = s_coef + (ks * p.kc + c) * BK * 2;
          for (int rr = tid >> 1; rr < p.a_rows; rr += kConsumers / 2) {
            const int t = ti.t0 + ti.min_off + rr;
            if (t < 0 || t >= p.T) continue;               // TMA zero fill = conv padding
            const uint32_t row_off = static_cast<uint32_t>(rr) * SW;
            const int swz = (row_off >> 7) & (CPR - 1);
#pragma unroll
            for (int q = 0; q < CPT; ++q) {
              const int pc = (CPR >= 2) ? (tid & 1) * CPT + q : 0;      // physical chunk
              if (CPR < 2 && (tid & 1)) continue;
              const int lc = pc ^ swz;                                  // logical chunk
              uint4* ptr = reinterpret_cast<uint4*>(sub + row_off + pc * 16);
              const uint4 u = *ptr;
              const float4* c4 = reinterpret_cast<const float4*>(cf + lc * 16);
              const float4 k0 = c4[0], k1 = c4[1], k2 = c4[2], k3 = c4[3];   // (a,d) x 8 channels
              const float2 f0 = unpack_bf16(u.x), f1 = unpack_bf16(u.y);
              const float2 f2 = unpack_bf16(u.z), f3 = unpack_bf16(u.w);
              uint4 o;
              o.x = pack_bf16(silu_tanh(f0.x * k0.x + k0.y), silu_tanh(f0.y * k0.z + k0.w));
              o.y = pack_bf16(silu_tanh(f1.x * k1.x + k1.y), silu_tanh(f1.y * k1.z + k1.w));
              o.z = pack_bf16(silu_tanh(f2.x * k2.x + k2.y), silu_tanh(f2.y * k2.z + k2.w));
              o.w = pack_bf16(silu_tanh(f3.x * k3.x + k3.y), silu_tanh(f3.y * k3.z + k3.w));
              *ptr = o;
            }
          }
        }
        fence_proxy_async_smem();
        named_bar_sync(1, kConsumers);
      }
      wgmma_fence();
      const uint64_t sdesc = desc0 + static_cast<uint64_t>(s * stage_u);
      for (int c = 0; c < p.kc; ++c) {
        const uint64_t adesc = sdesc + c * a_sub_u + wg_row_u;
        const uint64_t wdesc = sdesc + w_base_u + c * p.max_taps * w_sub_u;
        for (int tap = 0; tap < ti.ntaps; ++tap) {
#pragma unroll
          for (int kk = 0; kk < BK / 16; ++kk) {
            Wgmma<BN>::template ss<0, 0>(acc, adesc + ((tap * SW + kk * 32) >> 4),
                                         wdesc + tap * w_sub_u + ((kk * 32) >> 4), accumulate);
            accumulate = 1;
          }
        }
      }
      wgmma_commit();
      // one stage in flight: the previous one has been read -> hand its slot back
      wgmma_wait<1>();
      if (prev_s >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev_s]);
      }
      prev_s = s;
      if (++s == p.n_stages) { s = 0; ph ^= 1; }
    }
    wgmma_wait<0>();
    acc_fence(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[prev_s]);

    // ------------------------------------------------------------------------ epilogue
    if (do_stats && ti.b != cur_b) {
      if (cur_b >= 0) publish_stats(cur_b);
      cur_b = ti.b;
    }
    const int t_lo = ti.t0 + r0, t_hi = t_lo + 8;
    const bool ok_lo = t_lo < p.T, ok_hi = t_hi < p.T;
    const size_t col_off = static_cast<size_t>(ti.phase) * p.n_valid;
    const size_t off_lo = (static_cast<size_t>(ti.b) * p.T + (ok_lo ? t_lo : 0)) * p.ldo + col_off;
    const size_t off_hi = (static_cast<size_t>(ti.b) * p.T + (ok_hi ? t_hi : 0)) * p.ldo + col_off;
    const float* gate_row = p.gate ? p.gate + static_cast<size_t>(ti.b) * p.ld_gate : nullptr;
#pragma unroll
    for (int jb = 0; jb < BN / 8; ++jb) {
      if (ti.ch0 + jb * 8 >= p.n_valid) break;        // padded columns (n_valid % 8 == 0: uniform)
      const int ch = ti.ch0 + jb * 8 + cq;
      const float2 bb = p.bias ? make_float2(__ldg(p.bias + ch), __ldg(p.bias + ch + 1)) : make_float2(0.f, 0.f);
      const float2 gg = gate_row ? make_float2(__ldg(gate_row + ch), __ldg(gate_row + ch + 1)) : make_float2(1.f, 1.f);
      float v[4];
      v[0] = (acc[4 * jb + 0] + bb.x) * gg.x; v[1] = (acc[4 * jb + 1] + bb.y) * gg.y;
      v[2] = (acc[4 * jb + 2] + bb.x) * gg.x; v[3] = (acc[4 * jb + 3] + bb.y) * gg.y;
      if (p.out_fp32) {
        float* o = reinterpret_cast<float*>(p.out);
        if (ok_lo) *reinterpret_cast<float2*>(o + off_lo + ch) = make_float2(v[0], v[1]);
        if (ok_hi) *reinterpret_cast<float2*>(o + off_hi + ch) = make_float2(v[2], v[3]);
        continue;
      }
      if (p.residual) {
        if (ok_lo) {
          const float2 r = unpack_bf16(__ldg(reinterpret_cast<const unsigned int*>(p.residual + off_lo + ch)));
          v[0] += r.x; v[1] += r.y;
        }
        if (ok_hi) {
          const float2 r = unpack_bf16(__ldg(reinterpret_cast<const unsigned int*>(p.residual + off_hi + ch)));
          v[2] += r.x; v[3] += r.y;
        }
      }
      const uint32_t o_lo = pack_bf16(v[0], v[1]), o_hi = pack_bf16(v[2], v[3]);
      if (ok_lo) *reinterpret_cast<uint32_t*>(p.out + off_lo + ch) = o_lo;
      if (ok_hi) *reinterpret_cast<uint32_t*>(p.out + off_hi + ch) = o_hi;
      if (do_stats) {      // statistics of the ROUNDED values the next layer reads
        const float2 q_lo = ok_lo ? unpack_bf16(o_lo) : make_float2(0.f, 0.f);
        const float2 q_hi = ok_hi ? unpack_bf16(o_hi) : make_float2(0.f, 0.f);
        if (p.group_shift >= 3) {          // the 8-column block lies in one group: warp-uniform
          const int g = ch >> p.group_shift;
          acc_st.add(q_lo.x, g, s_part, warp, lane); acc_st.add(q_lo.y, g, s_part, warp, lane);
          acc_st.add(q_hi.x, g, s_part, warp, lane); acc_st.add(q_hi.y, g, s_part, warp, lane);
        } else {                           // groups narrower than 8 channels (rare): lane 0 adds
          const float q[4] = {q_lo.x, q_lo.y, q_hi.x, q_hi.y};   // every lane's values in lane order
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int cc = ch + (i & 1);
            const int g = p.group_shift >= 0 ? cc >> p.group_shift : cc / p.group_size;
            for (int src = 0; src < 32; ++src) {
              const float v = __shfl_sync(0xffffffffu, q[i], src);
              const int gs = __shfl_sync(0xffffffffu, g, src);
              if (lane == 0 && v != 0.f) { s_part[2 * gs][warp] += v; s_part[2 * gs + 1][warp] += v * v; }
            }
          }
        }
      }
    }
  }
  if (do_stats && cur_b >= 0) publish_stats(cur_b);
}

template <int BN, int SW, bool XF>
static int launch_gemm2(const adp_conv_gemm_args& a, cudaStream_t stream) {
  constexpr int BK = SW / 2;
  auto kernel = conv_gemm2_kernel<BN, SW, XF>;
  const int tiles_per_batch = (a.T + kBM - 1) / kBM;
  const bool up = a.up_factor > 1;
  const int max_taps = up ? 2 : a.ntaps;
  const int span = up ? 1 : a.ntaps - 1;
  const int a_rows = kBM + span;
  const int k_chunks = a.c_in / BK;

  Gemm2Params p;
  p.a_sub_bytes = (a_rows * SW + 1023) / 1024 * 1024;
  p.w_sub_bytes = (BN * SW + 1023) / 1024 * 1024;
  p.max_taps = max_taps;
  const int chunk_bytes = p.a_sub_bytes + max_taps * p.w_sub_bytes;

  // CTAs per SM: short-K tiles are bound by the epilogue, which overlaps another CTA's MMAs
  // when 2-3 CTAs share an SM; long-K tiles want deep rings of fat stages instead.
  const int w_iters = k_chunks * max_taps;
  int occ = 1;
  if (BN <= 64 && w_iters <= 8) occ = 3;
  else if (BN <= 128 && w_iters <= 12) occ = 2;
  if (XF && occ > (BN <= 64 ? 2 : 1)) occ = BN <= 64 ? 2 : 1;
  if (g_debug[3] > 0) occ = g_debug[3];
  static int static_smem = -1;
  if (static_smem < 0) {
    cudaFuncAttributes fa;
    ADP_CUDA(cudaFuncGetAttributes(&fa, kernel));
    static_smem = static_cast<int>(fa.sharedSizeBytes);
  }
  auto budget_of = [&](int o) {   // ring bytes per CTA: 1 KB reserved per CTA, 1 KB alignment slack
    int per_cta = kSmemPerSM / o - 1024;
    if (per_cta > kSmemPerBlock) per_cta = kSmemPerBlock;
    return per_cta - static_smem - 1024;
  };
  while (occ > 1 && budget_of(occ) < 2 * chunk_bytes) --occ;   // need >= 2 stages in the ring
  const int budget = budget_of(occ);
  // chunks per stage: amortise one mbarrier round trip over >= 8 MMAs where smem allows
  int kc = 1;
  while (kc * 2 <= 4 && k_chunks % (kc * 2) == 0 && kc * max_taps * (BK / 16) < 8 &&
         2 * (kc * 2) * chunk_bytes <= budget)
    kc *= 2;
  if (g_debug[5] > 0 && k_chunks % g_debug[5] == 0) kc = g_debug[5];
  p.kc = kc;
  p.k_stages = k_chunks / kc;
  p.stage_bytes = kc * chunk_bytes;
  int n_stages = budget / p.stage_bytes;
  if (n_stages > kMaxStages) n_stages = kMaxStages;
  if (n_stages < 2)
    return set_error("adp_conv_gemm: stage of %d bytes does not fit (BN=%d)", p.stage_bytes, BN);
  p.n_stages = n_stages;
  const size_t smem = static_cast<size_t>(n_stages) * p.stage_bytes + 1024;

  CUtensorMap tmA, tmW;
  {
    const uint64_t dims[3] = {(uint64_t)a.c_in, (uint64_t)a.T, (uint64_t)a.B};
    const uint64_t strides[2] = {(uint64_t)a.lda * 2, (uint64_t)a.T * a.lda * 2};
    const uint32_t box[3] = {(uint32_t)BK, (uint32_t)a_rows, 1};
    if (int e = make_tmap_bf16(&tmA, a.a, 3, dims, strides, box, SW)) return e;
  }
  {
    const uint64_t dims[2] = {(uint64_t)a.k_total, (uint64_t)a.phases * a.n_pad};
    const uint64_t strides[1] = {(uint64_t)a.k_total * 2};
    const uint32_t box[2] = {(uint32_t)BK, (uint32_t)BN};
    if (int e = make_tmap_bf16(&tmW, a.w, 2, dims, strides, box, SW)) return e;
  }

  static SmemAttrCache smem_cache;
  ADP_CUDA(ensure_dyn_smem(kernel, smem, smem_cache));
  int occ_hw = 1;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_hw, kernel, kGemmThreads, smem) != cudaSuccess ||
      occ_hw < 1)
    occ_hw = 1;
  if (occ > occ_hw) occ = occ_hw;

  p.out = static_cast<__nv_bfloat16*>(a.out);
  p.residual = static_cast<const __nv_bfloat16*>(a.residual);
  p.bias = a.bias;
  p.gate = a.gate;
  p.stats = a.stats;
  p.B = a.B;
  p.T = a.T;
  p.tiles_per_batch = tiles_per_batch;
  p.c_in = a.c_in;
  p.ldo = a.ldo;
  p.n_pad = a.n_pad;
  p.n_valid = a.n_valid;
  p.ntaps = a.ntaps;
  p.tap_off0 = a.tap_off[0];
  p.up_factor = a.up_factor;
  p.groups = a.stats ? a.groups : 0;
  p.group_size = a.stats ? a.n_valid / a.groups : 1;
  p.group_shift = -1;
  for (int sft = 0; sft < 16; ++sft)
    if ((1 << sft) == p.group_size) p.group_shift = sft;
  p.out_fp32 = a.out_fp32;
  p.ld_gate = a.ld_gate > 0 ? a.ld_gate : a.n_valid;
  p.n_tiles_n = a.phases * a.n_pad / BN;
  p.total_tiles = a.B * tiles_per_batch * p.n_tiles_n;
  p.a_rows = a_rows;
  p.early_w = g_debug[2];
  p.gn_stats = a.gn_stats;
  p.gn_gamma = a.gn_gamma;
  p.gn_beta = a.gn_beta;
  p.gn_eps = a.gn_eps;
  p.gn_groups = a.gn_groups > 0 ? a.gn_groups : 1;

  const int slots = occ * num_sms();
  int grid = p.total_tiles < slots ? p.total_tiles : slots;
  p.tiles_per_cta = (p.total_tiles + grid - 1) / grid;
  grid = (p.total_tiles + p.tiles_per_cta - 1) / p.tiles_per_cta;
  ADP_CUDA(launch_k(kernel, dim3(grid), dim3(kGemmThreads), smem, stream, tmA, tmW, p));
  ADP_LAUNCH_CHECK();
  return 0;
}

template <int SW>
static int dispatch_bn2(const adp_conv_gemm_args& a, int bn, cudaStream_t s) {
  if (a.gn_stats) {
    switch (bn) {
      case 16: return launch_gemm2<16, SW, true>(a, s);
      case 32: return launch_gemm2<32, SW, true>(a, s);
      case 64: return launch_gemm2<64, SW, true>(a, s);
      case 128: return launch_gemm2<128, SW, true>(a, s);
      case 256: return launch_gemm2<256, SW, true>(a, s);
    }
  }
  switch (bn) {
    case 16: return launch_gemm2<16, SW, false>(a, s);
    case 32: return launch_gemm2<32, SW, false>(a, s);
    case 64: return launch_gemm2<64, SW, false>(a, s);
    case 128: return launch_gemm2<128, SW, false>(a, s);
    case 256: return launch_gemm2<256, SW, false>(a, s);
  }
  return set_error("adp_conv_gemm: unsupported N tile %d", bn);
}

}  // namespace adp

namespace adp { extern int g_mid_threads; }

extern "C" int adp_debug_set(int key, int value) {
  if (key == 8) {            // threads per block of the thin-level ConvBlock kernels (128 or 256)
    if (value != 128 && value != 256) return adp::set_error("adp_debug_set: key 8 takes 128 or 256");
    adp::g_mid_threads = value;
    return 0;
  }
  if (key < 0 || key >= 8) return adp::set_error("adp_debug_set: bad key %d", key);
  adp::g_debug[key] = value;
  if (key == 6) adp::g_pdl = value;
  return 0;
}

extern "C" int adp_conv_gemm(const adp_conv_gemm_args* args, adp_stream_t stream) {
  using namespace adp;
  ADP_CHECK(args != nullptr, "adp_conv_gemm: null args");
  const adp_conv_gemm_args& a = *args;
  ADP_CHECK(a.a && a.w && a.out, "adp_conv_gemm: null a/w/out");
  ADP_CHECK(a.B > 0 && a.T > 0, "adp_conv_gemm: bad B=%d T=%d", a.B, a.T);
  ADP_CHECK(a.c_in >= 16 && a.c_in % 16 == 0, "adp_conv_gemm: c_in=%d must be a multiple of 16",
            a.c_in);
  ADP_CHECK(a.lda % 8 == 0 && a.ldo % 8 == 0 && a.k_total % 8 == 0 && a.lda >= a.c_in,
            "adp_conv_gemm: pitches lda=%d ldo=%d k_total=%d must be multiples of 8", a.lda, a.ldo,
            a.k_total);
  ADP_CHECK(a.n_valid > 0 && a.n_valid % 8 == 0 && a.n_valid <= a.n_pad && a.n_pad % 16 == 0,
            "adp_conv_gemm: n_valid=%d n_pad=%d", a.n_valid, a.n_pad);
  ADP_CHECK(a.phases >= 1, "adp_conv_gemm: phases=%d", a.phases);
  ADP_CHECK(a.ld_gate % 4 == 0, "adp_conv_gemm: ld_gate=%d must be a multiple of 4", a.ld_gate);
  if (a.up_factor > 1) {
    ADP_CHECK(a.phases == a.up_factor, "adp_conv_gemm: phases (%d) != up_factor (%d)", a.phases,
              a.up_factor);
    ADP_CHECK(a.k_total >= 2 * a.c_in, "adp_conv_gemm: upsample weights need 2 tap slots");
  } else {
    ADP_CHECK(a.ntaps >= 1 && a.ntaps <= 3 && a.phases == 1, "adp_conv_gemm: ntaps=%d phases=%d",
              a.ntaps, a.phases);
    ADP_CHECK(a.k_total >= a.ntaps * a.c_in, "adp_conv_gemm: k_total too small");
    for (int i = 1; i < a.ntaps; ++i)
      ADP_CHECK(a.tap_off[i] == a.tap_off[i - 1] + 1,
                "adp_conv_gemm: tap offsets must be consecutive and ascending");
  }
  if (a.out_fp32) {
    ADP_CHECK(!a.residual && !a.stats, "adp_conv_gemm: out_fp32 excludes residual/stats");
  }
  if (a.gn_stats) {
    ADP_CHECK(a.c_in <= 1024, "adp_conv_gemm: fused GroupNorm supports c_in <= 1024");
    ADP_CHECK(a.gn_gamma && a.gn_beta && a.gn_groups > 0 && a.c_in % a.gn_groups == 0 && a.lda == a.c_in,
              "adp_conv_gemm: fused GroupNorm needs gamma/beta, groups | c_in and a dense input");
  }
  if (a.stats) {
    ADP_CHECK(a.groups > 0 && a.groups <= kMaxGroups && a.n_valid % a.groups == 0,
              "adp_conv_gemm: groups=%d n_valid=%d (fused statistics handle <= %d groups)",
              a.groups, a.n_valid, kMaxGroups);
  }
  // N tile: persistent CTAs take care of SM fill; prefer 128 (W traffic dominates either way
  // and two accumulator buffers of 128 columns leave room for 2 CTAs/SM on short-K shapes)
  int bn = a.block_n;
  if (bn == 0) {
    const long m_tiles = (long)a.B * ((a.T + kBM - 1) / kBM);
    bn = 16;
    for (int cand = 128; cand >= 16; cand >>= 1) {
      if (a.n_pad % cand) continue;
      const long tiles = m_tiles * (a.phases * a.n_pad / cand);
      if (tiles >= 96 || cand <= 64) { bn = cand; break; }
    }
  }
  ADP_CHECK(a.n_pad % bn == 0, "adp_conv_gemm: N tile %d does not divide n_pad %d", bn, a.n_pad);
  cudaStream_t s = as_stream(stream);
  if (a.c_in % 64 == 0) return dispatch_bn2<128>(a, bn, s);
  if (a.c_in % 32 == 0) return dispatch_bn2<64>(a, bn, s);
  return dispatch_bn2<32>(a, bn, s);
}
