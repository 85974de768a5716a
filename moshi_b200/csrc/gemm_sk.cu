// Stream-K wgmma GEMM for the LM linears (see gemm_sk.cuh):  y[M][N] = epi(x[M][K] . w[N][K]^T), bf16 in,
// fp32 accumulate in registers, bf16 out.  M = concurrent sessions (<= 256), so the kernel is a weight
// streamer: every weight byte crosses HBM -> SMEM exactly once per launch and the whole chip pulls on it.
//
//   * Weights are repacked once at load into MMA-ready tiles: [n_tile][k_block][A][128 rows x 64 k] bf16,
//     each 16 KB tile already in the SWIZZLE_128B K-major shared-memory layout.  A pipeline stage is
//     therefore ONE contiguous `cp.async.bulk` (16 KB, or 32 KB for the gated MLP's gate+value pair).
//   * Work = the linear sequence of (n_tile, k_block) items, cut into equal contiguous ranges, one per
//     CTA (persistent, grid = #SMs): every SM streams the same number of bytes whatever N and K are
//     (out_proj has 32 n-tiles, the text head 250).  A tile whose k-range is cut across CTAs is
//     finished by whichever CTA arrives last: partial accumulators go to an L2-resident workspace and
//     are summed in CTA order, so the result is bit-reproducible and independent of arrival order.
//   * Warp roles (288 threads): warp 8 = bulk-copy/TMA producer, warps 0-7 = two consumer warpgroups
//     (wgmma with the weight tile as A, warpgroup w taking rows 64w..64w+63, the sessions as N), each running
//     the epilogue of its rows straight from the accumulator fragments.  The register accumulator bounds a
//     launch to 128 sessions (64 for the gated pair); run_linear runs larger batches as consecutive launches.
#include "gemm_sk.cuh"
#include "tc_prims.cuh"

namespace b200 {
namespace tc {

namespace {

constexpr int EPI_STORE = 0, EPI_RESADD = 1, EPI_GATE = 2;   // == lm::LIN_*
constexpr int BLOCK_ROWS = 128, BLOCK_K = 64, UMMA_K = 16;
constexpr int SK_MAX_NP = 128;     // sessions per launch of the stream-K kernel (register accumulators)
constexpr int SK_MAX_NP_GATE = 64; // ... of the gated MLP input (two accumulators)
constexpr int NUM_THREADS = 288;   // two consumer warpgroups + one producer warp
constexpr int PRODUCER_WARP = 8;
constexpr int TILE_BYTES = BLOCK_ROWS * BLOCK_K * 2;   // 16 KB
constexpr int MAX_STAGES = 12;
constexpr int MAX_DYN_SMEM = 220 * 1024;   // of the 227 KB a block may use; the kernels also have a few bytes of static shared memory

struct SkParams {
  int M, N, K, Mpad, gate_rows, out_rows;
  int stages, num_kb, n_tiles;
  int grid, whole_rounds, sk_tile0, sk_items;   // schedule: tiles [0, sk_tile0) whole, the rest stream-K items
  const uint8_t* wt;            // pre-tiled weights
  __nv_bfloat16* y; long long ldy;
  const __nv_bfloat16* res; long long ldr;
  float* ws;                    // partial slots: [2 * grid][A][Mpad][128] fp32
  int* counters;                // [n_tiles], zero between launches
  uint32_t stage_bytes;
  int stream_only;              // diagnostics: skip the MMAs (measures the copy pipeline alone)
  // int8 x int8 -> int32 (QLinear, utils/quantize.py:13-40): activations / weights are row-wise absmax int8, the
  // accumulator is dequantised as acc * sa[m] * sw[n] / 127^2; whole tiles only (exact integer sums)
  int i8; const float* sa; const float* sw;
};

using namespace tcp;
__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------
// schedule: every CTA first takes its share of the stream-K region (the n_tiles - W*G tiles that do
// not fill a whole round of the grid, cut by k-blocks into G equal contiguous item ranges), then W
// whole tiles (tile = w*G + c).  Partial accumulators are therefore written early in the kernel and
// their reduction overlaps the whole tiles.  All three warp roles walk the same segment list.
// ---------------------------------------------------------------------------------------------
struct Seg { int tile, kb0, kb1, slot; };   // slot: -1 = whole tile, else workspace slot of this partial

__device__ __forceinline__ int sk_begin(const SkParams& p, int c) { return (int)((long long)p.sk_items * c / p.grid); }
// CTA whose stream-K item range holds item j
__device__ __forceinline__ int sk_owner(const SkParams& p, int j) {
  int c = (int)((long long)j * p.grid / p.sk_items);
  while (c + 1 < p.grid && sk_begin(p, c + 1) <= j) ++c;
  while (c > 0 && sk_begin(p, c) > j) --c;
  return c;
}
__device__ __forceinline__ int seg_count(const SkParams& p, int c, int& n_sk) {
  const int a = sk_begin(p, c), b = sk_begin(p, c + 1);
  n_sk = a < b ? (b - 1) / p.num_kb - a / p.num_kb + 1 : 0;
  int n = n_sk;
  for (int w = 0; w < p.whole_rounds; ++w) n += (w * p.grid + c < p.sk_tile0) ? 1 : 0;
  return n;
}
__device__ __forceinline__ Seg seg_get(const SkParams& p, int c, int n_sk, int idx) {
  Seg s;
  if (idx < n_sk) {
    const int a = sk_begin(p, c), b = sk_begin(p, c + 1);
    const int first = a / p.num_kb;
    s.tile = p.sk_tile0 + first + idx;
    s.kb0 = idx == 0 ? a - first * p.num_kb : 0;
    s.kb1 = idx == n_sk - 1 ? (b - 1) % p.num_kb + 1 : p.num_kb;
    s.slot = (s.kb0 == 0 && s.kb1 == p.num_kb) ? -1 : 2 * c + (idx == 0 ? 0 : 1);
  } else {
    s.tile = (idx - n_sk) * p.grid + c;      // rounds are dense: a CTA without a tile in the last round has fewer segments
    s.kb0 = 0; s.kb1 = p.num_kb; s.slot = -1;
  }
  return s;
}

// accumulator word of output (m, weight row nw) as a float: fp32 bits, or int32 x the two row scales (int8 path)
__device__ __forceinline__ float acc_value(const SkParams& p, uint32_t bits, int m, int nw) {
  if (!p.i8) return __uint_as_float(bits);
  return (float)(int)bits * (p.sa[m] * p.sw[nw] * (1.f / 16129.f));
}

// sum of two partial accumulator words: fp32 values, or (int8 path) int32 bit patterns carried in float registers
__device__ __forceinline__ float part_add(bool i8, float a, float b) {
  return i8 ? __int_as_float(__float_as_int(a) + __float_as_int(b)) : a + b;
}

template <int EPI>
__device__ __forceinline__ float epilogue_value(const SkParams& p, float a, float b, int m, int n) {
  if (EPI == EPI_STORE) return a;
  if (EPI == EPI_RESADD) return __bfloat162float(p.res[(long long)m * p.ldr + n]) + bf16_round(a);
  const float g = bf16_round(a), u = bf16_round(b);
  return bf16_round(g / (1.f + expf(-g))) * u;     // bf16(silu(gate)) * value   (gating.py:18-20)
}

// The kernels below run 288 threads: warps 0-7 are two consumer warpgroups (wgmma into register accumulators, then the
// epilogue straight from the fragments; warpgroup w owns weight rows 64w..64w+63 of the 128-row tile), warp 8 is the
// bulk-copy / TMA producer.  NP = the session count padded to the wgmma width (the activation box has NP rows, rows beyond
// M are zero-filled by the TMA unit).
constexpr int CONSUMERS = 256;

// one k-block of MMAs of a consumer warpgroup: 4 k-steps of 32 bytes per row (16 bf16 or 32 int8)
template <int NP, int A>
__device__ __forceinline__ void sk_mma_kblock(uint32_t sa, uint32_t sb, int wg, bool i8, bool first, uint32_t (&d0)[NP / 2],
                                              uint32_t (&d1)[NP / 2]) {
  wg_fence();
#pragma unroll
  for (int k = 0; k < BLOCK_K / UMMA_K; ++k) {
    const uint64_t db = make_desc(sb + k * UMMA_K * 2);
    const uint32_t accum = (first && k == 0) ? 0u : 1u;
    const uint32_t a0 = sa + (uint32_t)wg * (TILE_BYTES / 2) + k * UMMA_K * 2;
    if (i8) {
      Wgmma<NP>::s8(d0, make_desc(a0), db, accum);
      if (A == 2) Wgmma<NP>::s8(d1, make_desc(a0 + TILE_BYTES), db, accum);
    } else {
      Wgmma<NP>::bf16(d0, make_desc(a0), db, accum);
      if (A == 2) Wgmma<NP>::bf16(d1, make_desc(a0 + TILE_BYTES), db, accum);
    }
  }
  wg_commit();
  wg_wait<0>();
  wg_hold(d0);
  if (A == 2) wg_hold(d1);
}

template <int EPI, int NP>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_sk_kernel(const __grid_constant__ CUtensorMap tmap_x, const SkParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ int s_last;
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;                 // SWIZZLE_128B tiles need 1024 B alignment
  const uint32_t bars = base + (uint32_t)p.stages * p.stage_bytes;
  const uint32_t full0 = bars, empty0 = bars + 8 * MAX_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int A_TILES = EPI == EPI_GATE ? 2 : 1;
  constexpr uint32_t a_bytes = A_TILES * TILE_BYTES;
  const int c = blockIdx.x;
  int n_sk = 0;
  const int n_seg = seg_count(p, c, n_sk);

  if (warp == PRODUCER_WARP && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_x) : "memory");
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, CONSUMERS / 32);   // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_trigger();

  if (warp == PRODUCER_WARP) {
    if (lane == 0) {
      // ===== producer: one contiguous bulk copy of the weight tile(s) + one TMA box of activations per k-block =====
      // Weights do not depend on the preceding kernel: the first `stages` weight tiles are requested before the
      // dependency wait, so under programmatic dependent launch the HBM stream starts while the producer of x
      // is still running.  The activation boxes (and everything the epilogue touches) come after pdl_wait.
      int s = 0; uint32_t ph = 0;
      int pre = 0;                                   // stages whose weight copy is already in flight
      {
        int ps = 0;
        for (int si = 0; si < n_seg && pre < p.stages; ++si) {
          const Seg sg = seg_get(p, c, n_sk, si);
          const uint8_t* src = p.wt + ((size_t)sg.tile * p.num_kb + sg.kb0) * a_bytes;
          for (int kb = sg.kb0; kb < sg.kb1 && pre < p.stages; ++kb, src += a_bytes, ++pre, ++ps) {
            mbar_expect_tx(full0 + 8 * ps, p.stage_bytes);
            bulk_load(base + (uint32_t)ps * p.stage_bytes, src, a_bytes, full0 + 8 * ps);
          }
        }
      }
      pdl_wait();
      int item = 0;
      for (int si = 0; si < n_seg; ++si) {
        const Seg sg = seg_get(p, c, n_sk, si);
        const uint8_t* src = p.wt + ((size_t)sg.tile * p.num_kb + sg.kb0) * a_bytes;
        for (int kb = sg.kb0; kb < sg.kb1; ++kb, src += a_bytes, ++item) {
          const uint32_t sa = base + (uint32_t)s * p.stage_bytes;
          if (item >= pre) {
            mbar_wait(empty0 + 8 * s, ph ^ 1u);
            mbar_expect_tx(full0 + 8 * s, p.stage_bytes);
            bulk_load(sa, src, a_bytes, full0 + 8 * s);
          }
          tma_load_2d(sa + a_bytes, &tmap_x, full0 + 8 * s, kb * (p.i8 ? 2 * BLOCK_K : BLOCK_K), 0);   // 128 bytes of K either way
          if (++s == p.stages) { s = 0; ph ^= 1u; }
        }
      }
    }
    return;
  }
  // ===== consumers: MMAs of a segment, then its epilogue from the accumulator fragments =====
  const int wg = warp >> 2, t = threadIdx.x & 127;
  const int et = threadIdx.x;                    // 0..255
  const size_t slot_floats = (size_t)A_TILES * BLOCK_ROWS * p.Mpad;
  uint32_t d0[NP / 2], d1[NP / 2];
  int s = 0; uint32_t ph = 0;
  pdl_wait();                                    // y / res / workspace / counters may still be in use by the predecessor
  for (int si = 0; si < n_seg; ++si) {
    const Seg sg = seg_get(p, c, n_sk, si);
    for (int kb = sg.kb0; kb < sg.kb1; ++kb) {
      mbar_wait(full0 + 8 * s, ph);
      const uint32_t sa = base + (uint32_t)s * p.stage_bytes;
      if (!p.stream_only) sk_mma_kblock<NP, A_TILES>(sa, sa + a_bytes, wg, p.i8 != 0, kb == sg.kb0, d0, d1);
      __syncwarp();
      if (lane == 0) mbar_arrive(empty0 + 8 * s);  // the smem stage is free once this warp's MMAs have read it
      if (++s == p.stages) { s = 0; ph ^= 1u; }
    }
    if (p.stream_only) continue;
    if (sg.slot < 0) {
#pragma unroll
      for (int i = 0; i < NP / 2; ++i) {
        const int row = 64 * wg + frag_row(t, i), m = frag_col(t, i);
        const int n = sg.tile * BLOCK_ROWS + row;
        if (m < p.M && n < p.out_rows) {
          float v;
          if (EPI == EPI_RESADD) v = __bfloat162float(p.res[(long long)m * p.ldr + n]) + bf16_round(acc_value(p, d0[i], m, n));
          else v = epilogue_value<EPI>(p, acc_value(p, d0[i], m, n), EPI == EPI_GATE ? acc_value(p, d1[i], m, p.gate_rows + n) : 0.f, m, n);
          p.y[(long long)m * p.ldy + n] = __float2bfloat16_rn(v);
        }
      }
    } else {
      // partial accumulator -> workspace slot, layout [A][128 rows][Mpad]
      float* ws = p.ws + (size_t)sg.slot * slot_floats;
#pragma unroll
      for (int i = 0; i < NP / 2; i += 2) {
        const int row = 64 * wg + frag_row(t, i), m = frag_col(t, i);
        if (m < p.Mpad) {
          __stcg(reinterpret_cast<float2*>(ws + (size_t)row * p.Mpad + m), make_float2(__uint_as_float(d0[i]), __uint_as_float(d0[i + 1])));
          if (EPI == EPI_GATE)
            __stcg(reinterpret_cast<float2*>(ws + (size_t)(BLOCK_ROWS + row) * p.Mpad + m),
                   make_float2(__uint_as_float(d1[i]), __uint_as_float(d1[i + 1])));
        }
      }
      // publish, count arrivals; the last arriver of this tile reduces all partials in CTA order
      __threadfence();
      named_bar(1, CONSUMERS);
      const int rel = sg.tile - p.sk_tile0;
      const int first_c = sk_owner(p, rel * p.num_kb), last_c = sk_owner(p, (rel + 1) * p.num_kb - 1);
      if (et == 0) {
        const int old = atomicAdd(p.counters + sg.tile, 1);
        const int last = old == last_c - first_c;
        s_last = last;
        if (last) p.counters[sg.tile] = 0;                     // ready for the next launch
      }
      named_bar(1, CONSUMERS);
      if (s_last) {
        __threadfence();
        const int row = et & 127, n = sg.tile * BLOCK_ROWS + row;
        const bool n_ok = n < p.out_rows;
        // 16 columns per pass (the two halves of the consumers take alternate passes): every contribution's 4 (gate: 8)
        // 16-byte loads are issued before the adds
        for (int m0 = (et >> 7) * 16; m0 < p.M; m0 += 32) {
          float av[16], bv[16];
#pragma unroll
          for (int j = 0; j < 16; ++j) { av[j] = 0.f; bv[j] = 0.f; }
#pragma unroll 2
          for (int cc = first_c; cc <= last_c; ++cc) {
            const int sl = 2 * cc + ((sk_begin(p, cc) / p.num_kb == rel) ? 0 : 1);
            const float4* w2 = reinterpret_cast<const float4*>(p.ws + (size_t)sl * slot_floats + (size_t)row * p.Mpad + m0);
            float4 v[4], u[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) v[j] = __ldcg(w2 + j);
            if (EPI == EPI_GATE) {
#pragma unroll
              for (int j = 0; j < 4; ++j) u[j] = __ldcg(w2 + (size_t)BLOCK_ROWS * p.Mpad / 4 + j);
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const bool q8 = p.i8 != 0;
              av[4 * j] = part_add(q8, av[4 * j], v[j].x); av[4 * j + 1] = part_add(q8, av[4 * j + 1], v[j].y);
              av[4 * j + 2] = part_add(q8, av[4 * j + 2], v[j].z); av[4 * j + 3] = part_add(q8, av[4 * j + 3], v[j].w);
              if (EPI == EPI_GATE) {
                bv[4 * j] = part_add(q8, bv[4 * j], u[j].x); bv[4 * j + 1] = part_add(q8, bv[4 * j + 1], u[j].y);
                bv[4 * j + 2] = part_add(q8, bv[4 * j + 2], u[j].z); bv[4 * j + 3] = part_add(q8, bv[4 * j + 3], u[j].w);
              }
            }
          }
          if (n_ok) {
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              const int m = m0 + j;
              if (m < p.M) {
                // fp32 zero and int32 zero share a bit pattern, so the accumulators start right on both paths
                const float a = acc_value(p, __float_as_uint(av[j]), m, n);
                const float b = EPI == EPI_GATE ? acc_value(p, __float_as_uint(bv[j]), m, p.gate_rows + n) : 0.f;
                p.y[(long long)m * p.ldy + n] = __float2bfloat16_rn(epilogue_value<EPI>(p, a, b, m, n));
              }
            }
          }
        }
      }
      named_bar(1, CONSUMERS);                   // s_last is reused by the next segment
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Cluster split-K ("ck") for the few-tile GEMMs at more than 32 sessions (out_proj / linear_out: 32 row tiles).
// A cluster of CS CTAs owns one 128-row tile; rank r streams k-blocks [r*kb_per, (r+1)*kb_per) into its own register
// accumulator.  The partials are then reduce-scattered over distributed shared memory: rank q is sent columns
// [q*Wc, (q+1)*Wc) of everybody's accumulator (st.shared::cluster into slot r of its receive buffer), one cluster barrier,
// and every rank sums its column block in rank order (deterministic) and runs the epilogue for it.  No global
// workspace, no atomics; CS x more SMs pull on the weights and the epilogue is spread over the cluster too.
// ---------------------------------------------------------------------------------------------
struct CkParams {
  int M, N, K, Mpad, CS, Wc, kb_per, num_kb, stages;
  const uint8_t* wt;
  __nv_bfloat16* y; long long ldy;
  const __nv_bfloat16* res; long long ldr;
  uint32_t stage_bytes;
  int i8; const float* sa; const float* sw;      // int8 operands: partials are exact int32, scaled once after the reduction
};

template <int EPI, int NP>      // EPI_STORE or EPI_RESADD
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_ck_kernel(const __grid_constant__ CUtensorMap tmap_x, const CkParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const uint32_t bars = base + (uint32_t)p.stages * p.stage_bytes;
  const uint32_t full0 = bars, empty0 = bars + 8 * MAX_STAGES;
  // receive buffer [CS][128 rows][Wc + 4] fp32 (rows padded against bank conflicts), after the barrier block
  const int ldw = p.Wc + 4;
  const uint32_t recv = (bars + 16 * MAX_STAGES + 15u) & ~15u;
  const float* recv_generic = reinterpret_cast<const float*>(smem_raw + (recv - raw));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x / p.CS, me = blockIdx.x - tile * p.CS;
  const int kb0 = me * p.kb_per, kb1 = min(p.num_kb, kb0 + p.kb_per);

  if (warp == PRODUCER_WARP && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_x) : "memory");
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, CONSUMERS / 32);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");   // waited for before the first remote store
  pdl_trigger();

  uint32_t d[NP / 2], dummy[NP / 2];
#pragma unroll
  for (int i = 0; i < NP / 2; ++i) d[i] = 0u;    // a rank without k-blocks contributes zeros
  if (warp == PRODUCER_WARP) {
    if (lane == 0) {
      // weights first (they do not depend on the preceding kernel), activations after the dependency wait
      const uint8_t* src = p.wt + ((size_t)tile * p.num_kb + kb0) * TILE_BYTES;
      const int n_items = kb1 - kb0;
      const int pre = n_items < p.stages ? n_items : p.stages;
      for (int i = 0; i < pre; ++i) {
        mbar_expect_tx(full0 + 8 * i, p.stage_bytes);
        bulk_load(base + (uint32_t)i * p.stage_bytes, src + (size_t)i * TILE_BYTES, TILE_BYTES, full0 + 8 * i);
      }
      pdl_wait();
      int s = 0; uint32_t ph = 0;
      for (int i = 0; i < n_items; ++i) {
        const uint32_t sa = base + (uint32_t)s * p.stage_bytes;
        if (i >= pre) {
          mbar_wait(empty0 + 8 * s, ph ^ 1u);
          mbar_expect_tx(full0 + 8 * s, p.stage_bytes);
          bulk_load(sa, src + (size_t)i * TILE_BYTES, TILE_BYTES, full0 + 8 * s);
        }
        tma_load_2d(sa + TILE_BYTES, &tmap_x, full0 + 8 * s, (kb0 + i) * (p.i8 ? 2 * BLOCK_K : BLOCK_K), 0);
        if (++s == p.stages) { s = 0; ph ^= 1u; }
      }
    }
    __syncwarp();
    asm volatile("barrier.cluster.wait.aligned;" ::: "memory");
  } else {
    const int wg = warp >> 2, t = threadIdx.x & 127;
    int s = 0; uint32_t ph = 0;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(full0 + 8 * s, ph);
      const uint32_t sa = base + (uint32_t)s * p.stage_bytes;
      sk_mma_kblock<NP, 1>(sa, sa + TILE_BYTES, wg, p.i8 != 0, kb == kb0, d, dummy);
      __syncwarp();
      if (lane == 0) mbar_arrive(empty0 + 8 * s);
      if (++s == p.stages) { s = 0; ph ^= 1u; }
    }
    pdl_wait();
    asm volatile("barrier.cluster.wait.aligned;" ::: "memory");   // every rank's receive buffer exists
    // column m of the accumulator goes to rank m / Wc, slot `me`, row `row`
#pragma unroll
    for (int i = 0; i < NP / 2; i += 2) {
      const int row = 64 * wg + frag_row(t, i), m = frag_col(t, i);
      if (m < p.Mpad) {
        const int q = m / p.Wc;
        const uint32_t dst = map_to_rank(recv + (uint32_t)(((me * BLOCK_ROWS + row) * ldw) + (m - q * p.Wc)) * 4u, (uint32_t)q);
        st_cluster_v2(dst, d[i], d[i + 1]);
      }
    }
  }
  cluster_sync_all();                          // every partial has landed in its owner's receive buffer
  if (warp != PRODUCER_WARP) {
    const int et = threadIdx.x, row = et & 127;
    const int n = tile * BLOCK_ROWS + row;
    const bool n_ok = n < p.N;
    for (int c0 = (et >> 7) * 8; c0 < p.Wc; c0 += 16) {
      float rv[8];
      if (EPI == EPI_RESADD) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int m = me * p.Wc + c0 + j;
          rv[j] = (m < p.M && n_ok) ? __bfloat162float(p.res[(long long)m * p.ldr + n]) : 0.f;
        }
      }
      float acc[8];
      if (p.i8) {                            // exact: the partials are int32 bit patterns
        int isum[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) isum[j] = 0;
        for (int r = 0; r < p.CS; ++r) {
          const int4 a = *reinterpret_cast<const int4*>(recv_generic + (size_t)(r * BLOCK_ROWS + row) * ldw + c0);
          const int4 b = *reinterpret_cast<const int4*>(recv_generic + (size_t)(r * BLOCK_ROWS + row) * ldw + c0 + 4);
          isum[0] += a.x; isum[1] += a.y; isum[2] += a.z; isum[3] += a.w;
          isum[4] += b.x; isum[5] += b.y; isum[6] += b.z; isum[7] += b.w;
        }
        const float swn = n_ok ? p.sw[n] : 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int m = me * p.Wc + c0 + j;
          acc[j] = m < p.M ? (float)isum[j] * (p.sa[m] * swn * (1.f / 16129.f)) : 0.f;     // same expression as acc_value()
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
        for (int r = 0; r < p.CS; ++r) {       // rank order: the sum does not depend on which rank does it
          const float4 a = *reinterpret_cast<const float4*>(recv_generic + (size_t)(r * BLOCK_ROWS + row) * ldw + c0);
          const float4 b = *reinterpret_cast<const float4*>(recv_generic + (size_t)(r * BLOCK_ROWS + row) * ldw + c0 + 4);
          acc[0] += a.x; acc[1] += a.y; acc[2] += a.z; acc[3] += a.w;
          acc[4] += b.x; acc[5] += b.y; acc[6] += b.z; acc[7] += b.w;
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int m = me * p.Wc + c0 + j;
        if (m < p.M && n_ok) {
          const float v = EPI == EPI_RESADD ? rv[j] + bf16_round(acc[j]) : acc[j];
          p.y[(long long)m * p.ldy + n] = __float2bfloat16_rn(v);
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// GEMV path for one or two sessions (up to four compiled).  With so few activation rows there is nothing for a tensor core to reuse: the GEMM
// above is then just a weight stream through the bulk-copy engine, so the same pre-tiled weights are read with LDG.128 here: a CTA owns one 128-row tile (tile pair for the gated MLP) over a k-range, a thread
// owns one 16-byte chunk position of four rows (the SWIZZLE_128B layout puts logical k-chunk (pos ^ (row & 7)) at position
// pos, and row & 7 is the same for a thread's four rows, so it multiplies all of them with the same 8 activations), two
// k-blocks of weights are in flight per thread (register double buffering), fp32 accumulation, 8-lane tree reduction at the
// end, split partials summed in split order by the last CTA to arrive (deterministic), same epilogues as the GEMM.
// ---------------------------------------------------------------------------------------------
constexpr int GV_THREADS = 256;
constexpr int GV_MAX_M = 4;                // compiled for up to 4 rows; used for <= 2 by default (b200_op_set_gemv_max_rows)
constexpr int GV_MAX_KBPS = 44;            // k-blocks per split: M * 44 * 64 bf16 of activations in shared memory (<= 22.5 KB)

struct GvParams {
  int M, N, K, out_rows, gate_rows, n_tiles, num_kb, S, kbps;
  const uint8_t* wt; const __nv_bfloat16* x; long long ldx;
  __nv_bfloat16* y; long long ldy; const __nv_bfloat16* res; long long ldr;
  float* ws; int* counters;               // partials [tile][split][A][M][128] fp32, arrival counters [tile] (zero between launches)
  const __nv_bfloat16* norm_alpha;        // NORM: x is the residual stream, the linear's input is rmsnorm(x, alpha) (transformer.py:45-58)
};

__device__ __forceinline__ void gv_unpack8(const uint4& v, float* f) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}

template <int EPI>
__device__ __forceinline__ void gv_store(const GvParams& p, int m, int n, float a, float b) {
  float v;
  if (EPI == EPI_STORE) v = a;
  else if (EPI == EPI_RESADD) v = __bfloat162float(p.res[(long long)m * p.ldr + n]) + bf16_round(a);
  else { const float g = bf16_round(a), u = bf16_round(b); v = bf16_round(g / (1.f + expf(-g))) * u; }
  p.y[(long long)m * p.ldy + n] = __float2bfloat16_rn(v);
}

template <int EPI, int M, bool NORM>
__global__ void __launch_bounds__(GV_THREADS) gemv_kernel(const GvParams p) {
  constexpr int A = EPI == EPI_GATE ? 2 : 1;
  extern __shared__ __align__(16) uint8_t gv_smem[];
  __nv_bfloat16* xs = reinterpret_cast<__nv_bfloat16*>(gv_smem);          // [M][kbps * 64]
  __shared__ int s_last;
  __shared__ float s_red[GV_THREADS / 32][M];
  __shared__ float s_rs[M];
  const int t = threadIdx.x;
  const int tile = blockIdx.x / p.S, sp = blockIdx.x - tile * p.S;
  const int kb0 = sp * p.kbps, kb1 = min(p.num_kb, kb0 + p.kbps);
  const int span = p.kbps * BLOCK_K;
  const int pos = t & 7, r0 = t >> 3;                 // rows r0, r0 + 32, r0 + 64, r0 + 96 of the tile
  const int kc = (pos ^ (r0 & 7)) * 8;                // the 8 activations this thread multiplies with, inside a k-block
  const uint4* wbase = reinterpret_cast<const uint4*>(p.wt + ((size_t)tile * p.num_kb + kb0) * (size_t)(A * TILE_BYTES)) + t;
  pdl_trigger();

  struct Group { uint4 w[A][4]; };
  auto load_group = [&](int i, Group& g) {            // k-block kb0 + i of this split
    const uint4* src = wbase + (size_t)i * (A * TILE_BYTES / 16);
#pragma unroll
    for (int a = 0; a < A; ++a)
#pragma unroll
      for (int j = 0; j < 4; ++j) g.w[a][j] = __ldg(src + a * (TILE_BYTES / 16) + j * GV_THREADS);
  };
  Group ga, gb;
  const int n_kb = kb1 - kb0;
  if (n_kb > 0) load_group(0, ga);                    // weights do not depend on the preceding kernel
  pdl_wait();
  if (NORM) {
    // RMSNorm folded into the staging (the row is 8 KB: every CTA takes the sum of squares of the whole row itself, which
    // saves a kernel and a dependency per linear): xn = bf16(x * (alpha * rsqrt(eps + mean x^2))), eps 1e-8 (rms_norm_f32)
    float ss[M];
#pragma unroll
    for (int m = 0; m < M; ++m) ss[m] = 0.f;
    for (int k = t * 8; k < p.K; k += GV_THREADS * 8) {
#pragma unroll
      for (int m = 0; m < M; ++m) {
        float f[8];
        gv_unpack8(*reinterpret_cast<const uint4*>(p.x + (long long)m * p.ldx + k), f);
#pragma unroll
        for (int e = 0; e < 8; ++e) ss[m] = fmaf(f[e], f[e], ss[m]);
      }
    }
#pragma unroll
    for (int m = 0; m < M; ++m) {
      float v = ss[m];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if ((t & 31) == 0) s_red[t >> 5][m] = v;
    }
    __syncthreads();
    if (t < M) {
      float tot = 0.f;
#pragma unroll
      for (int w = 0; w < GV_THREADS / 32; ++w) tot += s_red[w][t];
      s_rs[t] = rsqrtf(1e-8f + tot / (float)p.K);
    }
    __syncthreads();
  }
  // activations of this k-range -> shared memory (zero beyond K)
  for (int i = t * 8; i < M * span; i += GV_THREADS * 8) {
    const int m = i / span, k = kb0 * BLOCK_K + (i - m * span);
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (k < p.K) {
      v = *reinterpret_cast<const uint4*>(p.x + (long long)m * p.ldx + k);     // K % 8 == 0
      if (NORM) {
        float f[8], al[8];
        gv_unpack8(v, f);
        gv_unpack8(*reinterpret_cast<const uint4*>(p.norm_alpha + k), al);
        const float r = s_rs[m];
        __nv_bfloat162 o[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) o[e] = __floats2bfloat162_rn(f[2 * e] * (al[2 * e] * r), f[2 * e + 1] * (al[2 * e + 1] * r));
        v = *reinterpret_cast<const uint4*>(o);
      }
    }
    *reinterpret_cast<uint4*>(xs + i) = v;
  }
  __syncthreads();

  float acc[A][4][M];
#pragma unroll
  for (int a = 0; a < A; ++a)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int m = 0; m < M; ++m) acc[a][j][m] = 0.f;
  auto reduce_group = [&](int i, const Group& g) {
    float xv[M][8];
#pragma unroll
    for (int m = 0; m < M; ++m) gv_unpack8(*reinterpret_cast<const uint4*>(xs + m * span + i * BLOCK_K + kc), xv[m]);
#pragma unroll
    for (int a = 0; a < A; ++a)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float wf[8];
        gv_unpack8(g.w[a][j], wf);
#pragma unroll
        for (int m = 0; m < M; ++m)
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[a][j][m] = fmaf(wf[e], xv[m][e], acc[a][j][m]);
      }
  };
  for (int i = 0; i < n_kb; i += 2) {
    if (i + 1 < n_kb) load_group(i + 1, gb);
    reduce_group(i, ga);
    if (i + 1 < n_kb) {
      if (i + 2 < n_kb) load_group(i + 2, ga);
      reduce_group(i + 1, gb);
    }
  }
  // the 8 lanes of a row hold the 8 chunk positions of its k-blocks
#pragma unroll
  for (int a = 0; a < A; ++a)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int m = 0; m < M; ++m) {
        float v = acc[a][j][m];
        v += __shfl_xor_sync(0xffffffffu, v, 1);
        v += __shfl_xor_sync(0xffffffffu, v, 2);
        v += __shfl_xor_sync(0xffffffffu, v, 4);
        acc[a][j][m] = v;
      }
  if (p.S == 1) {
    if (pos == 0) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int n = tile * BLOCK_ROWS + r0 + 32 * j;
        if (n < p.out_rows) {
#pragma unroll
          for (int m = 0; m < M; ++m) gv_store<EPI>(p, m, n, acc[0][j][m], A == 2 ? acc[A - 1][j][m] : 0.f);
        }
      }
    }
    return;
  }
  float* slot = p.ws + ((size_t)tile * p.S + sp) * (size_t)(A * M * BLOCK_ROWS);
  if (pos == 0) {
#pragma unroll
    for (int a = 0; a < A; ++a)
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int m = 0; m < M; ++m) __stcg(slot + (a * M + m) * BLOCK_ROWS + r0 + 32 * j, acc[a][j][m]);
  }
  __threadfence();
  __syncthreads();
  if (t == 0) {
    const int old = atomicAdd(p.counters + tile, 1);
    s_last = old == p.S - 1;
    if (s_last) p.counters[tile] = 0;                // ready for the next launch
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const float* tbase = p.ws + (size_t)tile * p.S * (size_t)(A * M * BLOCK_ROWS);
  for (int idx = t; idx < M * BLOCK_ROWS; idx += GV_THREADS) {
    const int m = idx / BLOCK_ROWS, r = idx - m * BLOCK_ROWS;
    const int n = tile * BLOCK_ROWS + r;
    float a0 = 0.f, a1 = 0.f;
    for (int s2 = 0; s2 < p.S; ++s2) {               // split order: the sum does not depend on who arrives last
      const float* sl = tbase + (size_t)s2 * (A * M * BLOCK_ROWS);
      a0 += __ldcg(sl + m * BLOCK_ROWS + r);
      if (A == 2) a1 += __ldcg(sl + (M + m) * BLOCK_ROWS + r);
    }
    if (n < p.out_rows) gv_store<EPI>(p, m, n, a0, a1);
  }
}

template <int EPI, bool NORM>
static cudaError_t gv_launch_m(const cudaLaunchConfig_t& cfg, const GvParams& p) {
  switch (p.M) {
    case 1: return cudaLaunchKernelEx(&cfg, gemv_kernel<EPI, 1, NORM>, p);
    case 2: return cudaLaunchKernelEx(&cfg, gemv_kernel<EPI, 2, NORM>, p);
    case 3: return cudaLaunchKernelEx(&cfg, gemv_kernel<EPI, 3, NORM>, p);
    default: return cudaLaunchKernelEx(&cfg, gemv_kernel<EPI, 4, NORM>, p);
  }
}
template <int EPI>
static cudaError_t gv_launch(const cudaLaunchConfig_t& cfg, const GvParams& p) {
  return p.norm_alpha ? gv_launch_m<EPI, true>(cfg, p) : gv_launch_m<EPI, false>(cfg, p);
}

// load-time repack: w [rows][K] row-major -> tiles [n_tile][kb][A][128 x 64] in the SWIZZLE_128B layout
// (16-byte chunk c of row r sits at r*128 + ((c ^ (r & 7)) << 4)); rows/cols beyond the tensor are zero.
__global__ void pack_tiles_kernel(const __nv_bfloat16* __restrict__ w, uint4* __restrict__ out, int rows, int K, int n_tiles,
                                  int num_kb, int a_tiles, int gate_rows) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;        // one 16-byte chunk each
  const long long total = (long long)n_tiles * num_kb * a_tiles * (TILE_BYTES / 16);
  if (idx >= total) return;
  const int chunk = (int)(idx % (TILE_BYTES / 16));
  long long t = idx / (TILE_BYTES / 16);
  const int a = (int)(t % a_tiles); t /= a_tiles;
  const int kb = (int)(t % num_kb);
  const int tile = (int)(t / num_kb);
  const int r = chunk >> 3, cpos = chunk & 7;
  const int csrc = cpos ^ (r & 7);                               // logical chunk stored at this position
  const int limit = a_tiles == 2 ? gate_rows : rows;
  const int rr = tile * BLOCK_ROWS + r;
  const int k = kb * BLOCK_K + csrc * 8;
  uint4 v = make_uint4(0u, 0u, 0u, 0u);
  if (rr < limit && k < K) v = *reinterpret_cast<const uint4*>(w + (long long)(rr + a * gate_rows) * K + k);
  out[idx] = v;
}

// ---- int8 quantisation (QLinear: bnb int8_vectorwise_quant, utils/quantize.py:16-20,38) -----------------------------------
// row-wise absmax of w[rows][K] taken on the fp16 values (the reference quantises weight.to(float16))
__global__ void row_absmax_f16_kernel(const __nv_bfloat16* __restrict__ w, float* __restrict__ out, int rows, int K) {
  const int row = blockIdx.x;
  float mx = 0.f;
  for (int k = threadIdx.x; k < K; k += blockDim.x)
    mx = fmaxf(mx, fabsf(__half2float(__float2half_rn(__bfloat162float(w[(long long)row * K + k])))));
  __shared__ float red[32];
  mx = warp_max(mx);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < (int)(blockDim.x + 31) / 32; ++i) t = fmaxf(t, red[i]);
    out[row] = t;
  }
}
__device__ __forceinline__ int quant_i8(float v, float inv) {           // round(v * 127 / absmax), ties to even (torch.round)
  int q = __float2int_rn(v * inv);
  return q > 127 ? 127 : (q < -127 ? -127 : q);
}
// w [rows][K] -> int8 tiles [n_tile][kb][A][128 rows x 128 k] in the SWIZZLE_128B layout (one 16-byte chunk = 16 k per thread)
__global__ void pack_tiles_i8_kernel(const __nv_bfloat16* __restrict__ w, const float* __restrict__ absmax, uint4* __restrict__ out,
                                     int rows, int K, int n_tiles, int num_kb, int a_tiles, int gate_rows) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)n_tiles * num_kb * a_tiles * (TILE_BYTES / 16);
  if (idx >= total) return;
  const int chunk = (int)(idx % (TILE_BYTES / 16));
  long long t = idx / (TILE_BYTES / 16);
  const int a = (int)(t % a_tiles); t /= a_tiles;
  const int kb = (int)(t % num_kb);
  const int tile = (int)(t / num_kb);
  const int r = chunk >> 3, cpos = chunk & 7;
  const int csrc = cpos ^ (r & 7);
  const int limit = a_tiles == 2 ? gate_rows : rows;
  const int rr = tile * BLOCK_ROWS + r;
  const int k0 = kb * 128 + csrc * 16;
  uint32_t words[4] = {0u, 0u, 0u, 0u};
  if (rr < limit) {
    const long long srow = (long long)(rr + a * gate_rows);
    const float am = absmax[srow];
    const float inv = am > 0.f ? 127.f / am : 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int k = k0 + j;
      int q = 0;
      if (k < K) q = quant_i8(__half2float(__float2half_rn(__bfloat162float(w[srow * K + k]))), inv);
      words[j >> 2] |= (uint32_t)(q & 0xFF) << (8 * (j & 3));
    }
  }
  out[idx] = make_uint4(words[0], words[1], words[2], words[3]);
}
// already-quantised weights (a QLinear's CB as stored in model.q8.safetensors): q int8 [rows][K] -> the same int8 tiles
__global__ void pack_tiles_i8_pre_kernel(const int8_t* __restrict__ q, uint4* __restrict__ out, int rows, int K, int n_tiles, int num_kb,
                                         int a_tiles, int gate_rows) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)n_tiles * num_kb * a_tiles * (TILE_BYTES / 16);
  if (idx >= total) return;
  const int chunk = (int)(idx % (TILE_BYTES / 16));
  long long t = idx / (TILE_BYTES / 16);
  const int a = (int)(t % a_tiles); t /= a_tiles;
  const int kb = (int)(t % num_kb);
  const int tile = (int)(t / num_kb);
  const int r = chunk >> 3, cpos = chunk & 7;
  const int csrc = cpos ^ (r & 7);
  const int limit = a_tiles == 2 ? gate_rows : rows;
  const int rr = tile * BLOCK_ROWS + r;
  const int k0 = kb * 128 + csrc * 16;
  uint32_t words[4] = {0u, 0u, 0u, 0u};
  if (rr < limit) {
    const long long srow = (long long)(rr + a * gate_rows);
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int k = k0 + j;
      const int v = k < K ? (int)q[srow * K + k] : 0;
      words[j >> 2] |= (uint32_t)(v & 0xFF) << (8 * (j & 3));
    }
  }
  out[idx] = make_uint4(words[0], words[1], words[2], words[3]);
}
// activations: x [M][K] bf16 (row stride ldx) -> xq int8 [M][K], sa[m] = absmax of the row
__global__ void __launch_bounds__(256) quantize_rows_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, int8_t* __restrict__ xq,
                                                           float* __restrict__ sa, int K) {
  const int row = blockIdx.x;
  const __nv_bfloat16* xr = x + (long long)row * ldx;
  float mx = 0.f;
  pdl_wait();          // x comes from the preceding kernel; xq / sa may still be read by the GEMM before that one
  pdl_trigger();       // the GEMM that follows starts streaming its weight tiles while the rows are quantised
  for (int k = threadIdx.x * 8; k < K; k += 256 * 8) {
    const uint4 v = *reinterpret_cast<const uint4*>(xr + k);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __bfloat1622float2(h[i]);
      mx = fmaxf(mx, fmaxf(fabsf(f.x), fabsf(f.y)));
    }
  }
  __shared__ float red[8];
  mx = warp_max(mx);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  float am = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) am = fmaxf(am, red[i]);
  if (threadIdx.x == 0) sa[row] = am;
  const float inv = am > 0.f ? 127.f / am : 0.f;
  for (int k = threadIdx.x * 8; k < K; k += 256 * 8) {
    const uint4 v = *reinterpret_cast<const uint4*>(xr + k);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
    uint32_t w0 = 0u, w1 = 0u;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __bfloat1622float2(h[i]);
      const uint32_t a = (uint32_t)(quant_i8(f.x, inv) & 0xFF), b = (uint32_t)(quant_i8(f.y, inv) & 0xFF);
      if (i < 2) w0 |= (a | (b << 8)) << (16 * i);
      else w1 |= (a | (b << 8)) << (16 * (i - 2));
    }
    *reinterpret_cast<uint2*>(xq + (long long)row * K + k) = make_uint2(w0, w1);
  }
}

int g_gemv_max_m = 2;            // b200_op_set_gemv_max_rows (0..4): 0 sends every batch size through the tensor-core GEMM
bool g_attr_set = false;

template <class F>
static cudaError_t smem_attr(F* kernel) {
  return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_DYN_SMEM);
}
template <int NP>
static int set_smem_attrs_np() {
  B200_CUDA(smem_attr(gemm_sk_kernel<EPI_STORE, NP>));
  B200_CUDA(smem_attr(gemm_sk_kernel<EPI_RESADD, NP>));
  B200_CUDA(smem_attr(gemm_sk_kernel<EPI_GATE, (NP < SK_MAX_NP_GATE ? NP : SK_MAX_NP_GATE)>));
  return B200_OK;
}
static int set_smem_attrs() {
  B200_TRY(set_smem_attrs_np<16>());
  B200_TRY(set_smem_attrs_np<32>());
  B200_TRY(set_smem_attrs_np<64>());
  B200_TRY(set_smem_attrs_np<128>());
  B200_CUDA(smem_attr(gemm_ck_kernel<EPI_STORE, 64>));
  B200_CUDA(smem_attr(gemm_ck_kernel<EPI_STORE, 128>));
  B200_CUDA(smem_attr(gemm_ck_kernel<EPI_STORE, 256>));
  B200_CUDA(smem_attr(gemm_ck_kernel<EPI_RESADD, 64>));
  B200_CUDA(smem_attr(gemm_ck_kernel<EPI_RESADD, 128>));
  B200_CUDA(smem_attr(gemm_ck_kernel<EPI_RESADD, 256>));
  return B200_OK;
}

}  // namespace

int linear_init() {
  if (!g_attr_set) {
    B200_TRY(set_smem_attrs());
    g_attr_set = true;
  }
  return B200_OK;
}

int linear_prepare() {
  B200_TRY(ns_init());
  return linear_init();
}

int sk_gemv_max_m() { return g_gemv_max_m; }

int sk_set_gemv_max_m(int max_m) {
  const int before = g_gemv_max_m;
  g_gemv_max_m = max_m < 0 ? 0 : max_m > GV_MAX_M ? GV_MAX_M : max_m;
  return before;
}

size_t sk_packed_bytes(int N, int K, int epi, int gate_rows) {
  const int a = epi == EPI_GATE ? 2 : 1;
  const int rows = epi == EPI_GATE ? gate_rows : N;
  return (size_t)((rows + BLOCK_ROWS - 1) / BLOCK_ROWS) * ((K + BLOCK_K - 1) / BLOCK_K) * a * TILE_BYTES;
}

int sk_pack_weights(const __nv_bfloat16* w, void* out, int N, int K, int epi, int gate_rows, cudaStream_t stream) {
  const int a = epi == EPI_GATE ? 2 : 1;
  const int rows = epi == EPI_GATE ? gate_rows : N;
  const int n_tiles = (rows + BLOCK_ROWS - 1) / BLOCK_ROWS, num_kb = (K + BLOCK_K - 1) / BLOCK_K;
  if (K % 8) B200_FAIL(B200_ERR_SHAPE, "sk_pack_weights: K must be a multiple of 8");
  const long long total = (long long)n_tiles * num_kb * a * (TILE_BYTES / 16);
  pack_tiles_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(w, static_cast<uint4*>(out), epi == EPI_GATE ? 2 * gate_rows : N,
                                                                       K, n_tiles, num_kb, a, epi == EPI_GATE ? gate_rows : 0);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return check_launch("pack_tiles");
}

size_t sk_packed_bytes_i8(int N, int K, int epi, int gate_rows) {
  const int a = epi == EPI_GATE ? 2 : 1;
  const int rows = epi == EPI_GATE ? gate_rows : N;
  return (size_t)((rows + BLOCK_ROWS - 1) / BLOCK_ROWS) * ((K + 127) / 128) * a * TILE_BYTES;
}

int sk_quant_pack_weights(const __nv_bfloat16* w, void* out_tiles, float* out_scales, int N, int K, int epi, int gate_rows,
                          cudaStream_t stream) {
  if (K % 16) B200_FAIL(B200_ERR_SHAPE, "sk_quant_pack_weights: K must be a multiple of 16");
  const int a = epi == EPI_GATE ? 2 : 1;
  const int w_rows = epi == EPI_GATE ? 2 * gate_rows : N;
  const int rows = epi == EPI_GATE ? gate_rows : N;
  const int n_tiles = (rows + BLOCK_ROWS - 1) / BLOCK_ROWS, num_kb = (K + 127) / 128;
  row_absmax_f16_kernel<<<w_rows, 256, 0, stream>>>(w, out_scales, w_rows, K);
  const long long total = (long long)n_tiles * num_kb * a * (TILE_BYTES / 16);
  pack_tiles_i8_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(w, out_scales, static_cast<uint4*>(out_tiles), w_rows, K,
                                                                           n_tiles, num_kb, a, epi == EPI_GATE ? gate_rows : 0);
  g_launches.fetch_add(2, std::memory_order_relaxed);
  return check_launch("quant_pack_tiles");
}

int sk_pack_weights_i8(const int8_t* q, void* out_tiles, int N, int K, int epi, int gate_rows, cudaStream_t stream) {
  if (K % 16) B200_FAIL(B200_ERR_SHAPE, "sk_pack_weights_i8: K must be a multiple of 16");
  const int a = epi == EPI_GATE ? 2 : 1;
  const int w_rows = epi == EPI_GATE ? 2 * gate_rows : N;
  const int rows = epi == EPI_GATE ? gate_rows : N;
  const int n_tiles = (rows + BLOCK_ROWS - 1) / BLOCK_ROWS, num_kb = (K + 127) / 128;
  const long long total = (long long)n_tiles * num_kb * a * (TILE_BYTES / 16);
  pack_tiles_i8_pre_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(q, static_cast<uint4*>(out_tiles), w_rows, K, n_tiles, num_kb,
                                                                              a, epi == EPI_GATE ? gate_rows : 0);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return check_launch("pack_tiles_i8_pre");
}

int sk_quantize_rows(const __nv_bfloat16* x, long long ldx, void* xq, float* sa, int M, int K, cudaStream_t stream, int pdl) {
  if (K % 8 || ldx % 8) B200_FAIL(B200_ERR_SHAPE, "sk_quantize_rows: K and the row stride must be multiples of 8");
  return launch("quantize_rows", quantize_rows_kernel, dim3((unsigned)M), dim3(256), 0, stream, LaunchOpts{pdl}, x, ldx,
                static_cast<int8_t*>(xq), sa, K);
}

size_t sk_workspace_bytes(int max_M) {
  const int Mpad = ((max_M + 15) / 16) * 16;
  return (size_t)2 * SK_MAX_GRID * 2 * Mpad * BLOCK_ROWS * 4;  // 2 slots per CTA, gate + value accumulators
}

bool sk_supported(int M, int N, int K, int epi) {
  (void)N; (void)epi;
  return M >= 1 && M <= 256 && K >= 8 && K % 8 == 0;
}

namespace {

int add_block(LinearPlan& P, const LinearBlock& b) {
  if (P.n_blocks == LINEAR_MAX_BLOCKS) B200_FAIL(B200_ERR_SHAPE, "linear plan: more than %d launches", LINEAR_MAX_BLOCKS);
  P.blocks[P.n_blocks++] = b;
  return B200_OK;
}

// The LM's choice of NS unit and K-split for a shape:
//   * >= 40 pairs of tiles (in_proj 48, the gated MLP's input 88, the text head 125): N = 256 units, two K-splits while both CTAs
//     of every unit are resident at once (in_proj: 96 CTAs), else one;
//   * fewer (out_proj / linear_out: 32 tiles, depformer_in: 64): single-tile units (N = 128) so that more SMs pull on the
//     weights, K cut over the largest power of two <= 4 that keeps the grid resident (32 x 4, 64 x 2 = 128 CTAs).
void ns_default_plan(int n_tiles, int num_kb, int epi, int sms, int* unit_tiles, int* cs) {
  if (epi == EPI_GATE) { *unit_tiles = 2; *cs = 1; return; }
  const int pairs = (n_tiles + 1) / 2;
  if (pairs >= 40) {
    *unit_tiles = 2;
    *cs = (2 * pairs <= sms && num_kb >= 8) ? 2 : 1;
    return;
  }
  *unit_tiles = 1;
  int c = 1;
  while (c < 4 && n_tiles * c * 2 <= sms && num_kb / (c * 2) >= 4) c *= 2;
  *cs = c;
}

// NS over rows [m0, m0 + M): the accumulator [128 sessions x 256 weight rows] lives in the registers of the two consumer
// warpgroups, so above 128 sessions the batch runs as two launches (each streams the weights again)
int plan_ns(LinearPlan& P, int m0, int M, int sms, int cluster, int unit_tiles) {
  if (M > 128) {
    B200_TRY(plan_ns(P, m0, 128, sms, cluster, unit_tiles));
    return plan_ns(P, m0 + 128, M - 128, sms, cluster, unit_tiles);
  }
  const int epi = P.epi;
  const int out_rows = epi == EPI_GATE ? P.gate_rows : P.N;
  const int n_tiles = (out_rows + BLOCK_ROWS - 1) / BLOCK_ROWS;
  const int num_kb = (P.K + BLOCK_K - 1) / BLOCK_K;
  int def_ut = 2, def_cs = 1;
  ns_default_plan(n_tiles, num_kb, epi, sms, &def_ut, &def_cs);
  if (unit_tiles == 0) unit_tiles = cluster > 0 ? 2 : def_ut;
  const int ut = (unit_tiles == 1 && epi != EPI_GATE) ? 1 : 2;
  const uint32_t stage_bytes = (uint32_t)ut * TILE_BYTES + (uint32_t)NS_A_BYTES;
  const int n_units = (epi == EPI_GATE || ut == 1) ? n_tiles : (n_tiles + 1) / 2;
  int cs = cluster > 0 ? cluster : def_cs;
  if (epi == EPI_GATE) cs = 1;
  if (cs > NS_MAX_CS) cs = NS_MAX_CS;
  if (cs > num_kb) cs = num_kb;
  const int kb_per = (num_kb + cs - 1) / cs;
  // receive buffer rows: the widest column share + 4, an odd number of 16-byte units (conflict-free float4 rows)
  int wmax = 0;
  for (int q = 0; q < cs; ++q) {
    const int a = q >= cs ? 256 : ((256 * q / cs) >> 4) << 4, b = q + 1 >= cs ? 256 : ((256 * (q + 1) / cs) >> 4) << 4;
    if (b - a > wmax) wmax = b - a;
  }
  int ldw = wmax + 4;
  if (((ldw / 4) & 1) == 0) ldw += 4;
  int stages = (200 * 1024) / (int)stage_bytes;
  if (stages > NS_MAX_STAGES) stages = NS_MAX_STAGES;
  if (stages > kb_per && kb_per >= 2) stages = kb_per;
  if (stages < 2) stages = 2;
  const size_t recv_bytes = cs > 1 ? (size_t)cs * 128 * ldw * 4 : 0;
  while ((size_t)stages * stage_bytes < recv_bytes) ++stages;          // the ring doubles as the receive buffer
  if (stages > NS_MAX_STAGES || (size_t)stages * stage_bytes > 204 * 1024)
    B200_FAIL(B200_ERR_SHAPE, "ns GEMM: the receive buffer of a %d-way split does not fit", cs);
  LinearBlock b;
  memset(&b, 0, sizeof(b));
  b.kernel = LK_NS; b.m0 = m0; b.rows = M;
  b.grid = n_units * cs; b.cluster = cs; b.smem = (int)((size_t)stages * stage_bytes + 1024 + 16 * NS_MAX_STAGES + 64);
  b.stages = stages; b.stage_bytes = (int)stage_bytes; b.np = 128; b.kb_per = kb_per; b.unit_tiles = ut; b.ldw = ldw;
  return add_block(P, b);
}

// the kernel and launch parameters for rows [m0, m0 + M); batches larger than one swap-AB launch holds recurse per block of rows
int plan_rows(LinearPlan& P, int m0, int M, bool norm, bool ld_aligned, int sms, int gemv_max_m, const LinearForce& f) {
  const int N = P.N, K = P.K, epi = P.epi, gate_rows = P.gate_rows;
  const bool i8 = P.i8 != 0;
  if (f.kernel == LK_NS) return plan_ns(P, m0, M, sms, f.ns_splits, f.ns_unit_tiles);
  LinearBlock b;
  memset(&b, 0, sizeof(b));
  b.m0 = m0; b.rows = M;
  // one to four sessions: stream the tiles with plain loads on the CUDA cores (no bulk-copy engine ceiling)
  if (!i8 && M <= GV_MAX_M && f.sk_grid == 0 && f.ck_cluster == 0 && !f.stream_only && gemv_max_m >= M) {
    const int out_rows = epi == EPI_GATE ? gate_rows : N;
    const int n_tiles = (out_rows + BLOCK_ROWS - 1) / BLOCK_ROWS;
    const int num_kb = (K + BLOCK_K - 1) / BLOCK_K;
    if (n_tiles > SK_MAX_TILES) B200_FAIL(B200_ERR_SHAPE, "gemv: more than %d row tiles", SK_MAX_TILES);
    const int A = epi == EPI_GATE ? 2 : 1;
    // enough CTAs for ~4 per SM, every CTA streams at least 4 k-blocks, the activation slice fits in shared memory
    int S = (4 * sms + n_tiles - 1) / n_tiles;
    if (S > num_kb / 4) S = num_kb / 4;
    if (S < 1) S = 1;
    const int s_min = (num_kb + GV_MAX_KBPS - 1) / GV_MAX_KBPS;
    if (S < s_min) S = s_min;
    const size_t slot_bytes = (size_t)A * M * BLOCK_ROWS * 4;
    while (S > s_min && (size_t)n_tiles * S * slot_bytes > sk_workspace_bytes(M)) --S;
    b.kbps = (num_kb + S - 1) / S;
    b.S = (num_kb + b.kbps - 1) / b.kbps;
    if ((size_t)n_tiles * b.S * slot_bytes <= sk_workspace_bytes(M)) {
      b.kernel = LK_GEMV;
      b.grid = n_tiles * b.S;
      b.smem = M * b.kbps * BLOCK_K * 2;
      P.norm_folded = norm ? 1 : 0;
      return add_block(P, b);
    }
    b.kbps = b.S = 0;
  }
  // 33..256 sessions: activations as the A operand, two weight tiles (N = 256) per wgmma (gemm_ns.cu)
  if (f.kernel != LK_SK && !i8 && M > 32 && f.sk_grid == 0 && f.ck_cluster == 0 && !f.stream_only && ld_aligned)
    return plan_ns(P, m0, M, sms, 0, 0);
  // more than 32 sessions and few row tiles: a cluster of CTAs per tile, split along K, reduced over DSMEM
  if (i8 && K % 16) B200_FAIL(B200_ERR_SHAPE, "int8 GEMM: K must be a multiple of 16 and both scale vectors given");
  if (epi != EPI_GATE && f.sk_grid == 0 && M > 32) {
    const int n_tiles = (N + BLOCK_ROWS - 1) / BLOCK_ROWS, num_kb = i8 ? (K + 127) / 128 : (K + BLOCK_K - 1) / BLOCK_K;
    int cs = 1;
    while (cs < 8 && n_tiles * cs * 2 <= sms && num_kb / (cs * 2) >= 4) cs *= 2;
    if (f.ck_cluster > 0) cs = f.ck_cluster;
    if (cs > 1) {
      const int quantum = 8 * cs < 16 ? 16 : 8 * cs;       // wgmma N is a multiple of 16; every rank owns whole 8-column groups
      const int Mpad = ((M + quantum - 1) / quantum) * quantum;
      const int Wc = Mpad / cs;
      int np = 64;                                          // wgmma width: the padded session count (M > 32 here)
      while (np < Mpad) np <<= 1;
      if (Mpad <= 256 && Wc <= 64) {
        const int kb_per = (num_kb + cs - 1) / cs;
        const uint32_t stage_bytes = (uint32_t)(TILE_BYTES + np * BLOCK_K * 2);          // 128 bytes of K per row, bf16 or int8
        const size_t recv_bytes = (size_t)cs * BLOCK_ROWS * (Wc + 4) * 4;
        int stages = (int)((200 * 1024 - recv_bytes) / stage_bytes);
        if (stages > MAX_STAGES) stages = MAX_STAGES;
        if (stages > kb_per) stages = kb_per;
        if (stages >= 2) {
          b.kernel = LK_CK;
          b.grid = n_tiles * cs; b.cluster = cs;
          b.smem = (int)((size_t)stages * stage_bytes + 1024 + 16 * MAX_STAGES + 16 + recv_bytes);
          b.stages = stages; b.stage_bytes = (int)stage_bytes; b.np = np; b.Mpad = Mpad; b.kb_per = kb_per; b.Wc = Wc;
          return add_block(P, b);
        }
      }
    }
  }
  // The accumulator of a CTA lives in the registers of its two consumer warpgroups: at most 128 sessions per launch (64 for
  // the gated MLP's two accumulators).  Larger batches run as consecutive launches over blocks of sessions, each streaming
  // the weights again.
  const int max_np = epi == EPI_GATE ? SK_MAX_NP_GATE : SK_MAX_NP;
  if (M > max_np) {
    for (int mm = 0; mm < M; mm += max_np)
      B200_TRY(plan_rows(P, m0 + mm, M - mm < max_np ? M - mm : max_np, false, ld_aligned, sms, gemv_max_m, f));
    return B200_OK;
  }
  const int out_rows = epi == EPI_GATE ? gate_rows : N;
  const int Mpad = ((M + 15) / 16) * 16;
  const int num_kb = i8 ? (K + 127) / 128 : (K + BLOCK_K - 1) / BLOCK_K;      // a k-block is 128 bytes of K per row
  const int n_tiles = (out_rows + BLOCK_ROWS - 1) / BLOCK_ROWS;
  if (n_tiles > 1024) B200_FAIL(B200_ERR_SHAPE, "sk GEMM: more than 1024 row tiles");
  int grid = f.sk_grid > 0 ? f.sk_grid : sms;
  if (grid > SK_MAX_GRID) grid = SK_MAX_GRID;
  if (grid > n_tiles * num_kb) grid = n_tiles * num_kb;
  // a CTA should stream at least ~8 k-blocks (128-256 KB): below that the per-CTA set-up and the partial exchange dominate
  if (f.sk_grid == 0 && grid > (n_tiles * num_kb) / 8) grid = (n_tiles * num_kb) / 8 > 0 ? (n_tiles * num_kb) / 8 : 1;
  // Cutting a tile into S pieces moves S fp32 partials of [128 x Mpad] through L2 (written + read back): allow it
  // only while that stays under half of the tile's weight bytes, i.e. S <= 8 * num_kb / Mpad.
  int s_max = (8 * num_kb) / Mpad;      // int8 partials are int32 and add exactly
  // with more than 32 sessions the publish / count / re-read protocol costs more than the idle SMs it recovers, so tiles stay
  // whole there (a forced grid cuts them at every M: the parity tests exercise the tile-cutting path so)
  if (Mpad > 32 && f.sk_grid == 0) s_max = 1;
  if (s_max < 1) s_max = 1;
  if (n_tiles < grid && (long long)n_tiles * s_max < grid) grid = n_tiles * s_max;   // fewer CTAs, fewer pieces
  // whole rounds of the grid, then the remainder as a stream-K region shared by all CTAs
  b.kernel = LK_SK;
  b.grid = grid;
  b.whole_rounds = n_tiles / grid;
  int rem = n_tiles - b.whole_rounds * grid;
  const bool split = rem > 0 && s_max > 1 && rem * 8 < grid * 7 && (long long)rem * s_max >= grid;
  if (rem > 0 && !split) { b.whole_rounds += 1; rem = 0; }
  b.sk_tile0 = n_tiles - rem;
  b.sk_items = rem * num_kb;
  const int a_tiles = epi == EPI_GATE ? 2 : 1;
  int np = 16;                                                        // wgmma width: the padded session count
  while (np < Mpad) np <<= 1;
  b.np = np; b.Mpad = Mpad;
  b.stage_bytes = a_tiles * TILE_BYTES + np * BLOCK_K * 2;
  int stages = (f.stage_budget > 0 ? f.stage_budget : 200 * 1024) / b.stage_bytes;
  if (stages > MAX_STAGES) stages = MAX_STAGES;
  if (stages < 2) stages = 2;
  b.stages = stages;
  b.smem = stages * b.stage_bytes + 1024 + 16 * MAX_STAGES + 64;
  return add_block(P, b);
}

using GvKernel = void (*)(GvParams);
using CkKernel = void (*)(CUtensorMap, CkParams);
using SkKernel = void (*)(CUtensorMap, SkParams);

template <int EPI, bool NORM>
GvKernel gv_kernel_m(int M) {
  switch (M) {
    case 1: return gemv_kernel<EPI, 1, NORM>;
    case 2: return gemv_kernel<EPI, 2, NORM>;
    case 3: return gemv_kernel<EPI, 3, NORM>;
    default: return gemv_kernel<EPI, 4, NORM>;
  }
}
template <int EPI>
GvKernel gv_kernel(int M, bool norm) { return norm ? gv_kernel_m<EPI, true>(M) : gv_kernel_m<EPI, false>(M); }

template <int NP>
CkKernel ck_kernel(int epi) { return epi == EPI_STORE ? gemm_ck_kernel<EPI_STORE, NP> : gemm_ck_kernel<EPI_RESADD, NP>; }

template <int NP>
SkKernel sk_kernel(int epi) {
  if (epi == EPI_STORE) return gemm_sk_kernel<EPI_STORE, NP>;
  if (epi == EPI_RESADD) return gemm_sk_kernel<EPI_RESADD, NP>;
  return gemm_sk_kernel<EPI_GATE, (NP < SK_MAX_NP_GATE ? NP : SK_MAX_NP_GATE)>;
}

// the activation map of a block: rows [0, rows) of x, boxes of [box_rows x 128 bytes]; rows >= `rows` are zero-filled by the TMA unit
int cached_map(TensorMapCache& cache, const void* x, long long ldx, int rows, int K, int box_rows, int elem_bytes, const CUtensorMap** out) {
  MapKey key{x, ldx, rows, K, box_rows};
  auto it = cache.maps.find(key);
  if (it == cache.maps.end()) {
    CUtensorMap m;
    B200_TRY(act_map(&m, x, ldx, rows, K, box_rows, elem_bytes));
    it = cache.maps.emplace(key, m).first;
  }
  *out = &it->second;
  return B200_OK;
}

}  // namespace

int plan_linear(int M, int N, int K, int epi, int gate_rows, bool i8, bool norm, bool ld_aligned, int sms, int gemv_max_m,
                const LinearForce& force, LinearPlan* plan) {
  memset(plan, 0, sizeof(*plan));
  plan->M = M; plan->N = N; plan->K = K; plan->epi = epi; plan->gate_rows = gate_rows; plan->i8 = i8 ? 1 : 0;
  plan->stream_only = force.stream_only;
  if (!sk_supported(M, N, K, epi)) B200_FAIL(B200_ERR_SHAPE, "linear: unsupported shape M=%d N=%d K=%d", M, N, K);
  if (sms < 1) B200_FAIL(B200_ERR_INVALID, "linear: no multiprocessors to plan for");
  return plan_rows(*plan, 0, M, norm, ld_aligned, sms, gemv_max_m, force);
}

// y = epi(x . W^T) with W given as packed tiles, one launch per block of the plan
int run_linear(TensorMapCache& maps, const LinearPlan& P, const LinearArgs& a, cudaStream_t stream) {
  const int N = P.N, K = P.K, epi = P.epi;
  const bool i8 = P.i8 != 0;
  if (a.ldx % 8) B200_FAIL(B200_ERR_SHAPE, "linear: unsupported shape M=%d N=%d K=%d", P.M, N, K);
  if ((reinterpret_cast<uintptr_t>(a.x) | reinterpret_cast<uintptr_t>(a.w)) & 15)
    B200_FAIL(B200_ERR_SHAPE, "linear: operands must be 16-byte aligned");
  if (a.norm_alpha && !P.norm_folded)
    B200_FAIL(B200_ERR_STATE, "linear: a fused RMSNorm input is only available on the GEMV path (M=%d)", P.M);
  if (i8 && (!a.xq || !a.sa || !a.sw)) B200_FAIL(B200_ERR_SHAPE, "int8 GEMM: K must be a multiple of 16 and both scale vectors given");
  B200_TRY(linear_init());
  const int out_rows = epi == EPI_GATE ? P.gate_rows : N;
  const int n_tiles = (out_rows + BLOCK_ROWS - 1) / BLOCK_ROWS;
  const int num_kb = i8 ? (K + 127) / 128 : (K + BLOCK_K - 1) / BLOCK_K;
  for (int i = 0; i < P.n_blocks; ++i) {
    const LinearBlock& b = P.blocks[i];
    LinearArgs r = a;
    r.x = a.x + (long long)b.m0 * a.ldx;
    r.y = a.y + (long long)b.m0 * a.ldy;
    r.res = a.res ? a.res + (long long)b.m0 * a.ldr : nullptr;
    if (i8) { r.xq = static_cast<const int8_t*>(a.xq) + (long long)b.m0 * K; r.sa = a.sa + b.m0; }
    const LaunchOpts opts{a.pdl, b.kernel == LK_CK ? b.cluster : 0};
    const CUtensorMap* mx = nullptr;
    if (b.kernel == LK_GEMV) {
      GvParams p;
      p.M = b.rows; p.N = N; p.K = K; p.gate_rows = P.gate_rows; p.out_rows = out_rows; p.n_tiles = n_tiles; p.num_kb = num_kb;
      p.S = b.S; p.kbps = b.kbps;
      p.wt = static_cast<const uint8_t*>(r.w); p.x = r.x; p.ldx = r.ldx;
      p.y = r.y; p.ldy = r.ldy; p.res = r.res; p.ldr = r.ldr; p.ws = r.ws; p.counters = r.counters;
      p.norm_alpha = r.norm_alpha;
      const bool norm = p.norm_alpha != nullptr;
      const GvKernel k = epi == EPI_STORE ? gv_kernel<EPI_STORE>(p.M, norm) : epi == EPI_RESADD ? gv_kernel<EPI_RESADD>(p.M, norm)
                                                                                            : gv_kernel<EPI_GATE>(p.M, norm);
      B200_TRY(launch("gemv", k, dim3(b.grid), dim3(GV_THREADS), b.smem, stream, opts, p));
    } else if (b.kernel == LK_NS) {
      if ((reinterpret_cast<uintptr_t>(r.y) | reinterpret_cast<uintptr_t>(r.res)) & 15)
        B200_FAIL(B200_ERR_SHAPE, "ns GEMM: operands must be 16-byte aligned");
      if ((r.ldy % 8) || (r.res && r.ldr % 8)) B200_FAIL(B200_ERR_SHAPE, "ns GEMM: row strides must be multiples of 8");
      B200_TRY(cached_map(maps, r.x, r.ldx, b.rows, K, 128, 2, &mx));
      B200_TRY(ns_launch(*mx, P, b, r, stream));
    } else if (b.kernel == LK_CK) {
      if (i8) B200_TRY(cached_map(maps, r.xq, K, b.rows, K, b.np, 1, &mx));
      else B200_TRY(cached_map(maps, r.x, r.ldx, b.rows, K, b.np, 2, &mx));
      CkParams p;
      p.M = b.rows; p.N = N; p.K = K; p.CS = b.cluster; p.Mpad = b.Mpad; p.Wc = b.Wc;
      p.num_kb = num_kb; p.kb_per = b.kb_per; p.stages = b.stages; p.stage_bytes = (uint32_t)b.stage_bytes;
      p.wt = static_cast<const uint8_t*>(r.w);
      p.y = r.y; p.ldy = r.ldy; p.res = r.res; p.ldr = r.ldr;
      p.i8 = i8 ? 1 : 0; p.sa = r.sa; p.sw = r.sw;
      const CkKernel k = b.np == 64 ? ck_kernel<64>(epi) : b.np == 128 ? ck_kernel<128>(epi) : ck_kernel<256>(epi);
      B200_TRY(launch("gemm_ck", k, dim3(b.grid), dim3(NUM_THREADS), b.smem, stream, opts, *mx, p));
    } else {
      if (i8) B200_TRY(cached_map(maps, r.xq, K, b.rows, K, b.np, 1, &mx));
      else B200_TRY(cached_map(maps, r.x, r.ldx, b.rows, K, b.np, 2, &mx));
      SkParams p;
      p.M = b.rows; p.N = N; p.K = K; p.gate_rows = P.gate_rows; p.out_rows = out_rows; p.Mpad = b.Mpad;
      p.stages = b.stages; p.num_kb = num_kb; p.n_tiles = n_tiles;
      p.grid = b.grid; p.whole_rounds = b.whole_rounds; p.sk_tile0 = b.sk_tile0; p.sk_items = b.sk_items;
      p.wt = static_cast<const uint8_t*>(r.w);
      p.y = r.y; p.ldy = r.ldy; p.res = r.res; p.ldr = r.ldr;
      p.ws = r.ws; p.counters = r.counters;
      p.stage_bytes = (uint32_t)b.stage_bytes;
      p.stream_only = P.stream_only;
      p.i8 = i8 ? 1 : 0; p.sa = r.sa; p.sw = r.sw;
      const SkKernel k = b.np == 16 ? sk_kernel<16>(epi) : b.np == 32 ? sk_kernel<32>(epi) : b.np == 64 ? sk_kernel<64>(epi) : sk_kernel<128>(epi);
      B200_TRY(launch("gemm_sk", k, dim3(b.grid), dim3(NUM_THREADS), b.smem, stream, opts, *mx, p));
    }
  }
  return B200_OK;
}

}  // namespace tc
}  // namespace b200
