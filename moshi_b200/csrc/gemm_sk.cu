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
//     launch to 128 sessions (64 for the gated pair); sk_linear runs larger batches as consecutive launches.
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

__device__ __forceinline__ float bf16_round(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

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

__device__ __forceinline__ uint32_t map_to_rank(uint32_t local_smem_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void st_cluster_v2(uint32_t addr, uint32_t a, uint32_t b) {
  asm volatile("st.shared::cluster.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(a), "r"(b) : "memory");
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

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
constexpr int GV_MAX_M = 4;                // compiled for up to 4 rows; used for <= 2 by default (B200_GEMV_MAX_M)
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

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;
bool g_attr_set = false;
int g_sms = 0;
int g_gemv_max_m = 2;            // B200_GEMV_MAX_M (0..4): 0 sends every batch size through the tensor-core GEMM
int g_use_ns = 1;                // B200_GEMM_NS=0: keep the swap-AB kernels above 32 sessions (A/B measurements)

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

int init_once() {
  if (!g_encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    B200_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    if (!fn || qres != cudaDriverEntryPointSuccess) B200_FAIL(B200_ERR_CUDA, "cuTensorMapEncodeTiled not available");
    g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  }
  if (!g_attr_set) {
    B200_TRY(set_smem_attrs());
    int dev = 0;
    B200_CUDA(cudaGetDevice(&dev));
    B200_CUDA(cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, dev));
    if (const char* e = getenv("B200_GEMV_MAX_M")) g_gemv_max_m = atoi(e);
    if (const char* e = getenv("B200_GEMM_NS")) g_use_ns = atoi(e);
    g_attr_set = true;
  }
  return B200_OK;
}

}  // namespace

int prepare_plans(GemmPlanCache&) { B200_TRY(ns_prepare()); return init_once(); }

int sk_num_sms() { return init_once() == B200_OK ? g_sms : 0; }

int sk_gemv_max_m() { return init_once() == B200_OK ? g_gemv_max_m : 0; }

int sk_set_gemv_max_m(int max_m) {
  if (init_once() != B200_OK) return -1;
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
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)M); cfg.blockDim = dim3(256); cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = pdl ? 1 : 0;
  B200_CUDA(cudaLaunchKernelEx(&cfg, quantize_rows_kernel, x, ldx, static_cast<int8_t*>(xq), sa, K));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return check_launch("quantize_rows");
}

size_t sk_workspace_bytes(int max_M) {
  const int Mpad = ((max_M + 15) / 16) * 16;
  return (size_t)2 * SK_MAX_GRID * 2 * Mpad * BLOCK_ROWS * 4;  // 2 slots per CTA, gate + value accumulators
}

bool sk_supported(int M, int N, int K, int epi) {
  (void)N; (void)epi;
  return M >= 1 && M <= 256 && K >= 8 && K % 8 == 0;
}

// 2-D tensor map of the activations x [M][K] (row stride ldx elements) with a [box_rows x 128 bytes] SWIZZLE_128B box;
// elem_bytes = 2 (bf16) or 1 (int8)
static int x_map(GemmPlanCache& cache, const void* x, long long ldx, int M, int K, int box_rows, int elem_bytes,
                 const CUtensorMap** out) {
  PlanKey key{x, ldx, M, K, box_rows};
  auto it = cache.maps.find(key);
  if (it == cache.maps.end()) {
    CUtensorMap m;
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)M};
    cuuint64_t strides[1] = {(cuuint64_t)ldx * elem_bytes};
    cuuint32_t box[2] = {(cuuint32_t)(128 / elem_bytes), (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = g_encode(&m, elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 2,
                          const_cast<void*>(x), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) B200_FAIL(B200_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) M=%d K=%d ld=%lld", (int)r, M, K, ldx);
    it = cache.maps.emplace(key, m).first;
  }
  *out = &it->second;
  return B200_OK;
}

template <int NP>
static cudaError_t sk_launch(const cudaLaunchConfig_t& cfg, int epi, const CUtensorMap& mx, const SkParams& p) {
  if (epi == EPI_STORE) return cudaLaunchKernelEx(&cfg, gemm_sk_kernel<EPI_STORE, NP>, mx, p);
  if (epi == EPI_RESADD) return cudaLaunchKernelEx(&cfg, gemm_sk_kernel<EPI_RESADD, NP>, mx, p);
  return cudaLaunchKernelEx(&cfg, gemm_sk_kernel<EPI_GATE, (NP < SK_MAX_NP_GATE ? NP : SK_MAX_NP_GATE)>, mx, p);
}

// y = epi(x . W^T) with W given as packed tiles.  ws / counters: sk_workspace_bytes(M) and >= 1024 ints, zeroed once.
int sk_linear(GemmPlanCache& cache, const __nv_bfloat16* x, long long ldx, const void* w_tiles, __nv_bfloat16* y,
              long long ldy, const __nv_bfloat16* res, long long ldr, int M, int N, int K, int epi, int gate_rows,
              float* ws, int* counters, const SkTuning& tune, cudaStream_t stream) {
  if (!sk_supported(M, N, K, epi) || ldx % 8) B200_FAIL(B200_ERR_SHAPE, "sk GEMM: unsupported shape M=%d N=%d K=%d", M, N, K);
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(w_tiles)) & 15)
    B200_FAIL(B200_ERR_SHAPE, "sk GEMM: operands must be 16-byte aligned");
  B200_TRY(init_once());
  const bool i8 = tune.xq != nullptr;
  // one to four sessions: stream the tiles with plain loads on the CUDA cores (no bulk-copy engine ceiling)
  if (!i8 && M <= GV_MAX_M && tune.grid == 0 && tune.cluster == 0 && !tune.stream_only && g_gemv_max_m >= M) {
    GvParams p;
    p.M = M; p.N = N; p.K = K; p.gate_rows = gate_rows;
    p.out_rows = epi == EPI_GATE ? gate_rows : N;
    p.n_tiles = (p.out_rows + BLOCK_ROWS - 1) / BLOCK_ROWS;
    p.num_kb = (K + BLOCK_K - 1) / BLOCK_K;
    if (p.n_tiles > SK_MAX_TILES) B200_FAIL(B200_ERR_SHAPE, "gemv: more than %d row tiles", SK_MAX_TILES);
    const int A = epi == EPI_GATE ? 2 : 1;
    // enough CTAs for ~4 per SM, every CTA streams at least 4 k-blocks, the activation slice fits in shared memory
    int S = (4 * g_sms + p.n_tiles - 1) / p.n_tiles;
    if (S > p.num_kb / 4) S = p.num_kb / 4;
    if (S < 1) S = 1;
    const int s_min = (p.num_kb + GV_MAX_KBPS - 1) / GV_MAX_KBPS;
    if (S < s_min) S = s_min;
    const size_t slot_bytes = (size_t)A * M * BLOCK_ROWS * 4;
    while (S > s_min && (size_t)p.n_tiles * S * slot_bytes > sk_workspace_bytes(M)) --S;
    p.kbps = (p.num_kb + S - 1) / S;
    p.S = (p.num_kb + p.kbps - 1) / p.kbps;
    if ((size_t)p.n_tiles * p.S * slot_bytes <= sk_workspace_bytes(M)) {
      p.wt = static_cast<const uint8_t*>(w_tiles); p.x = x; p.ldx = ldx;
      p.y = y; p.ldy = ldy; p.res = res; p.ldr = ldr; p.ws = ws; p.counters = counters;
      p.norm_alpha = tune.norm_alpha;
      cudaLaunchConfig_t cfg;
      memset(&cfg, 0, sizeof(cfg));
      cfg.gridDim = dim3((unsigned)(p.n_tiles * p.S)); cfg.blockDim = dim3(GV_THREADS);
      cfg.dynamicSmemBytes = (size_t)M * p.kbps * BLOCK_K * 2; cfg.stream = stream;
      cudaLaunchAttribute attr[1];
      attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
      attr[0].val.programmaticStreamSerializationAllowed = 1;
      cfg.attrs = attr; cfg.numAttrs = tune.pdl ? 1 : 0;
      const cudaError_t le = epi == EPI_STORE ? gv_launch<EPI_STORE>(cfg, p) : epi == EPI_RESADD ? gv_launch<EPI_RESADD>(cfg, p) : gv_launch<EPI_GATE>(cfg, p);
      if (le != cudaSuccess) B200_FAIL(B200_ERR_CUDA, "gemv launch failed: %s", cudaGetErrorString(le));
      g_launches.fetch_add(1, std::memory_order_relaxed);
      return check_launch("gemv");
    }
  }
  if (tune.norm_alpha) B200_FAIL(B200_ERR_STATE, "sk GEMM: a fused RMSNorm input is only available on the GEMV path (M=%d)", M);
  // 33..256 sessions: activations as the A operand, two weight tiles (N = 256) per wgmma (gemm_ns.cu)
  if (!i8 && tune.ns >= 0 && (tune.ns > 0 || (g_use_ns && M > 32)) && M <= 256 && tune.grid == 0 && tune.cluster == 0 && !tune.stream_only &&
      !tune.force_split && ns_supported(M, N, K, epi) && ldy % 8 == 0 && (!res || ldr % 8 == 0))
    return ns_linear(cache, x, ldx, w_tiles, y, ldy, res, ldr, M, N, K, epi, gate_rows, 0, tune.pdl, stream);
  // more than 32 sessions and few row tiles: a cluster of CTAs per tile, split along K, reduced over DSMEM
  if (i8 && (K % 16 || !tune.sa || !tune.sw)) B200_FAIL(B200_ERR_SHAPE, "int8 GEMM: K must be a multiple of 16 and both scale vectors given");
  if (epi != EPI_GATE && tune.no_cluster == 0 && tune.grid == 0 && M > 32) {
    const int n_tiles = (N + BLOCK_ROWS - 1) / BLOCK_ROWS, num_kb = i8 ? (K + 127) / 128 : (K + BLOCK_K - 1) / BLOCK_K;
    int cs = 1;
    while (cs < 8 && n_tiles * cs * 2 <= g_sms && num_kb / (cs * 2) >= 4) cs *= 2;
    if (tune.cluster > 0) cs = tune.cluster;
    if (cs > 1) {
      CkParams p;
      p.M = M; p.N = N; p.K = K; p.CS = cs;
      const int quantum = 8 * cs < 16 ? 16 : 8 * cs;       // wgmma N is a multiple of 16; every rank owns whole 8-column groups
      p.Mpad = ((M + quantum - 1) / quantum) * quantum;
      p.Wc = p.Mpad / cs;
      int np = 64;                                          // wgmma width: the padded session count (M > 32 here)
      while (np < p.Mpad) np <<= 1;
      if (p.Mpad <= 256 && p.Wc <= 64) {
        p.num_kb = num_kb; p.kb_per = (num_kb + cs - 1) / cs;
        p.wt = static_cast<const uint8_t*>(w_tiles);
        p.y = y; p.ldy = ldy; p.res = res; p.ldr = ldr;
        p.i8 = i8 ? 1 : 0; p.sa = tune.sa; p.sw = tune.sw;
        p.stage_bytes = (uint32_t)(TILE_BYTES + np * BLOCK_K * 2);          // 128 bytes of K per row, bf16 or int8
        const size_t recv_bytes = (size_t)cs * BLOCK_ROWS * (p.Wc + 4) * 4;
        int stages = (int)((200 * 1024 - recv_bytes) / p.stage_bytes);
        if (stages > MAX_STAGES) stages = MAX_STAGES;
        if (stages > p.kb_per) stages = p.kb_per;
        if (stages >= 2) {
          p.stages = stages;
          const CUtensorMap* mx = nullptr;
          if (i8) B200_TRY(x_map(cache, tune.xq, K, M, K, np, 1, &mx));
          else B200_TRY(x_map(cache, x, ldx, M, K, np, 2, &mx));
          const size_t smem = (size_t)stages * p.stage_bytes + 1024 + 16 * MAX_STAGES + 16 + recv_bytes;
          cudaLaunchConfig_t cfg;
          memset(&cfg, 0, sizeof(cfg));
          cfg.gridDim = dim3(n_tiles * cs); cfg.blockDim = dim3(NUM_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
          cudaLaunchAttribute attr[2];
          attr[0].id = cudaLaunchAttributeClusterDimension;
          attr[0].val.clusterDim.x = cs; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
          attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
          attr[1].val.programmaticStreamSerializationAllowed = 1;
          cfg.attrs = attr; cfg.numAttrs = tune.pdl ? 2 : 1;
          cudaError_t le;
          if (np == 64) le = epi == EPI_STORE ? cudaLaunchKernelEx(&cfg, gemm_ck_kernel<EPI_STORE, 64>, *mx, p)
                                              : cudaLaunchKernelEx(&cfg, gemm_ck_kernel<EPI_RESADD, 64>, *mx, p);
          else if (np == 128) le = epi == EPI_STORE ? cudaLaunchKernelEx(&cfg, gemm_ck_kernel<EPI_STORE, 128>, *mx, p)
                                                    : cudaLaunchKernelEx(&cfg, gemm_ck_kernel<EPI_RESADD, 128>, *mx, p);
          else le = epi == EPI_STORE ? cudaLaunchKernelEx(&cfg, gemm_ck_kernel<EPI_STORE, 256>, *mx, p)
                                     : cudaLaunchKernelEx(&cfg, gemm_ck_kernel<EPI_RESADD, 256>, *mx, p);
          if (le != cudaSuccess) B200_FAIL(B200_ERR_CUDA, "gemm_ck launch failed: %s", cudaGetErrorString(le));
          g_launches.fetch_add(1, std::memory_order_relaxed);
          return check_launch("gemm_ck");
        }
      }
    }
  }
  // The accumulator of a CTA lives in the registers of its two consumer warpgroups: at most 128 sessions per launch (64 for
  // the gated MLP's two accumulators).  Larger batches run as consecutive launches over blocks of sessions, each streaming
  // the weights again.
  const int max_np = epi == EPI_GATE ? SK_MAX_NP_GATE : SK_MAX_NP;
  if (M > max_np) {
    for (int m0 = 0; m0 < M; m0 += max_np) {
      const int mc = M - m0 < max_np ? M - m0 : max_np;
      SkTuning t2 = tune;
      if (i8) { t2.xq = static_cast<const int8_t*>(tune.xq) + (long long)m0 * K; t2.sa = tune.sa + m0; }
      B200_TRY(sk_linear(cache, x + (long long)m0 * ldx, ldx, w_tiles, y + (long long)m0 * ldy, ldy, res ? res + (long long)m0 * ldr : nullptr,
                         ldr, mc, N, K, epi, gate_rows, ws, counters, t2, stream));
    }
    return B200_OK;
  }
  SkParams p;
  p.M = M; p.N = N; p.K = K; p.gate_rows = gate_rows;
  p.out_rows = epi == EPI_GATE ? gate_rows : N;
  p.Mpad = ((M + 15) / 16) * 16;
  p.wt = static_cast<const uint8_t*>(w_tiles);
  p.y = y; p.ldy = ldy; p.res = res; p.ldr = ldr;
  p.ws = ws; p.counters = counters;
  p.i8 = i8 ? 1 : 0; p.sa = tune.sa; p.sw = tune.sw;
  p.num_kb = i8 ? (K + 127) / 128 : (K + BLOCK_K - 1) / BLOCK_K;      // a k-block is 128 bytes of K per row
  p.n_tiles = (p.out_rows + BLOCK_ROWS - 1) / BLOCK_ROWS;
  if (p.n_tiles > 1024) B200_FAIL(B200_ERR_SHAPE, "sk GEMM: more than 1024 row tiles");
  int grid = tune.grid > 0 ? tune.grid : g_sms;
  if (grid > SK_MAX_GRID) grid = SK_MAX_GRID;
  if (grid > p.n_tiles * p.num_kb) grid = p.n_tiles * p.num_kb;
  // a CTA should stream at least ~8 k-blocks (128-256 KB): below that the per-CTA set-up and the partial exchange dominate
  if (tune.grid == 0 && grid > (p.n_tiles * p.num_kb) / 8) grid = (p.n_tiles * p.num_kb) / 8 > 0 ? (p.n_tiles * p.num_kb) / 8 : 1;
  // Cutting a tile into S pieces moves S fp32 partials of [128 x Mpad] through L2 (written + read back): allow it
  // only while that stays under half of the tile's weight bytes, i.e. S <= 8 * num_kb / Mpad.
  int s_max = tune.no_split ? 1 : (8 * p.num_kb) / p.Mpad;      // int8 partials are int32 and add exactly
  // with more than 32 sessions the publish / count / re-read protocol
  // costs more than the idle SMs it recovers, so tiles stay whole there
  if (p.Mpad > 32 && tune.force_split == 0) s_max = 1;
  if (s_max < 1) s_max = 1;
  if (p.n_tiles < grid && (long long)p.n_tiles * s_max < grid) grid = p.n_tiles * s_max;   // fewer CTAs, fewer pieces
  // whole rounds of the grid, then the remainder as a stream-K region shared by all CTAs
  p.grid = grid;
  p.whole_rounds = p.n_tiles / grid;
  int rem = p.n_tiles - p.whole_rounds * grid;
  const bool split = rem > 0 && s_max > 1 && rem * 8 < grid * 7 && (long long)rem * s_max >= grid;
  if (rem > 0 && !split) { p.whole_rounds += 1; rem = 0; }
  p.sk_tile0 = p.n_tiles - rem;
  p.sk_items = rem * p.num_kb;
  const int a_tiles = epi == EPI_GATE ? 2 : 1;
  int np = 16;                                                        // wgmma width: the padded session count
  while (np < p.Mpad) np <<= 1;
  p.stage_bytes = (uint32_t)(a_tiles * TILE_BYTES + np * BLOCK_K * 2);
  int stages = (tune.smem_budget > 0 ? tune.smem_budget : 200 * 1024) / (int)p.stage_bytes;
  if (stages > MAX_STAGES) stages = MAX_STAGES;
  if (stages < 2) stages = 2;
  p.stages = stages;
  p.stream_only = tune.stream_only;
  const CUtensorMap* mx = nullptr;
  if (i8) B200_TRY(x_map(cache, tune.xq, K, M, K, np, 1, &mx));
  else B200_TRY(x_map(cache, x, ldx, M, K, np, 2, &mx));
  const size_t smem = (size_t)stages * p.stage_bytes + 1024 + 16 * MAX_STAGES + 64;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(NUM_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = tune.pdl ? 1 : 0;
  cudaError_t le;
  if (np == 16) le = sk_launch<16>(cfg, epi, *mx, p);
  else if (np == 32) le = sk_launch<32>(cfg, epi, *mx, p);
  else if (np == 64) le = sk_launch<64>(cfg, epi, *mx, p);
  else le = sk_launch<128>(cfg, epi, *mx, p);
  if (le != cudaSuccess) B200_FAIL(B200_ERR_CUDA, "gemm_sk launch failed: %s", cudaGetErrorString(le));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return check_launch("gemm_sk");
}

}  // namespace tc
}  // namespace b200
