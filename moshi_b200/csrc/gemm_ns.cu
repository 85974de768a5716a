// wgmma GEMM for the LM linears at 33..256 sessions:  y[M][N] = epi(x[M][K] . w[N][K]^T), bf16 in, fp32 in registers, bf16 out.
//
// gemm_sk.cu feeds the 128-row weight tile as the MMA *A* operand and the sessions as N ("swap-AB"): right while the batch is
// tiny.  From 33 sessions on the operands keep their textbook roles here:
//
//   * A = the activations, one [128 sessions x 64 k] SWIZZLE_128B box per k-block (2-D TMA, rows beyond M zero-filled);
//     consumer warpgroup w multiplies sessions 64w..64w+63 (a warpgroup without sessions skips its MMAs).  Above 128
//     sessions the plan runs two launches, one per block of 128 sessions;
//   * B = TWO pre-tiled 128-row weight tiles side by side (N = 256 per instruction: twice the weight bytes per MMA);
//     for the gated MLP the pair is (gate rows, value rows) of the same outputs, already stored back to back, so the
//     accumulator holds gate in columns 0..127 and value in 128..255 of the SAME thread and silu(g) * u needs no exchange;
//   * D = [64 sessions x 256 weight rows] fp32 per warpgroup in registers; the epilogue runs straight from the fragments
//     (two consecutive outputs of one session per store).
//   * shapes with fewer units than SMs are cut along K over a cluster of 2..4 CTAs (in_proj: 48 pairs x 2; out_proj / linear_out:
//     32 single tiles x 4, N = 128 per instruction there so that 128 SMs pull on the weights); the partial accumulators are
//     reduce-scattered over distributed shared memory by output columns (the stage ring is dead by then and serves as the
//     receive buffer), summed in rank order (deterministic) and stored by the owning rank: no workspace, no atomics.
//     ns_default_plan() (gemm_sk.cu) holds the choice per shape.
//
// Same packed weights, same epilogues and cast points as gemm_sk.cu (residual add bf16(res + bf16(acc)), gated SiLU
// bf16(bf16(silu(g)) * u), gating.py:18-20); same PDL protocol (weights requested before griddepcontrol.wait).
#include "gemm_sk.cuh"
#include "tc_prims.cuh"

namespace b200 {
namespace tc {

namespace {

using namespace tcp;

constexpr int EPI_STORE = 0, EPI_RESADD = 1, EPI_GATE = 2;
constexpr int BLOCK_ROWS = 128, BLOCK_K = 64, UMMA_K = 16;
constexpr int NUM_THREADS = 288;             // warps 0-7: two consumer warpgroups (MMA + epilogue), warp 8: producer
constexpr int PRODUCER_WARP = 8;
constexpr int CONSUMERS = 256;
constexpr int TILE_BYTES = BLOCK_ROWS * BLOCK_K * 2;
constexpr int A_BYTES = NS_A_BYTES;         // one activation box: 128 session rows x 64 k
constexpr int MAX_STAGES = NS_MAX_STAGES;

struct NsParams {
  int M, N, K, out_rows, gate_rows, CS, num_kb, kb_per, stages, n_tiles, ldw;
  const uint8_t* wt;
  __nv_bfloat16* y; long long ldy;
  const __nv_bfloat16* res; long long ldr;
};

// first accumulator column of rank q's share of `width` columns (multiples of 16; the last rank takes the remainder)
__device__ __forceinline__ int col_begin(int width, int cs, int q) { return q >= cs ? width : ((width * q / cs) >> 4) << 4; }

// two consecutive outputs of one session row -> y (one 4-byte store; `valid` outputs remain in the row)
__device__ __forceinline__ void store2(__nv_bfloat16* dst, const float* v, int valid) {
  if (valid >= 2) *reinterpret_cast<__nv_bfloat162*>(dst) = __floats2bfloat162_rn(v[0], v[1]);
  else dst[0] = __float2bfloat16_rn(v[0]);
}
__device__ __forceinline__ void load2(const __nv_bfloat16* src, float* v, int valid) {
  if (valid >= 2) {
    const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(src));
    v[0] = f.x; v[1] = f.y;
  } else {
    v[0] = __bfloat162float(src[0]); v[1] = 0.f;
  }
}
// 16 consecutive outputs of one session row -> y (two 16-byte stores)
__device__ __forceinline__ void store16(__nv_bfloat16* dst, const float* v, int valid) {
  if (valid >= 16) {
    __nv_bfloat162 o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
    uint4* d4 = reinterpret_cast<uint4*>(dst);
    d4[0] = *reinterpret_cast<const uint4*>(&o[0]);
    d4[1] = *reinterpret_cast<const uint4*>(&o[4]);
  } else {
    for (int j = 0; j < valid; ++j) dst[j] = __float2bfloat16_rn(v[j]);
  }
}
__device__ __forceinline__ void load16(const __nv_bfloat16* src, float* v, int valid) {
  if (valid >= 16) {
    const uint4* s4 = reinterpret_cast<const uint4*>(src);
    const uint4 a = s4[0], b = s4[1];
    const __nv_bfloat162* ha = reinterpret_cast<const __nv_bfloat162*>(&a);
    const __nv_bfloat162* hb = reinterpret_cast<const __nv_bfloat162*>(&b);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __bfloat1622float2(ha[j]), g = __bfloat1622float2(hb[j]);
      v[2 * j] = f.x; v[2 * j + 1] = f.y; v[8 + 2 * j] = g.x; v[8 + 2 * j + 1] = g.y;
    }
  } else {
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = j < valid ? __bfloat162float(src[j]) : 0.f;
  }
}

template <int EPI, int UT>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_ns_kernel(const __grid_constant__ CUtensorMap tmap_x, const NsParams p) {
  constexpr int NW = 128 * UT;                                            // wgmma width: the weight rows of a unit
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  constexpr uint32_t a_off = (uint32_t)UT * TILE_BYTES;                   // stage = B (one or two weight tiles) | A (activation box)
  constexpr uint32_t stage_bytes = a_off + A_BYTES;
  const uint32_t bars = base + (uint32_t)p.stages * stage_bytes;
  const uint32_t full0 = bars, empty0 = bars + 8 * MAX_STAGES;
  const float* recv_generic = reinterpret_cast<const float*>(smem_raw + (base - raw));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int unit = blockIdx.x / p.CS, me = blockIdx.x - unit * p.CS;
  const int kb0 = me * p.kb_per, kb1 = min(p.num_kb, kb0 + p.kb_per);
  const int n_items = kb1 > kb0 ? kb1 - kb0 : 0;
  // weight tiles of this unit: the (gate, value) pair, or row tiles 2u and 2u+1 (the last unit of an odd count has one)
  const bool two = EPI == EPI_GATE || (UT == 2 && 2 * unit + 1 < p.n_tiles);
  const int tile0 = EPI == EPI_GATE ? unit : unit * UT;
  const int width = two ? 256 : 128;                                      // accumulator columns in use
  const uint32_t b_bytes = two ? 2u * TILE_BYTES : (uint32_t)TILE_BYTES;

  if (warp == PRODUCER_WARP && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_x) : "memory");
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, CONSUMERS / 32);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_trigger();

  uint32_t d[NW / 2];
#pragma unroll
  for (int i = 0; i < NW / 2; ++i) d[i] = 0u;    // a rank without k-blocks contributes zeros
  const int wg = warp >> 2, t = threadIdx.x & 127;
  if (warp == PRODUCER_WARP) {
    if (lane == 0) {
      auto load_b = [&](int i, int s) {
        const int kb = kb0 + i;
        const uint32_t sb = base + (uint32_t)s * stage_bytes;
        if (EPI == EPI_GATE) {
          bulk_load(sb, p.wt + ((size_t)unit * p.num_kb + kb) * (2 * TILE_BYTES), 2 * TILE_BYTES, full0 + 8 * s);
        } else {
          bulk_load(sb, p.wt + ((size_t)tile0 * p.num_kb + kb) * TILE_BYTES, TILE_BYTES, full0 + 8 * s);
          if (two) bulk_load(sb + TILE_BYTES, p.wt + ((size_t)(tile0 + 1) * p.num_kb + kb) * TILE_BYTES, TILE_BYTES, full0 + 8 * s);
        }
      };
      // weights first (they do not depend on the preceding kernel), activations after the dependency wait
      const int pre = n_items < p.stages ? n_items : p.stages;
      for (int i = 0; i < pre; ++i) {
        mbar_expect_tx(full0 + 8 * i, b_bytes + A_BYTES);
        load_b(i, i);
      }
      pdl_wait();
      int s = 0; uint32_t ph = 0;
      for (int i = 0; i < n_items; ++i) {
        if (i >= pre) {
          mbar_wait(empty0 + 8 * s, ph ^ 1u);
          mbar_expect_tx(full0 + 8 * s, b_bytes + A_BYTES);
          load_b(i, s);
        }
        tma_load_2d(base + (uint32_t)s * stage_bytes + a_off, &tmap_x, full0 + 8 * s, (kb0 + i) * BLOCK_K, 0);
        if (++s == p.stages) { s = 0; ph ^= 1u; }
      }
    }
    __syncwarp();
  } else {
    // warpgroup wg: sessions 64 wg .. 64 wg + 63 (a warpgroup without sessions only keeps the ring moving)
    const bool active = 64 * wg < p.M;
    int s = 0; uint32_t ph = 0;
    for (int i = 0; i < n_items; ++i) {
      mbar_wait(full0 + 8 * s, ph);
      if (active) {
        const uint32_t sb = base + (uint32_t)s * stage_bytes;
        const uint32_t sa = sb + a_off + (uint32_t)wg * (A_BYTES / 2);
        wg_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / UMMA_K; ++k)
          Wgmma<NW>::bf16(d, make_desc(sa + k * UMMA_K * 2), make_desc(sb + k * UMMA_K * 2), (i == 0 && k == 0) ? 0u : 1u);
        wg_commit();
        wg_wait<0>();
        wg_hold(d);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(empty0 + 8 * s);
      if (++s == p.stages) { s = 0; ph ^= 1u; }
    }
    pdl_wait();                                 // y / res may still be in use by the predecessor
  }

  if (p.CS == 1) {
    if (warp == PRODUCER_WARP) return;
    // straight from the fragments: element pair (i, i + 1) is outputs n, n + 1 of session m
    if (EPI == EPI_GATE) {
      // columns j (gate) and 128 + j (value) of the same output sit in registers i and i + 64 of the same thread
      const int nb = unit * BLOCK_ROWS;
#pragma unroll
      for (int i = 0; i < 64; i += 2) {
        const int m = 64 * wg + frag_row(t, i), n = nb + frag_col(t, i);
        if (m < p.M && n < p.out_rows) {
          float v[2];
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const float gt = bf16_round(__uint_as_float(d[i + j])), ut = bf16_round(__uint_as_float(d[64 + i + j]));
            v[j] = bf16_round(gt / (1.f + expf(-gt))) * ut;
          }
          store2(p.y + (long long)m * p.ldy + n, v, p.out_rows - n);
        }
      }
    } else {
      const int nb = tile0 * BLOCK_ROWS;
#pragma unroll
      for (int i = 0; i < NW / 2; i += 2) {
        const int m = 64 * wg + frag_row(t, i), c = frag_col(t, i), n = nb + c;
        if (c < width && m < p.M && n < p.out_rows) {
          float v[2] = {__uint_as_float(d[i]), __uint_as_float(d[i + 1])};
          if (EPI == EPI_RESADD) {
            float rv[2];
            load2(p.res + (long long)m * p.ldr + n, rv, p.out_rows - n);
            v[0] = rv[0] + bf16_round(v[0]); v[1] = rv[1] + bf16_round(v[1]);
          }
          store2(p.y + (long long)m * p.ldy + n, v, p.out_rows - n);
        }
      }
    }
    return;
  }
  // K split over the cluster: column c of every rank's accumulator goes to the rank that owns c, slot = sender rank
  cluster_sync_all();                            // every rank's MMAs have retired: the rings are free to receive
  if (warp != PRODUCER_WARP) {
#pragma unroll
    for (int i = 0; i < NW / 2; i += 2) {
      const int m = 64 * wg + frag_row(t, i), c = frag_col(t, i);
      if (c < width && m < p.M) {
        int q = 0;
        while (c >= col_begin(width, p.CS, q + 1)) ++q;
        const uint32_t dst = map_to_rank(base + (uint32_t)((me * 128 + m) * p.ldw + (c - col_begin(width, p.CS, q))) * 4u, (uint32_t)q);
        st_cluster_v2(dst, d[i], d[i + 1]);
      }
    }
  }
  cluster_sync_all();                            // every partial has landed in its owner's receive buffer
  if (warp != PRODUCER_WARP) {
    const int my_c0 = col_begin(width, p.CS, me), my_c1 = col_begin(width, p.CS, me + 1);
    const int et = threadIdx.x, m = et & 127;
    const int nb = tile0 * BLOCK_ROWS;
    if (m < p.M) {
      for (int c = my_c0 + (et >> 7) * 16; c < my_c1; c += 32) {
        const int valid = p.out_rows - (nb + c);
        if (valid <= 0) break;
        float acc[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) acc[j] = 0.f;
        float rv[16];
        if (EPI == EPI_RESADD) load16(p.res + (long long)m * p.ldr + nb + c, rv, valid);
        for (int r = 0; r < p.CS; ++r) {        // rank order: the sum does not depend on which rank does it
          const float4* src = reinterpret_cast<const float4*>(recv_generic + (size_t)(r * 128 + m) * p.ldw + (c - my_c0));
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float4 v = src[j];
            acc[4 * j] += v.x; acc[4 * j + 1] += v.y; acc[4 * j + 2] += v.z; acc[4 * j + 3] += v.w;
          }
        }
        if (EPI == EPI_RESADD) {
#pragma unroll
          for (int j = 0; j < 16; ++j) acc[j] = rv[j] + bf16_round(acc[j]);
        }
        store16(p.y + (long long)m * p.ldy + nb + c, acc, valid);
      }
    }
  }
  cluster_sync_all();                            // no CTA exits while a peer could still address its shared memory
}

using NsKernel = void (*)(CUtensorMap, NsParams);

}  // namespace

int ns_init() {
  static bool done = false;
  if (done) return B200_OK;
  const int max_smem = 220 * 1024;
  B200_CUDA(cudaFuncSetAttribute(gemm_ns_kernel<EPI_STORE, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
  B200_CUDA(cudaFuncSetAttribute(gemm_ns_kernel<EPI_RESADD, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
  B200_CUDA(cudaFuncSetAttribute(gemm_ns_kernel<EPI_STORE, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
  B200_CUDA(cudaFuncSetAttribute(gemm_ns_kernel<EPI_RESADD, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
  B200_CUDA(cudaFuncSetAttribute(gemm_ns_kernel<EPI_GATE, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
  done = true;
  return B200_OK;
}

// one block of an NS plan (plan_linear, gemm_sk.cu); the operands of `a` start at the block's first row
int ns_launch(const CUtensorMap& mx, const LinearPlan& plan, const LinearBlock& b, const LinearArgs& a, cudaStream_t stream) {
  B200_TRY(ns_init());
  const int epi = plan.epi;
  NsParams p;
  p.M = b.rows; p.N = plan.N; p.K = plan.K; p.gate_rows = plan.gate_rows;
  p.out_rows = epi == EPI_GATE ? plan.gate_rows : plan.N;
  p.n_tiles = (p.out_rows + BLOCK_ROWS - 1) / BLOCK_ROWS;
  p.num_kb = (plan.K + BLOCK_K - 1) / BLOCK_K;
  p.CS = b.cluster; p.kb_per = b.kb_per; p.ldw = b.ldw; p.stages = b.stages;
  p.wt = static_cast<const uint8_t*>(a.w);
  p.y = a.y; p.ldy = a.ldy; p.res = a.res; p.ldr = a.ldr;
  const NsKernel k = epi == EPI_GATE ? gemm_ns_kernel<EPI_GATE, 2>
                     : b.unit_tiles == 1 ? (epi == EPI_STORE ? gemm_ns_kernel<EPI_STORE, 1> : gemm_ns_kernel<EPI_RESADD, 1>)
                                         : (epi == EPI_STORE ? gemm_ns_kernel<EPI_STORE, 2> : gemm_ns_kernel<EPI_RESADD, 2>);
  return launch("gemm_ns", k, dim3((unsigned)b.grid), dim3(NUM_THREADS), b.smem, stream, LaunchOpts{a.pdl, b.cluster > 1 ? b.cluster : 0},
                mx, p);
}

}  // namespace tc
}  // namespace b200
