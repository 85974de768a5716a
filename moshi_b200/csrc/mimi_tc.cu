// mimi_tc_kernel: persistent TMA + wgmma tf32 implicit GEMM with 3xTF32 split products (see mimi_tc.cuh).
#include <cstdlib>
#include <cstring>

#include "mimi_tc.cuh"
#include "tc_host.cuh"
#include "tc_prims.cuh"

namespace b200 {
namespace mtc {

namespace {

using namespace tcp;

constexpr uint32_t A_TILE_BYTES = TC_ROWS * TC_KB * 4;      // 16 KB

struct Tile { int m, n, split, b0, t0, kb0, kb1; };

__device__ __forceinline__ Tile tile_at(const TcParams& p, int id) {
  Tile t;
  t.split = id % p.ksplit;
  const int mn = id / p.ksplit;
  t.n = mn % p.n_tiles_n;
  t.m = mn / p.n_tiles_n;
  const int tpg = (p.T + p.tt - 1) / p.tt;                  // tiles along the steps of one session group
  const int group = t.m / tpg, j = t.m - group * tpg;
  t.b0 = group * p.bb;
  t.t0 = j * p.tt;
  t.kb0 = t.split * p.kb_per_split;
  t.kb1 = min(p.num_kb, t.kb0 + p.kb_per_split);
  return t;
}

// Epilogue of V consecutive output features n0.. of GEMM row (b, t): shared by the kernel and the split-K reduction.
template <int V>
__device__ __forceinline__ void store_row_chunk(const TcParams& p, int b, int t, int n0, float* v) {
  if (p.epi == TC_EPI_GELU) {
#pragma unroll
    for (int i = 0; i < V; ++i) v[i] = gelu_erf(v[i]);
  } else if (p.epi == TC_EPI_RES_SCALE) {                       // x + layer_scale * update (transformer.py:769,777)
    const float* r = p.res + (long long)b * p.r_sb + (long long)t * p.r_row + n0;
#pragma unroll
    for (int i = 0; i < V; i += 2) {
      const float2 rv = *reinterpret_cast<const float2*>(r + i);
      const float2 sv = *reinterpret_cast<const float2*>(p.scale + n0 + i);
      v[i] = rv.x + sv.x * v[i]; v[i + 1] = rv.y + sv.y * v[i + 1];
    }
  } else {
    if (p.bias != nullptr) {
#pragma unroll
      for (int i = 0; i < V; ++i) v[i] += p.bias[(n0 + i) % p.bias_mod];
    }
    if (p.res != nullptr) {                                     // SEANetResnetBlock: u + v (seanet.py:90-93)
      const float* r = p.res + (long long)b * p.r_sb + (long long)t * p.r_row + n0;
#pragma unroll
      for (int i = 0; i < V; i += 2) {
        const float2 rv = *reinterpret_cast<const float2*>(r + i);
        v[i] += rv.x; v[i + 1] += rv.y;
      }
    }
  }
  if (p.y != nullptr) {
    float* y = p.y + (long long)b * p.y_sb + (long long)t * p.y_row + n0;
#pragma unroll
    for (int i = 0; i < V; i += 2) *reinterpret_cast<float2*>(y + i) = make_float2(v[i], v[i + 1]);
  }
  if (p.act_mode != TC_ACT_NONE) {
    if (p.act_elu) {
#pragma unroll
      for (int i = 0; i < V; ++i) v[i] = elu1(v[i]);
    }
    const long long o = (long long)b * p.a_sb + (long long)t * p.a_row + n0;
    if (p.act_mode == TC_ACT_FULL) {
#pragma unroll
      for (int i = 0; i < V; i += 2) *reinterpret_cast<float2*>(p.a_hi + o + i) = make_float2(v[i], v[i + 1]);
    } else {
      float lo[V];
#pragma unroll
      for (int i = 0; i < V; ++i) split_tf32(v[i], v[i], lo[i]);
#pragma unroll
      for (int i = 0; i < V; i += 2) {
        *reinterpret_cast<float2*>(p.a_hi + o + i) = make_float2(v[i], v[i + 1]);
        *reinterpret_cast<float2*>(p.a_lo + o + i) = make_float2(lo[i], lo[i + 1]);
      }
    }
  }
}

// NC: wgmma width; NT = nch * NC output features per tile (NC = 128 for full tiles, 16 for the narrow layers)
template <int NC>
__global__ void __launch_bounds__(TC_THREADS, 1)
mimi_tc_kernel(const __grid_constant__ CUtensorMap map_hi, const __grid_constant__ CUtensorMap map_lo, const TcParams p) {
  constexpr int MAXC = TC_MAX_NT / NC;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;                 // SWIZZLE_128B tiles need 1024 B alignment
  const uint32_t bars = base + (uint32_t)p.stages * p.stage_bytes;
  const uint32_t full0 = bars, empty0 = bars + 8 * TC_MAX_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tiles = p.m_tiles * p.n_tiles_n * p.ksplit;
  const uint32_t w_bytes = (uint32_t)p.NT * 128u;               // one weight tile (hi or lo)
  const int cb_per_tap = p.Cin / TC_KB;
  const int nch = p.NT / NC;

  if (warp == TC_PRODUCER_WARP && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_hi) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_lo) : "memory");
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, TC_CONSUMERS / 32);   // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_trigger();                                 // the next kernel of the frame may begin its own prologue and weight prefetch

  if (warp == TC_PRODUCER_WARP) {
    if (lane == 0) {
      // ===== producer =====
      // Programmatic dependent launch: the weights do not depend on the preceding kernel, so the first `stages` weight pairs of
      // this CTA's first tile are requested before the dependency wait (their HBM latency overlaps the predecessor's tail and
      // this kernel's own launch); the activation boxes, and everything the epilogue touches, come after it.
      int pre = 0;
      if ((int)blockIdx.x < n_tiles) {
        const Tile t0 = tile_at(p, blockIdx.x);
        const uint8_t* wsrc = p.wt + ((size_t)t0.n * p.num_kb + t0.kb0) * (size_t)(2 * w_bytes);
        for (int kb = t0.kb0; kb < t0.kb1 && pre < p.stages; ++kb, wsrc += 2 * w_bytes, ++pre) {
          mbar_expect_tx(full0 + 8 * pre, 2 * A_TILE_BYTES + 2 * w_bytes);
          bulk_load(base + (uint32_t)pre * p.stage_bytes + 2 * A_TILE_BYTES, wsrc, 2 * w_bytes, full0 + 8 * pre);
        }
      }
      pdl_wait();
      int s = 0; uint32_t ph = 0;
      int item = 0;
      for (int id = blockIdx.x; id < n_tiles; id += gridDim.x) {
        const Tile tl = tile_at(p, id);
        const uint8_t* wsrc = p.wt + ((size_t)tl.n * p.num_kb + tl.kb0) * (size_t)(2 * w_bytes);
        for (int kb = tl.kb0; kb < tl.kb1; ++kb, wsrc += 2 * w_bytes, ++item) {
          const int tap = kb / cb_per_tap, cb = kb - tap * cb_per_tap;
          const uint32_t sa = base + (uint32_t)s * p.stage_bytes;
          if (item >= pre) {
            mbar_wait(empty0 + 8 * s, ph ^ 1u);
            mbar_expect_tx(full0 + 8 * s, 2 * A_TILE_BYTES + 2 * w_bytes);
            bulk_load(sa + 2 * A_TILE_BYTES, wsrc, 2 * w_bytes, full0 + 8 * s);
          }
          const int row = p.row0 + tl.t0 * p.stride + tap * p.dil;
          tma_load_3d(sa, &map_hi, full0 + 8 * s, cb * TC_KB, row, tl.b0);
          tma_load_3d(sa + A_TILE_BYTES, &map_lo, full0 + 8 * s, cb * TC_KB, row, tl.b0);
          if (++s == p.stages) { s = 0; ph ^= 1u; }
        }
      }
    }
    return;
  }
  // ===== consumers: warpgroup wg owns GEMM rows 64 wg .. 64 wg + 63 (one (session, step) each) of every tile =====
  const int wg = warp >> 2, t = threadIdx.x & 127;
  uint32_t d[MAXC][NC / 2];
  int s = 0; uint32_t ph = 0;
  pdl_wait();                                    // outputs / residuals / the split-K workspace may still be in use by the predecessor
  for (int id = blockIdx.x; id < n_tiles; id += gridDim.x) {
    const Tile tl = tile_at(p, id);
    for (int kb = tl.kb0; kb < tl.kb1; ++kb) {
      mbar_wait(full0 + 8 * s, ph);
      const uint32_t a_hi = base + (uint32_t)s * p.stage_bytes + (uint32_t)wg * (A_TILE_BYTES / 2), a_lo = a_hi + A_TILE_BYTES;
      const uint32_t w_hi = base + (uint32_t)s * p.stage_bytes + 2 * A_TILE_BYTES, w_lo = w_hi + w_bytes;
      // per k-block 4 k-steps x (lo*hi + hi*lo + hi*hi): small terms first
      wg_fence();
#pragma unroll
      for (int k = 0; k < TC_KB / 8; ++k) {
        const uint32_t off = (uint32_t)k * 32u;          // 8 tf32 = 32 bytes of K per MMA
        const uint32_t first = (kb == tl.kb0 && k == 0) ? 0u : 1u;
#pragma unroll
        for (int c = 0; c < MAXC; ++c) {
          if (c < nch) {
            const uint32_t wc = (uint32_t)(c * NC) * 128u + off;
            Wgmma<NC>::tf32(d[c], make_desc(a_lo + off), make_desc(w_hi + wc), first);
            Wgmma<NC>::tf32(d[c], make_desc(a_hi + off), make_desc(w_lo + wc), 1u);
            Wgmma<NC>::tf32(d[c], make_desc(a_hi + off), make_desc(w_hi + wc), 1u);
          }
        }
      }
      wg_commit();
      wg_wait<0>();
#pragma unroll
      for (int c = 0; c < MAXC; ++c) wg_hold(d[c]);
      __syncwarp();
      if (lane == 0) mbar_arrive(empty0 + 8 * s);
      if (++s == p.stages) { s = 0; ph ^= 1u; }
    }
    // epilogue straight from the fragments: element pair (i, i + 1) = features n, n + 1 of GEMM row `row`
    const int n_base = tl.n * p.NT;
#pragma unroll
    for (int c = 0; c < MAXC; ++c) {
      if (c < nch) {
#pragma unroll
        for (int i = 0; i < NC / 2; i += 2) {
          const int row = 64 * wg + frag_row(t, i), n = n_base + c * NC + frag_col(t, i);
          const int bi = row / p.tt, ti = row - bi * p.tt;
          const int b = tl.b0 + bi, tt = tl.t0 + ti;
          float v[2] = {__uint_as_float(d[c][i]), __uint_as_float(d[c][i + 1])};
          if (p.ksplit > 1) {
            float* w = p.ws + ((size_t)tl.split * p.m_tiles * TC_ROWS + (size_t)tl.m * TC_ROWS + row) * (size_t)p.N + n;
            __stcg(reinterpret_cast<float2*>(w), make_float2(v[0], v[1]));
          } else if (b < p.n_sessions && tt < p.T) {
            store_row_chunk<2>(p, b, tt, n, v);
          }
        }
      }
    }
  }
}

// split-K: sum the partials in split order (deterministic) and run the epilogue; one thread per (row, 4 features)
__global__ void __launch_bounds__(256) mimi_tc_reduce_kernel(const TcParams p) {
  pdl_trigger();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int n4 = p.N / 4;
  const long long rows = (long long)p.m_tiles * TC_ROWS;
  if (i >= rows * n4) return;
  const long long grow = i / n4;
  const int n0 = (int)(i - grow * n4) * 4;
  const int m = (int)(grow / TC_ROWS), row = (int)(grow - (long long)m * TC_ROWS);
  const int tpg = (p.T + p.tt - 1) / p.tt;
  const int group = m / tpg, j = m - group * tpg;
  const int bi = row / p.tt, ti = row - bi * p.tt;
  const int b = group * p.bb + bi, t = j * p.tt + ti;
  if (b >= p.n_sessions || t >= p.T) return;
  float v[4] = {0.f, 0.f, 0.f, 0.f};
  for (int s = 0; s < p.ksplit; ++s) {
    const float4 a = __ldcg(reinterpret_cast<const float4*>(p.ws + ((size_t)s * rows + grow) * (size_t)p.N + n0));
    v[0] += a.x; v[1] += a.y; v[2] += a.z; v[3] += a.w;
  }
  store_row_chunk<4>(p, b, t, n0, v);
}

// load-time: w fp32 [N][n_taps * Cin] -> [n_tile][kb][hi | lo][NT rows][32] in the SWIZZLE_128B layout
// (16-byte chunk c of row r at r * 128 + ((c ^ (r & 7)) << 4)); rows beyond N are zero
__global__ void tc_pack_kernel(const float* __restrict__ w, float4* __restrict__ out, int N, int K, int NT, int n_tiles_n, int num_kb) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;      // one 16-byte chunk (4 floats) of a hi tile
  const long long per_tile = (long long)NT * 8;
  const long long total = (long long)n_tiles_n * num_kb * per_tile;
  if (idx >= total) return;
  const int chunk = (int)(idx % per_tile);
  long long t = idx / per_tile;
  const int kb = (int)(t % num_kb);
  const int nt = (int)(t / num_kb);
  const int r = chunk >> 3, cpos = chunk & 7;
  const int csrc = cpos ^ (r & 7);
  const int n = nt * NT + r, k = kb * TC_KB + csrc * 4;
  float hi[4] = {0.f, 0.f, 0.f, 0.f}, lo[4] = {0.f, 0.f, 0.f, 0.f};
  if (n < N) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (k + i < K) split_tf32(w[(long long)n * K + k + i], hi[i], lo[i]);
  }
  const long long o = (((long long)nt * num_kb + kb) * 2) * per_tile + chunk;
  out[o] = make_float4(hi[0], hi[1], hi[2], hi[3]);
  out[o + per_tile] = make_float4(lo[0], lo[1], lo[2], lo[3]);
}

bool g_attr = false;

}  // namespace

int tc_init() {
  if (!g_attr) {
    B200_CUDA(cudaFuncSetAttribute(mimi_tc_kernel<TC_MAX_NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
    B200_CUDA(cudaFuncSetAttribute(mimi_tc_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
    g_attr = true;
  }
  return B200_OK;
}

TcShape tc_shape(int kind, int N, int Cin, int n_taps, int dil, int stride, int bias_mod) {
  TcShape s;
  s.kind = kind; s.Cin = Cin; s.N = N; s.n_taps = n_taps; s.dil = dil; s.stride = stride;
  s.bias_mod = bias_mod > 0 ? bias_mod : N;
  s.NT = N >= TC_MAX_NT ? TC_MAX_NT : N;
  s.n_tiles_n = (N + s.NT - 1) / s.NT;
  s.num_kb = n_taps * (Cin / TC_KB);
  return s;
}

int plan_tc(const TcShape& s, int n_sessions, int T, int sms, size_t ws_bytes, TcSchedule* out) {
  if (n_sessions < 1 || T < 1 || sms < 1 || s.num_kb < 1 || s.NT < 1 || (s.kind == TC_LINEAR_ROWS && n_sessions != 1))
    B200_FAIL(B200_ERR_INVALID, "plan_tc: %d sessions of %d rows, %d SMs, %d k-blocks, kind %d", n_sessions, T, sms, s.num_kb, s.kind);
  TcSchedule q;
  q.n_sessions = n_sessions; q.T = T;
  q.tt = TC_ROWS;
  if (s.kind != TC_LINEAR_ROWS)
    while (q.tt > 1 && (T % q.tt || q.tt * s.stride > 256)) q.tt >>= 1;
  q.bb = TC_ROWS / q.tt;
  const int tpg = (T + q.tt - 1) / q.tt, groups = (n_sessions + q.bb - 1) / q.bb;
  q.m_tiles = tpg * groups;
  // deep-and-skinny layers: cut K so that the chip has a few hundred tiles, at least 4 k-blocks each
  int ks = 1;
  const long long mn = (long long)q.m_tiles * s.n_tiles_n;
  if (mn < sms && s.num_kb >= 8) {
    ks = (int)((2LL * sms + mn - 1) / mn);
    if (ks > s.num_kb / 4) ks = s.num_kb / 4;
    while (ks > 1 && (size_t)ks * q.m_tiles * TC_ROWS * (size_t)s.N * 4 > ws_bytes) --ks;
    if (ks < 1) ks = 1;
  }
  q.kb_per_split = (s.num_kb + ks - 1) / ks;
  q.ksplit = (s.num_kb + q.kb_per_split - 1) / q.kb_per_split;
  q.stage_bytes = 2 * A_TILE_BYTES + 2 * (uint32_t)s.NT * 128u;
  int stages = (200 * 1024) / (int)q.stage_bytes;
  if (stages > TC_MAX_STAGES) stages = TC_MAX_STAGES;
  q.stages = stages;
  const long long tiles = mn * q.ksplit;
  q.grid = (int)(tiles < sms ? tiles : sms);
  q.smem = (size_t)stages * q.stage_bytes + 1024 + 16 * TC_MAX_STAGES + 64;
  *out = q;
  return B200_OK;
}

size_t tc_packed_bytes(const TcShape& s) { return (size_t)s.n_tiles_n * s.num_kb * 2 * s.NT * 128; }

int tc_pack_weights(const float* w_dev, void* out_dev, const TcShape& s, cudaStream_t st) {
  if (s.Cin % TC_KB || s.N % 16 || (s.N > TC_MAX_NT && s.N % TC_MAX_NT))
    B200_FAIL(B200_ERR_SHAPE, "tc_pack_weights: Cin %d must be a multiple of 32, N %d a multiple of 16 (of 128 above 128)", s.Cin, s.N);
  const long long total = (long long)s.n_tiles_n * s.num_kb * s.NT * 8;
  tc_pack_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(w_dev, static_cast<float4*>(out_dev), s.N, s.n_taps * s.Cin, s.NT,
                                                                 s.n_tiles_n, s.num_kb);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return check_launch("tc_pack");
}

int tc_bind(TcLayer& L, const TcSchedule& q, const TcParams& epi, const float* in_hi, const float* in_lo, long long rows_per_session,
            float* ws) {
  B200_TRY(tc_init());
  const TcShape& s = L.s;
  TcParams& p = L.p;
  p = epi;
  p.tt = q.tt; p.bb = q.bb; p.T = q.T; p.n_sessions = q.n_sessions;
  p.n_taps = s.n_taps; p.dil = s.dil; p.stride = s.stride; p.row0 = 0; p.Cin = s.Cin;
  p.wt = L.wt; p.NT = s.NT; p.n_tiles_n = s.n_tiles_n; p.num_kb = s.num_kb; p.N = s.N;
  p.m_tiles = q.m_tiles; p.ksplit = q.ksplit; p.kb_per_split = q.kb_per_split; p.ws = ws;
  p.bias = L.bias; p.bias_mod = s.bias_mod;
  p.stage_bytes = q.stage_bytes; p.stages = q.stages;
  L.grid = q.grid; L.smem = q.smem;
  // 3-D maps over base[b][row][Cin]: a box of 32 channels x tt rows (element stride = conv stride) x bb sessions
  cuuint64_t dims[3] = {(cuuint64_t)s.Cin, (cuuint64_t)rows_per_session, (cuuint64_t)q.n_sessions};
  cuuint64_t strides[2] = {(cuuint64_t)s.Cin * 4, (cuuint64_t)(rows_per_session * s.Cin) * 4};
  cuuint32_t box[3] = {(cuuint32_t)TC_KB, (cuuint32_t)(q.tt * s.stride), (cuuint32_t)q.bb};
  cuuint32_t estr[3] = {1, (cuuint32_t)s.stride, 1};
  if (box[1] > 256 || box[2] > 256) B200_FAIL(B200_ERR_SHAPE, "tc_make_map: box %u x %u exceeds the TMA limit of 256", box[1], box[2]);
  B200_TRY(encode_tiled(&L.map_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, in_hi, dims, strides, box, estr, "tc_make_map"));
  return encode_tiled(&L.map_lo, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, in_lo, dims, strides, box, estr, "tc_make_map");
}

int tc_launch(const TcLayer& L, cudaStream_t st) {
  // programmatic dependent launch (B200_MIMI_PDL=0: off): the kernel may start while its predecessor drains; it requests its
  // first weight tiles, then waits (griddepcontrol.wait) before it reads an activation or writes anything
  static const int pdl = [] { const char* e = getenv("B200_MIMI_PDL"); return e ? atoi(e) : 1; }();
  B200_TRY(launch("mimi_tc", L.p.NT == TC_MAX_NT ? mimi_tc_kernel<TC_MAX_NT> : mimi_tc_kernel<16>, dim3((unsigned)L.grid), dim3(TC_THREADS),
                  L.smem, st, LaunchOpts{pdl}, L.map_hi, L.map_lo, L.p));
  if (L.p.ksplit > 1) {
    const long long n = (long long)L.p.m_tiles * TC_ROWS * (L.p.N / 4);
    mimi_tc_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(L.p);
    g_launches.fetch_add(1, std::memory_order_relaxed);
  }
  return check_launch("mimi_tc");
}

}  // namespace mtc
}  // namespace b200
