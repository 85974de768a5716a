// The Depth transformer of one frame as ONE persistent kernel (LMGen.depformer_step, lm.py:809-850, with
// LMModel.forward_depformer lm.py:450-493 and the weights-per-step layers of transformer.py:291-318 inside).
//
// The depformer is 8 dependent sub-steps x 6 layers of tiny GEMMs (1.23 GB of weights per frame, M = sessions):
// as separate launches that is ~430 kernels whose launch / set-up / drain latency is 10-20x their HBM time.
// Here one CTA per SM stays resident for the whole frame and the ~50 phases of a sub-step are separated by
// grid barriers (all CTAs are co-resident: cooperative launch, 1 CTA/SM by shared-memory size, grid <= #SMs):
//
//   per sub-step k:   [row phase]   x = depformer_in[k](transformer_out) + emb_k(prev token); xn = rmsnorm(x)
//     per layer l:    [GEMM]        in_proj partials            (wgmma, split-K units over all CTAs)
//                     [warp phase]  q,k,v = bf16(sum partials); KV append; attention over k+1 keys -> ao
//                     [GEMM]        out_proj partials
//                     [row phase]   x = bf16(x + bf16(sum)); xn = rmsnorm(x)
//                     [GEMM]        gated-MLP input partials (gate and value accumulators)
//                     [elem phase]  h = bf16(bf16(silu(g)) * u)
//                     [GEMM]        linear_out partials
//                     [row phase]   x = bf16(x + bf16(sum)); xn = rmsnorm(x) for the next layer
//                     ...
//                     [GEMM]        logits partials (linears[k])
//                     [row phase]   logits = bf16(sum) ; token = sample(logits) ; next sub-step's input row
//
// GEMM phases use the same machinery as gemm_sk.cu (pre-tiled SWIZZLE_128B weights streamed by cp.async.bulk, the
// activation box by 2-D TMA, wgmma into register accumulators of one consumer warpgroup, epilogue from the fragments); a
// unit = (128-row weight tile, k-split, block of 64 sessions) and every unit writes its fp32 partial [64 x 128] to an
// L2-resident workspace; the consumer phase
// sums the splits in split order (deterministic, independent of the batch) and applies the reference's cast points.
#include "gemm_sk.cuh"
#include "tc_prims.cuh"
#include "lm_kernels.cuh"

namespace b200 {
namespace tc {

namespace {

using lm::bf16;

constexpr int BLOCK_ROWS = 128, BLOCK_K = 64, UMMA_K = 16;
constexpr int THREADS = 256;                 // GEMM phases: warp 0 producer, warps 4-7 the consumer warpgroup; all in the SIMT phases
constexpr int MC = 64;                       // sessions per GEMM unit (wgmma N): the warpgroup holds 128 rows x MC x 2 accumulators
constexpr int TILE_BYTES = BLOCK_ROWS * BLOCK_K * 2;
constexpr int MAX_STAGES = 8;
constexpr int DD = 64;                       // depformer head dim
static_assert(THREADS == lm::SAMPLE_THREADS, "sample_row needs a SAMPLE_THREADS-wide CTA");

using namespace tcp;
__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

struct Pipe { int s; uint32_t ph; int pre; };   // per-role pipeline cursor, carried across phases
// (pre: producer only — stages of the upcoming GEMM phase whose weight copy is already in flight)

// Grid barrier: one release-reduction per CTA and acquire polling by one thread (all CTAs are co-resident).
// The CTA's own writes are ordered before the reduction by __syncthreads (cumulativity of the gpu-scope release).
__device__ __forceinline__ void grid_sync(unsigned* bar, unsigned& epoch, unsigned long long* trace = nullptr) {
  __syncthreads();
  if (threadIdx.x == 0) {
    epoch += 1;
    const unsigned target = epoch * gridDim.x;
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(bar) : "memory");
    unsigned spins = 0;
    uint64_t t0 = 0;
    while (ld_acquire(bar) < target) {               // all CTAs are co-resident (cooperative launch): bounded by wall clock only
      if ((++spins & 4095u) == 0u) {
        const uint64_t now = global_timer_ns();
        if (t0 == 0) t0 = now;
        else if (now - t0 > WAIT_LIMIT_NS) __trap();
      }
    }
    if (trace != nullptr && blockIdx.x == 0 && epoch < (unsigned)DEP_TRACE_SLOTS) trace[epoch] = global_timer_ns();
  }
  __syncthreads();
}

__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < THREADS / 32; ++w) t += red[w];
  return t;
}

// rows handled by this CTA: m = blockIdx.x, blockIdx.x + gridDim.x, ...   (same mapping in every row phase, so a row's
// sampled token is consumed by the CTA that produced it without a barrier)
//   x_new = has_sum ? bf16(x + bf16(sum_s part[s][m][:])) : x (already written);  xn = rmsnorm(x_new, alpha)
template <int NV, class P>                                    // dd <= NV * THREADS
__device__ void row_phase(const P& p, int dd, int S, const float* part, int N, bool has_sum, const bf16* alpha, float* red) {
  for (int m = blockIdx.x; m < p.B; m += gridDim.x) {
    float vals[NV];
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int j = threadIdx.x + i * THREADS;
      float v = 0.f;
      if (j < dd) {
        v = bf2f(p.x[(long long)m * dd + j]);
        if (has_sum) {
          float a = 0.f;
          for (int s = 0; s < S; ++s) a += __ldcg(part + ((long long)s * p.B + m) * N + j);
          v = rbf(v + rbf(a));                                // x_orig + update, both bf16 (transformer.py:769,777)
          p.x[(long long)m * dd + j] = f2bf(v);
        }
        ss += v * v;
      }
      vals[i] = v;
    }
    if (alpha != nullptr) {
      const float tot = block_sum(ss, red);
      const float r = rsqrtf(1e-8f + tot / (float)dd);
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int j = threadIdx.x + i * THREADS;
        if (j < dd) p.xn[(long long)m * dd + j] = f2bf(vals[i] * (bf2f(alpha[j]) * r));
      }
    }
  }
}

// x = depformer_in[schedule[k]](transformer_out) + emb_k(prev)   (lm.py:475-486; token -1 -> zero row, lm_utils.py:103-121)
__device__ void input_rows(const DepParams& p, int k) {
  const long long* prev = k == 0 ? p.text_token : p.audio_tokens + (long long)(k - 1) * p.B;
  const bf16* table = p.tables[k];
  const bf16* din = p.din + p.din_col[k];
  for (int m = blockIdx.x; m < p.B; m += gridDim.x) {
    const long long id = prev[m];
    const bool ok = lm::embed_id_ok(id, k == 0 ? p.text_card : p.card, p.err);
    for (int j = threadIdx.x; j < p.dd; j += THREADS) {
      const float e = ok ? bf2f(table[id * p.dd + j]) : 0.f;
      p.x[(long long)m * p.dd + j] = f2bf(bf2f(din[(long long)m * p.din_ld + j]) + e);
    }
  }
  __syncthreads();                                            // row_phase re-reads x written by other threads of this CTA
}

// q,k,v = bf16(sum of in_proj partials); append k,v at slot `step`; attention over step+1 keys (no RoPE in the depformer)
__device__ void attn_phase(const DepParams& p, int S, int layer, int step) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int C = p.dd, N = 3 * C;
  bf16* kc = p.kc[layer];
  bf16* vc = p.vc[layer];
  for (int it = blockIdx.x * (THREADS / 32) + warp; it < p.B * p.H; it += gridDim.x * (THREADS / 32)) {
    const int b = it / p.H, h = it - b * p.H;
    float q[2] = {0.f, 0.f}, kk[2] = {0.f, 0.f}, vv[2] = {0.f, 0.f};
    for (int s = 0; s < S; ++s) {
      const float* row = p.part0 + ((long long)s * p.B + b) * N + h * DD + 2 * lane;
      const float2 a = __ldcg(reinterpret_cast<const float2*>(row));
      const float2 c = __ldcg(reinterpret_cast<const float2*>(row + C));
      const float2 d = __ldcg(reinterpret_cast<const float2*>(row + 2 * C));
      q[0] += a.x; q[1] += a.y; kk[0] += c.x; kk[1] += c.y; vv[0] += d.x; vv[1] += d.y;
    }
    const long long rowo = ((long long)b * p.H + h) * p.dep_q;
    *reinterpret_cast<__nv_bfloat162*>(kc + (rowo + step) * DD + 2 * lane) = __floats2bfloat162_rn(kk[0], kk[1]);
    *reinterpret_cast<__nv_bfloat162*>(vc + (rowo + step) * DD + 2 * lane) = __floats2bfloat162_rn(vv[0], vv[1]);
    __syncwarp();
    const float qx = rbf(q[0]), qy = rbf(q[1]);
    float sc[lm::DEP_MAX_Q];
    float mx = -INFINITY;
    for (int j = 0; j <= step; ++j) {
      const float2 kv = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(kc + (rowo + j) * DD + 2 * lane));
      const float d = warp_sum(qx * kv.x + qy * kv.y) * 0.125f;
      sc[j] = d;
      mx = fmaxf(mx, d);
    }
    float sum = 0.f;
    for (int j = 0; j <= step; ++j) { sc[j] = expf(sc[j] - mx); sum += sc[j]; }
    const float inv = 1.f / sum;
    float a0 = 0.f, a1 = 0.f;
    for (int j = 0; j <= step; ++j) {
      const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(vc + (rowo + j) * DD + 2 * lane));
      a0 = fmaf(sc[j] * inv, v.x, a0);
      a1 = fmaf(sc[j] * inv, v.y, a1);
    }
    *reinterpret_cast<__nv_bfloat162*>(p.ao + (long long)b * C + h * DD + 2 * lane) = __floats2bfloat162_rn(a0, a1);
  }
}

// h = bf16(bf16(silu(bf16 gate)) * bf16 value)   (gating.py:18-20)
template <class P>
__device__ void gate_phase(const P& p, int S) {
  const long long total = (long long)p.B * p.F;
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < total; i += (long long)gridDim.x * THREADS) {
    float g = 0.f, u = 0.f;
    for (int s = 0; s < S; ++s) {
      g += __ldcg(p.part0 + (long long)s * total + i);
      u += __ldcg(p.part1 + (long long)s * total + i);
    }
    g = rbf(g); u = rbf(u);
    p.hbuf[i] = f2bf(rbf(g / (1.f + expf(-g))) * u);
  }
}

// logits = bf16(sum partials) -> sample -> audio_tokens[k]
__device__ void sample_phase(const DepParams& p, int S, int k) {
  for (int m = blockIdx.x; m < p.B; m += gridDim.x) {
    bf16* lg = p.logits + ((long long)k * p.B + m) * p.card;
    for (int j = threadIdx.x; j < p.card; j += THREADS) {
      float a = 0.f;
      for (int s = 0; s < S; ++s) a += __ldcg(p.part0 + ((long long)s * p.B + m) * p.card + j);
      lg[j] = f2bf(a);
    }
    __syncthreads();
    float temp = p.temp;
    int top_k = p.top_k;
    lm::row_sampling(p.rows, m, false, &temp, &top_k);
    lm::sample_row(lg, p.noise + (long long)m * p.noise_ld + p.noise_off + (long long)k * p.ka, p.audio_tokens + (long long)k * p.B + m,
                   p.card, p.use_sampling, temp, top_k);
    __syncthreads();
  }
}

// One GEMM phase: units u = blockIdx.x, += gridDim.x; unit = (tile, split, block of MC sessions), the session block fastest
// (the CTAs that share a weight slice run side by side, so all but the first read it from L2);
// partial [MC x 128] -> part[split][m][tile*128 + row]
__device__ __forceinline__ void unit_at(const Gemm& g, int mch, int u, int& tile, int& sp, int& mc) {
  mc = u % mch;
  const int ts = u / mch;
  tile = ts / g.S;
  sp = ts - tile * g.S;
}

template <class P>
__device__ void gemm_phase(const P& p, const Gemm& g, const Gemm* next, const CUtensorMap* xmap, uint32_t base, uint32_t full0,
                           uint32_t empty0, Pipe& pipe) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int mch = (p.B + MC - 1) / MC;
  const int units = g.n_tiles * g.S * mch;
  const uint32_t a_bytes = (uint32_t)g.A * TILE_BYTES;
  constexpr uint32_t x_bytes = (uint32_t)MC * BLOCK_K * 2;
  if (warp == 0) {
    if (lane == 0) {
      asm volatile("fence.proxy.async;" ::: "memory");        // activations were written with generic stores by other CTAs
      int item = 0;
      for (int u = blockIdx.x; u < units; u += gridDim.x) {
        int tile, sp, mc;
        unit_at(g, mch, u, tile, sp, mc);
        const int kb0 = sp * g.kbps, kb1 = min(g.num_kb, kb0 + g.kbps);
        const uint8_t* src = g.wt + ((size_t)tile * g.num_kb + kb0) * a_bytes;
        for (int kb = kb0; kb < kb1; ++kb, src += a_bytes, ++item) {
          const uint32_t sa = base + (uint32_t)pipe.s * p.stage_bytes;
          if (item >= pipe.pre) {                              // (else: requested at the end of the previous GEMM phase)
            mbar_wait(empty0 + 8 * pipe.s, pipe.ph ^ 1u);
            mbar_expect_tx(full0 + 8 * pipe.s, a_bytes + x_bytes);
            bulk_load(sa, src, a_bytes, full0 + 8 * pipe.s);
          }
          tma_load_2d(sa + 2 * TILE_BYTES, xmap, full0 + 8 * pipe.s, kb * BLOCK_K, mc * MC);
          if (++pipe.s == p.stages) { pipe.s = 0; pipe.ph ^= 1u; }
        }
      }
      // Weights never depend on the phases in between: request the next GEMM phase's first tiles now, so its HBM
      // latency (and, at large batch, most of its stream) overlaps the SIMT phase and the two grid barriers ahead.
      pipe.pre = 0;
      if (next != nullptr) {
        const uint32_t nb = (uint32_t)next->A * TILE_BYTES;
        int s2 = pipe.s; uint32_t ph2 = pipe.ph;
        const int nunits = next->n_tiles * next->S * mch;
        for (int u = blockIdx.x; u < nunits && pipe.pre < p.stages; u += gridDim.x) {
          int tile, sp, mc;
          unit_at(*next, mch, u, tile, sp, mc);
          const int kb0 = sp * next->kbps, kb1 = min(next->num_kb, kb0 + next->kbps);
          const uint8_t* src = next->wt + ((size_t)tile * next->num_kb + kb0) * nb;
          for (int kb = kb0; kb < kb1 && pipe.pre < p.stages; ++kb, src += nb, ++pipe.pre) {
            mbar_wait(empty0 + 8 * s2, ph2 ^ 1u);
            mbar_expect_tx(full0 + 8 * s2, nb + x_bytes);
            bulk_load(base + (uint32_t)s2 * p.stage_bytes, src, nb, full0 + 8 * s2);
            if (++s2 == p.stages) { s2 = 0; ph2 ^= 1u; }
          }
        }
      }
    }
  } else if (warp >= 4) {
    // the consumer warpgroup: weight rows 0..63 and 64..127 of the tile (h), one accumulator per weight tile (a)
    const int t = threadIdx.x & 127;
    for (int u = blockIdx.x; u < units; u += gridDim.x) {
      int tile, sp, mc;
      unit_at(g, mch, u, tile, sp, mc);
      const int kb0 = sp * g.kbps, kb1 = min(g.num_kb, kb0 + g.kbps);
      uint32_t d00[MC / 2], d01[MC / 2], d10[MC / 2], d11[MC / 2];    // d<h><a>
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(full0 + 8 * pipe.s, pipe.ph);
        const uint32_t sa = base + (uint32_t)pipe.s * p.stage_bytes;
        const uint32_t sb = sa + 2 * TILE_BYTES;
        wg_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / UMMA_K; ++k) {
          const uint64_t db = make_desc(sb + k * UMMA_K * 2);
          const uint32_t accum = (kb == kb0 && k == 0) ? 0u : 1u;
          const uint32_t a0 = sa + k * UMMA_K * 2;
          Wgmma<MC>::bf16(d00, make_desc(a0), db, accum);
          Wgmma<MC>::bf16(d10, make_desc(a0 + TILE_BYTES / 2), db, accum);
          if (g.A == 2) {
            Wgmma<MC>::bf16(d01, make_desc(a0 + TILE_BYTES), db, accum);
            Wgmma<MC>::bf16(d11, make_desc(a0 + TILE_BYTES + TILE_BYTES / 2), db, accum);
          }
        }
        wg_commit();
        wg_wait<0>();
        wg_hold(d00); wg_hold(d10);
        if (g.A == 2) { wg_hold(d01); wg_hold(d11); }
        __syncwarp();
        if (lane == 0) mbar_arrive(empty0 + 8 * pipe.s);
        if (++pipe.s == p.stages) { pipe.s = 0; pipe.ph ^= 1u; }
      }
      float* o0 = p.part0 + (long long)sp * p.B * g.N;
      float* o1 = p.part1 + (long long)sp * p.B * g.N;
#pragma unroll
      for (int i = 0; i < MC / 2; ++i) {
        const int m = mc * MC + frag_col(t, i);
        const int n0 = tile * BLOCK_ROWS + frag_row(t, i), n1 = n0 + 64;
        if (m < p.B) {
          if (n0 < g.N) {
            __stcg(o0 + (long long)m * g.N + n0, __uint_as_float(d00[i]));
            if (g.A == 2) __stcg(o1 + (long long)m * g.N + n0, __uint_as_float(d01[i]));
          }
          if (n1 < g.N) {
            __stcg(o0 + (long long)m * g.N + n1, __uint_as_float(d10[i]));
            if (g.A == 2) __stcg(o1 + (long long)m * g.N + n1, __uint_as_float(d11[i]));
          }
        }
      }
    }
  }
}

__global__ void __launch_bounds__(THREADS, 1)
dep_fused_kernel(const __grid_constant__ CUtensorMap map_xn, const __grid_constant__ CUtensorMap map_ao,
                 const __grid_constant__ CUtensorMap map_h, const __grid_constant__ CUtensorMap map_x, const DepParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ float red[THREADS / 32];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const uint32_t bars = base + (uint32_t)p.stages * p.stage_bytes;
  const uint32_t full0 = bars, empty0 = bars + 8 * MAX_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_xn) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_ao) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_h) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_x) : "memory");
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, 4);          // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  Pipe pipe{0, 0u, 0};
  unsigned epoch = 0;
  if (p.trace != nullptr && blockIdx.x == 0 && threadIdx.x == 0) p.trace[0] = global_timer_ns();
  // GEMM phases in execution order: per sub-step k, per layer l: in_proj, out_proj, linear_in, linear_out; then the head
  auto gemm_at = [&](int k, int l, int which) -> Gemm {
    Gemm g;
    if (which == 4) { g = p.g_head; g.wt = p.heads[k]; return g; }
    const DepLayerW w = p.w[k * p.L + l];
    if (which == 0) { g = p.g_in; g.wt = w.in_w; }
    else if (which == 1) { g = p.g_out; g.wt = w.out_w; }
    else if (which == 2) { g = p.g_lin_in; g.wt = w.lin_in; }
    else { g = p.g_lin_out; g.wt = w.lin_out; }
    return g;
  };
  Gemm cur = gemm_at(0, 0, 0);
  for (int k = 0; k < p.dep_q; ++k) {
    input_rows(p, k);
    row_phase<4>(p, p.dd, 0, nullptr, 0, false, p.n1[0], red);
    grid_sync(p.bar, epoch, p.trace);
    for (int l = 0; l < p.L; ++l) {
      Gemm nxt = gemm_at(k, l, 1);
      gemm_phase(p, cur, &nxt, &map_xn, base, full0, empty0, pipe);
      grid_sync(p.bar, epoch, p.trace);
      attn_phase(p, cur.S, l, k);
      grid_sync(p.bar, epoch, p.trace);
      cur = nxt; nxt = gemm_at(k, l, 2);
      gemm_phase(p, cur, &nxt, &map_ao, base, full0, empty0, pipe);
      grid_sync(p.bar, epoch, p.trace);
      row_phase<4>(p, p.dd, cur.S, p.part0, cur.N, true, p.n2[l], red);
      grid_sync(p.bar, epoch, p.trace);
      cur = nxt; nxt = gemm_at(k, l, 3);
      gemm_phase(p, cur, &nxt, &map_xn, base, full0, empty0, pipe);
      grid_sync(p.bar, epoch, p.trace);
      gate_phase(p, cur.S);
      grid_sync(p.bar, epoch, p.trace);
      cur = nxt; nxt = l + 1 < p.L ? gemm_at(k, l + 1, 0) : gemm_at(k, 0, 4);
      gemm_phase(p, cur, &nxt, &map_h, base, full0, empty0, pipe);
      grid_sync(p.bar, epoch, p.trace);
      // depformer_norms is Identity (lm.py:197-198): after the last layer the head reads x itself
      row_phase<4>(p, p.dd, cur.S, p.part0, cur.N, true, l + 1 < p.L ? p.n1[l + 1] : nullptr, red);
      grid_sync(p.bar, epoch, p.trace);
      cur = nxt;
    }
    const bool last = k + 1 == p.dep_q;
    Gemm nxt = last ? cur : gemm_at(k + 1, 0, 0);
    gemm_phase(p, cur, last ? nullptr : &nxt, &map_x, base, full0, empty0, pipe);
    grid_sync(p.bar, epoch, p.trace);
    sample_phase(p, cur.S, k);       // the next sub-step's input rows are the same rows of the same CTA: no barrier needed
    cur = nxt;
  }
}

Gemm plan(int N, int K, int A, int M, int grid) {
  Gemm g;
  g.wt = nullptr; g.A = A; g.N = N;
  g.n_tiles = (N + BLOCK_ROWS - 1) / BLOCK_ROWS;
  g.num_kb = (K + BLOCK_K - 1) / BLOCK_K;
  // splits: enough units for ~2 per CTA, but the fp32 partials (written + re-read through L2) stay under ~6 MB (12 MB gated)
  long long want = (2LL * grid + g.n_tiles - 1) / g.n_tiles;
  const long long per_split = (long long)M * N * 4 * A;
  long long cap = ((long long)(A == 2 ? 12 : 6) << 20) / (per_split > 0 ? per_split : 1);
  if (cap < 1) cap = 1;
  long long S = want < cap ? want : cap;
  if (S > g.num_kb) S = g.num_kb;
  if (S < 1) S = 1;
  g.kbps = (int)((g.num_kb + S - 1) / S);
  g.S = (g.num_kb + g.kbps - 1) / g.kbps;
  return g;
}

}  // namespace

int plan_depformer(int dep_q, int dd, int H, int F, int card, int B, bool cfg, bool i8, int sms, int gemv_max_m, int mode,
                   DepformerPlan* out) {
  if (!out || dep_q < 0 || dep_q > lm::DEP_MAX_Q || (dep_q > 0 && (dd < 1 || H < 1 || F < 1 || card < 1)) || B < 1 ||
      (cfg ? 2 * B : B) > 256 || sms < 1 || gemv_max_m < 0 || gemv_max_m > 4 || mode < B200_DEPFORMER_AUTO || mode > B200_DEPFORMER_FUSED)
    B200_FAIL(B200_ERR_INVALID, "depformer plan: dep_q %d, dd %d, %d sessions, %d SMs, GEMV rows %d, mode %d out of range", dep_q, dd, B,
              sms, gemv_max_m, mode);
  DepformerPlan& P = *out;
  memset(&P, 0, sizeof(P));
  P.path = dep_q == 0 ? DEP_NONE : DEP_CHAIN;
  // One or two sessions: the depformer's linears take the GEMV path and the PDL-chained launches beat the persistent kernel
  // (a grid barrier per phase costs more than the launch it saves); B200_DEPFORMER_FUSED takes the kernel at any batch.  Under
  // classifier-free guidance the two halves of the batch meet before every sampler (lm.py:828-833), and the kernel has no int8
  // GEMM phases: launch chain.  Its row phases hold dd <= 4 * THREADS in registers.
  if (dep_q == 0 || mode == B200_DEPFORMER_CHAIN || cfg || i8 || (B <= gemv_max_m && mode != B200_DEPFORMER_FUSED) || dd > 4 * THREADS ||
      dd % 64)
    return B200_OK;
  if (dd / H != DD || F % 8) B200_FAIL(B200_ERR_INVALID, "fused depformer: unsupported configuration");
  P.stage_bytes = 2 * TILE_BYTES + MC * BLOCK_K * 2;
  P.stages = std::min((200 * 1024) / P.stage_bytes, MAX_STAGES);
  if (P.stages < 2) B200_FAIL(B200_ERR_INVALID, "fused depformer: batch too large for the stage ring");
  P.path = DEP_FUSED;
  P.grid = sms;
  P.g_in = plan(3 * dd, dd, 1, B, sms);
  P.g_out = plan(dd, dd, 1, B, sms);
  P.g_lin_in = plan(F, dd, 2, B, sms);
  P.g_lin_out = plan(dd, F, 1, B, sms);
  P.g_head = plan(card, dd, 1, B, sms);
  for (const Gemm* g : {&P.g_in, &P.g_out, &P.g_lin_in, &P.g_lin_out, &P.g_head})
    P.part_floats = std::max(P.part_floats, (long long)g->S * B * g->N);
  P.smem = P.stages * P.stage_bytes + 1024 + 16 * MAX_STAGES + 64;
  return B200_OK;
}

// ---- host side -------------------------------------------------------------------------------------------------------
struct DepFused {
  DepParams p;
  CUtensorMap map_xn, map_ao, map_h, map_x;
  int grid = 0; size_t smem = 0;
  void* dev_tables = nullptr;     // one allocation holding the pointer tables
};

int dep_fused_create(const DepformerPlan& P, const DepParams& host, DepFused** out) {
  if (P.path != DEP_FUSED) B200_FAIL(B200_ERR_INVALID, "fused depformer: the plan takes another path");
  DepFused* d = new DepFused();
  DepParams& p = d->p;
  p = host;
  d->grid = P.grid;
  p.Mpad = ((p.B + 15) / 16) * 16;
  p.stages = P.stages; p.stage_bytes = (uint32_t)P.stage_bytes;
  p.g_in = P.g_in; p.g_out = P.g_out; p.g_lin_in = P.g_lin_in; p.g_lin_out = P.g_lin_out; p.g_head = P.g_head;
  // pointer tables and the din columns -> one device allocation
  const size_t nq = (size_t)p.dep_q * 8, nl = (size_t)p.L * 8;
  const void* src[8] = {host.w, host.heads, host.tables, host.n1, host.n2, host.kc, host.vc, host.din_col};
  const size_t n[8] = {p.dep_q * p.L * sizeof(DepLayerW), nq, nq, nl, nl, nl, nl, (size_t)p.dep_q * sizeof(int)};
  size_t off[9] = {0};
  for (int i = 0; i < 8; ++i) off[i + 1] = off[i] + n[i];
  std::vector<uint8_t> hp(off[8]);
  for (int i = 0; i < 8; ++i) memcpy(hp.data() + off[i], src[i], n[i]);
  if (cudaMalloc(&d->dev_tables, off[8]) != cudaSuccess) { delete d; B200_FAIL(B200_ERR_CUDA, "fused depformer: cudaMalloc failed"); }
  B200_CUDA(cudaMemcpy(d->dev_tables, hp.data(), off[8], cudaMemcpyHostToDevice));
  uint8_t* dv = static_cast<uint8_t*>(d->dev_tables);
  p.w = reinterpret_cast<const DepLayerW*>(dv + off[0]);
  p.heads = reinterpret_cast<const uint8_t* const*>(dv + off[1]);
  p.tables = reinterpret_cast<const bf16* const*>(dv + off[2]);
  p.n1 = reinterpret_cast<const bf16* const*>(dv + off[3]);
  p.n2 = reinterpret_cast<const bf16* const*>(dv + off[4]);
  p.kc = reinterpret_cast<bf16* const*>(dv + off[5]);
  p.vc = reinterpret_cast<bf16* const*>(dv + off[6]);
  p.din_col = reinterpret_cast<const int*>(dv + off[7]);
  B200_TRY(act_map(&d->map_xn, p.xn, p.dd, p.B, p.dd, MC, 2));
  B200_TRY(act_map(&d->map_ao, p.ao, p.dd, p.B, p.dd, MC, 2));
  B200_TRY(act_map(&d->map_h, p.hbuf, p.F, p.B, p.F, MC, 2));
  B200_TRY(act_map(&d->map_x, p.x, p.dd, p.B, p.dd, MC, 2));
  d->smem = (size_t)P.smem;
  B200_CUDA(cudaFuncSetAttribute(dep_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  int per_sm = 0, coop = 0, dev = 0;
  B200_CUDA(cudaGetDevice(&dev));
  B200_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
  B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, dep_fused_kernel, THREADS, d->smem));
  if (!coop || per_sm < 1) {
    dep_fused_destroy(d);
    B200_FAIL(B200_ERR_CUDA, "fused depformer: the device cannot co-schedule %d CTAs of %zu B shared memory", d->grid, d->smem);
  }
  *out = d;
  return B200_OK;
}

void dep_fused_set_sampling(DepFused* d, int use_sampling, float temp, int top_k) {
  if (!d) return;
  d->p.use_sampling = use_sampling; d->p.temp = temp; d->p.top_k = top_k;
}

void dep_fused_destroy(DepFused* d) {
  if (!d) return;
  if (d->dev_tables) cudaFree(d->dev_tables);
  delete d;
}

// Cooperative launch: the driver guarantees that all CTAs of the grid are co-resident (or fails the launch), so the grid
// barrier cannot deadlock against another handle's persistent kernel, an MPS neighbour or a second replica on the same GPU.
int dep_fused_launch(DepFused* d, cudaStream_t stream) {
  B200_CUDA(cudaMemsetAsync(d->p.bar, 0, sizeof(unsigned), stream));
  LaunchOpts o;
  o.cooperative = true;
  return launch("dep_fused", dep_fused_kernel, dim3((unsigned)d->grid), dim3(THREADS), d->smem, stream, o, d->map_xn, d->map_ao, d->map_h,
                d->map_x, d->p);
}

}  // namespace tc
}  // namespace b200
