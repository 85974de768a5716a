// SIMT fp32 kernels of the Mimi codec: the learnt down-sampling conv, the depth-wise up-sampling, state commits and resets,
// the residual VQ and load-time re-layouts.  Every other contraction of the codec is on the tensor cores (mimi_tc.cuh).
// The down-sampling conv and the RVQ run in plain fp32 FMA arithmetic (no TF32 / bf16) because the RVQ indices must match
// the reference's.
//
// Activations are addressed through explicit (batch, channel, time) strides, so a kernel can read / write either the
// reference's [B, C, T] layout or the token-major [B, T, C] layout of the transformer kernels without a transposition.
#pragma once

#include "common.cuh"

namespace b200 {
namespace mimi {

// ---------------------------------------------------------------------------------------------
// StreamingConv1d (conv.py:245-274) as a split-K fp32 GEMM over packed weights [M = Cout][Kd = K * Cin] (tap-major, channel
// fastest) and N = sessions x Tout output columns.
// ---------------------------------------------------------------------------------------------
struct ConvSplitK {
  const float* x; long long xb, xc, xt; int Tin;   // input x[b][ci][t] through strides, Tin steps
  float* st; int P;                  // carried left context [B][Cin][P]
  uint8_t* first;                    // replicate-pad flags [B] or nullptr
  const float* w; const float* bias; // [M][Kd]; [M] or nullptr
  float* y; long long yb, yc, yt;
  int Cin, stride, dil, Tout, elu_in;
  int M, N, Kd;

  __device__ __forceinline__ float ext(int b, int ci, int j) const {
    // sample j of cat(previous, x) for row b, channel ci   (conv.py:261)
    if (j < P) {
      if (first != nullptr && first[b]) {           // conv.py:254-259 (replicate mode, first step)
        float v = x[b * xb + ci * xc];
        return elu_in ? elu1(v) : v;
      }
      return st[((long long)b * Cin + ci) * P + j];
    }
    float v = x[b * xb + ci * xc + (long long)(j - P) * xt];
    return elu_in ? elu1(v) : v;
  }
};

// ---------------------------------------------------------------------------------------------
// Deep-and-skinny convolution (the learnt down-sampling conv, resample.py:14-65: Cin = Cout = 512, K = 4, one output step
// per frame): N = sessions x T_out columns against K * Cin = 2048 reduction steps and 4 MB of weights.  As a plain tile
// GEMM that is 16 CTAs walking 2048 k each (249 us at 104 sessions, 209 us at one); here the reduction is cut into KS
// slices so that (Cout / 64) x KS CTAs stream the weights once, and a second pass adds the slices in slice order
// (deterministic).  The partials take KS * N * M floats.
// ---------------------------------------------------------------------------------------------
constexpr int DS_CO = 64, DS_KP = 64, DS_NC = 32;
inline int ds_splits(int Kd) { return ceil_div(Kd, DS_KP); }     // KS for Kd = K * Cin reduction steps
static __global__ void __launch_bounds__(256) conv_splitk_kernel(const ConvSplitK p, float* __restrict__ part, int KS) {
  __shared__ float ws[DS_KP][DS_CO + 1];
  __shared__ float xs[DS_KP][DS_NC + 1];
  const int tid = threadIdx.x;
  const int co0 = blockIdx.x * DS_CO, k0 = blockIdx.y * DS_KP;
  for (int idx = tid; idx < DS_CO * DS_KP; idx += 256) {
    const int co = idx / DS_KP, kk = idx - co * DS_KP;
    ws[kk][co] = (co0 + co < p.M && k0 + kk < p.Kd) ? p.w[(long long)(co0 + co) * p.Kd + k0 + kk] : 0.f;
  }
  const int co = tid & 63, ng = tid >> 6;
  for (int n0 = 0; n0 < p.N; n0 += DS_NC) {
    __syncthreads();
    for (int idx = tid; idx < DS_KP * DS_NC; idx += 256) {
      const int n = idx / DS_KP, kk = idx - n * DS_KP;
      float v = 0.f;
      if (n0 + n < p.N && k0 + kk < p.Kd) {
        const int b = (n0 + n) / p.Tout, t = (n0 + n) - b * p.Tout;
        const int kw = (k0 + kk) / p.Cin, ci = (k0 + kk) - kw * p.Cin;
        v = p.ext(b, ci, t * p.stride + kw * p.dil);
      }
      xs[kk][n] = v;
    }
    __syncthreads();
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll 8
    for (int kk = 0; kk < DS_KP; ++kk) {
      const float w = ws[kk][co];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = fmaf(w, xs[kk][ng * 8 + j], acc[j]);
    }
    if (co0 + co < p.M) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int n = n0 + ng * 8 + j;
        if (n < p.N) part[((long long)blockIdx.y * p.N + n) * p.M + co0 + co] = acc[j];
      }
    }
  }
  (void)KS;
}
static __global__ void __launch_bounds__(256) conv_splitk_reduce_kernel(const ConvSplitK p, const float* __restrict__ part, int KS) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= (long long)p.N * p.M) return;
  const int n = (int)(i / p.M), m = (int)(i - (long long)n * p.M);
  float a = 0.f;
  for (int s0 = 0; s0 < KS; s0 += 8) {            // 8 independent loads in flight, added in slice order
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = s0 + j < KS ? part[((long long)(s0 + j) * p.N + n) * p.M + m] : 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) a += v[j];
  }
  const int b = n / p.Tout, t = n - b * p.Tout;
  p.y[b * p.yb + m * p.yc + t * p.yt] = a + (p.bias ? p.bias[m] : 0.f);
}

// ---------------------------------------------------------------------------------------------
// state commits (run after the layer kernels of a step; only rows with exec_mask change)
// ---------------------------------------------------------------------------------------------
// previous <- last P samples of cat(previous, act(x)) (conv.py:263-267), then the session's replicate flag is cleared.
// One CTA per session; the flag is cleared after every thread of the CTA has read it.
static __global__ void conv_commit_kernel(const ConvSplitK p, const uint8_t* exec_mask) {
  const int b = blockIdx.x;
  if (!exec_mask[b]) return;
  for (int ci = threadIdx.x; ci < p.Cin; ci += blockDim.x) {
    float* s = p.st + ((long long)b * p.Cin + ci) * p.P;
    for (int j = 0; j < p.P; ++j) s[j] = p.ext(b, ci, p.Tin + j);   // reads run ahead of writes
  }
  __syncthreads();
  if (threadIdx.x == 0 && p.first != nullptr) p.first[b] = 0;
}

// partial <- scratch (conv.py:357-360), per_row = Cout * S
static __global__ void convtr_commit_kernel(float* partial, const float* scratch, int per_row, const uint8_t* exec_mask, int B) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * per_row) return;
  if (exec_mask[i / per_row]) partial[i] = scratch[i];
}

// reset: zero the state of the rows in reset_mask (conv.py:166-169, 281-286)
static __global__ void zero_rows_kernel(float* buf, long long per_row, const uint8_t* mask, int B) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * per_row) return;
  if (mask == nullptr || mask[i / per_row]) buf[i] = 0.f;
}
static __global__ void reset_flags_kernel(uint8_t* first, long long* off_a, long long* off_b, uint8_t* exec_mask,
                                          const uint8_t* mask, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  if (mask != nullptr && !mask[b]) return;
  exec_mask[b] = 1;                                       // State.reset (streaming.py:41-42)
  first[b] = 1;
  if (off_a) off_a[b] = 0;                                // _MHAState.reset / RingKVCache.reset
  if (off_b) off_b[b] = 0;
}

// ---------------------------------------------------------------------------------------------
// depth-wise ConvTranspose1d up-sampling (resample.py:68-119 with channel_wise=True, k=2S, no bias)
// latent [B][C] (one frame) -> tokens [B][S][C] (token-major for the decoder transformer)
// ---------------------------------------------------------------------------------------------
static __global__ void upsample_dw_kernel(const float* __restrict__ lat, long long lb, long long lc, long long lt, int T,
                                   const float* __restrict__ w /*[C][2S]*/, const float* __restrict__ partial,
                                   float* __restrict__ scratch, float* __restrict__ y /*[B][T*S][C]*/,
                                   int B, int C, int S) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)B * (T + 1) * S * C;
  if (i >= total) return;
  const int c = i % C;
  long long r0 = i / C;
  const int r = r0 % S; r0 /= S;
  const int t = r0 % (T + 1);
  const int b = r0 / (T + 1);
  const float* xr = lat + b * lb + c * lc;
  const long long sidx = ((long long)b * C + c) * S + r;
  if (t == T) { scratch[sidx] = w[c * 2 * S + r + S] * xr[(long long)(T - 1) * lt]; return; }
  float v = w[c * 2 * S + r] * xr[(long long)t * lt];
  if (t == 0) v += partial[sidx];
  else v += w[c * 2 * S + r + S] * xr[(long long)(t - 1) * lt];
  y[((long long)b * T * S + (long long)t * S + r) * C + c] = v;
}

// per-session token counters of a bottleneck transformer (== RingKVCache.end_offset == _MHAState.offset), advanced where exec_mask
static __global__ void advance_offsets_kernel(long long* off, const uint8_t* exec_mask, int B, int T) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B && exec_mask[b]) off[b] += T;
}

// ---------------------------------------------------------------------------------------------
// Residual VQ, level-parallel form: the nearest-code search of one level is spread over
// (code chunks x query tiles x quantizers) CTAs; the sequential dependency between levels is the
// launch order.  Per level:  rvq_search_kernel -> partial (best score, index) per code chunk;
// rvq_pick_kernel -> argmin over chunks (first minimum on ties), code written, residual updated.
// ---------------------------------------------------------------------------------------------
constexpr int RVQ_CHUNK = 128;    // codes per CTA (= threads)
constexpr int RVQ_QT = 8;         // queries per CTA

struct RvqLevelArgs {
  float* res[2];             // residuals [Q][Dq] per quantizer
  const float* cbT[2];       // this level's transposed codebook [Dq][bins]
  const float* cb[2];        // this level's codebook [bins][Dq]
  const float* cnorm[2];     // [bins]
  float* part_best[2];       // [Q][n_chunks]
  int* part_idx[2];
  int active[2];             // quantizer has this level
  int code_index[2];         // output codebook index of this level
  long long* codes; long long cs_b, cs_k, cs_f;
  int n_query, n_frames, Dq, bins, n_chunks;
};

// res[which][q][m] = sum_k Wt[k][m] * lat[q][k]   (vq.py:135: 1x1 conv, no bias)
// A CTA projects RVQ_PQ queries onto 64 outputs: 256 threads = 64 outputs x 4 slices of the input channels, 8 independent FMA
// chains per weight load (one per query), the slices added in slice order.  (One CTA per query with a 512-long dependent chain
// per thread took 85-100 us and re-read the 512 KB weight matrix for every query.)
constexpr int RVQ_PQ = 8;
static __global__ void __launch_bounds__(256) rvq_project_kernel(const float* __restrict__ lat, long long lb, long long lc,
                                                          long long lt, int n_frames, int n_query, const float* __restrict__ wT0,
                                                          const float* __restrict__ wT1, float* __restrict__ res0,
                                                          float* __restrict__ res1, int Cin, int Dq) {
  extern __shared__ float s_lat[];           // [RVQ_PQ][Cin], then [4][RVQ_PQ][64] partial sums
  float* s_part = s_lat + RVQ_PQ * Cin;
  const int q0 = blockIdx.x * RVQ_PQ, which = blockIdx.y, m0 = blockIdx.z * 64;
  for (int i = threadIdx.x; i < RVQ_PQ * Cin; i += blockDim.x) {
    const int j = i / Cin, c = i - j * Cin, q = q0 + j;
    float v = 0.f;
    if (q < n_query) { const int b = q / n_frames, f = q % n_frames; v = lat[b * lb + c * lc + f * lt]; }
    s_lat[i] = v;
  }
  __syncthreads();
  const float* wT = which ? wT1 : wT0;
  float* res = which ? res1 : res0;
  const int m = threadIdx.x & 63, sl = threadIdx.x >> 6;
  const int kper = (Cin + 3) / 4, k0 = sl * kper, k1 = min(Cin, k0 + kper);
  float acc[RVQ_PQ];
#pragma unroll
  for (int j = 0; j < RVQ_PQ; ++j) acc[j] = 0.f;
  if (m0 + m < Dq) {
#pragma unroll 4
    for (int k = k0; k < k1; ++k) {
      const float w = wT[(long long)k * Dq + m0 + m];
#pragma unroll
      for (int j = 0; j < RVQ_PQ; ++j) acc[j] = fmaf(w, s_lat[j * Cin + k], acc[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < RVQ_PQ; ++j) s_part[(sl * RVQ_PQ + j) * 64 + m] = acc[j];
  __syncthreads();
  for (int i = threadIdx.x; i < RVQ_PQ * 64; i += blockDim.x) {
    const int j = i >> 6, mm = i & 63, q = q0 + j;
    if (q < n_query && m0 + mm < Dq)
      res[(long long)q * Dq + m0 + mm] = ((s_part[(0 * RVQ_PQ + j) * 64 + mm] + s_part[(1 * RVQ_PQ + j) * 64 + mm]) +
                                          s_part[(2 * RVQ_PQ + j) * 64 + mm]) + s_part[(3 * RVQ_PQ + j) * 64 + mm];
  }
}

static __global__ void __launch_bounds__(RVQ_CHUNK) rvq_search_kernel(const RvqLevelArgs a) {
  const int which = blockIdx.z;
  if (!a.active[which]) return;
  extern __shared__ float s_res[];            // [Dq][RVQ_QT]  (queries fastest: two broadcast LDS.128 per dim)
  __shared__ float s_best[RVQ_QT][RVQ_CHUNK / 32];
  __shared__ int s_bidx[RVQ_QT][RVQ_CHUNK / 32];
  const int tid = threadIdx.x;
  const int q0 = blockIdx.y * RVQ_QT;
  const int code = blockIdx.x * RVQ_CHUNK + tid;
  const float* res = a.res[which];
  for (int i = tid; i < RVQ_QT * a.Dq; i += RVQ_CHUNK) {
    const int q = i / a.Dq, d = i - q * a.Dq;
    s_res[d * RVQ_QT + q] = (q0 + q < a.n_query) ? res[(long long)(q0 + q) * a.Dq + d] : 0.f;
  }
  __syncthreads();
  float dots[RVQ_QT];
#pragma unroll
  for (int q = 0; q < RVQ_QT; ++q) dots[q] = 0.f;
  const bool ok = code < a.bins;
  const float* col = a.cbT[which] + (ok ? code : 0);
  // 32 codebook loads in flight per thread (8 made every batch of FMAs wait a full L2 round trip: 32 round trips per level)
  for (int d0 = 0; d0 < a.Dq; d0 += 32) {
    float cv[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) cv[j] = d0 + j < a.Dq ? col[(long long)(d0 + j) * a.bins] : 0.f;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      if (d0 + j >= a.Dq) break;
      const float4 r0 = *reinterpret_cast<const float4*>(&s_res[(d0 + j) * RVQ_QT]);
      const float4 r1 = *reinterpret_cast<const float4*>(&s_res[(d0 + j) * RVQ_QT + 4]);
      dots[0] = fmaf(cv[j], r0.x, dots[0]); dots[1] = fmaf(cv[j], r0.y, dots[1]);
      dots[2] = fmaf(cv[j], r0.z, dots[2]); dots[3] = fmaf(cv[j], r0.w, dots[3]);
      dots[4] = fmaf(cv[j], r1.x, dots[4]); dots[5] = fmaf(cv[j], r1.y, dots[5]);
      dots[6] = fmaf(cv[j], r1.z, dots[6]); dots[7] = fmaf(cv[j], r1.w, dots[7]);
    }
  }
  const float cn = ok ? a.cnorm[which][code] : 0.f;
#pragma unroll
  for (int q = 0; q < RVQ_QT; ++q) {
    float best = ok ? cn - 2.f * dots[q] : INFINITY;       // |c|^2 - 2 x.c  (core_vq.py:270-276 without the constant |x|^2)
    int bidx = ok ? code : 0x7fffffff;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bidx, o);
      if (ob < best || (ob == best && oi < bidx)) { best = ob; bidx = oi; }
    }
    if ((tid & 31) == 0) { s_best[q][tid >> 5] = best; s_bidx[q][tid >> 5] = bidx; }
  }
  __syncthreads();
  if (tid < RVQ_QT && q0 + tid < a.n_query) {
    float best = s_best[tid][0];
    int bidx = s_bidx[tid][0];
#pragma unroll
    for (int w = 1; w < RVQ_CHUNK / 32; ++w) {
      const float ob = s_best[tid][w];
      const int oi = s_bidx[tid][w];
      if (ob < best || (ob == best && oi < bidx)) { best = ob; bidx = oi; }
    }
    a.part_best[which][(long long)(q0 + tid) * a.n_chunks + blockIdx.x] = best;
    a.part_idx[which][(long long)(q0 + tid) * a.n_chunks + blockIdx.x] = bidx;
  }
}

// one CTA per (query, quantizer): argmin over the chunk partials, emit the code, res -= c[idx] (core_vq.py:514-516)
static __global__ void __launch_bounds__(128) rvq_pick_kernel(const RvqLevelArgs a) {
  const int which = blockIdx.y;
  if (!a.active[which]) return;
  const int q = blockIdx.x;
  __shared__ int s_choice;
  if (threadIdx.x < 32) {
    float best = INFINITY;
    int bidx = 0x7fffffff;
    for (int c = threadIdx.x; c < a.n_chunks; c += 32) {
      const float ob = a.part_best[which][(long long)q * a.n_chunks + c];
      const int oi = a.part_idx[which][(long long)q * a.n_chunks + c];
      if (ob < best || (ob == best && oi < bidx)) { best = ob; bidx = oi; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bidx, o);
      if (ob < best || (ob == best && oi < bidx)) { best = ob; bidx = oi; }
    }
    if (threadIdx.x == 0) {
      s_choice = bidx;
      const int b = q / a.n_frames, f = q % a.n_frames;
      a.codes[b * a.cs_b + a.code_index[which] * a.cs_k + f * a.cs_f] = bidx;
    }
  }
  __syncthreads();
  const float* c = a.cb[which] + (long long)s_choice * a.Dq;
  float* r = a.res[which] + (long long)q * a.Dq;
  for (int d = threadIdx.x; d < a.Dq; d += blockDim.x) r[d] -= c[d];
}

// codes [B][K][n] -> latent (vq.py:281-287): out = Wo_first . c0[idx0] + Wo_rest . sum_l c_l[idx_l]
struct RvqDecArgs {
  const long long* codes; long long cs_b, cs_k, cs_f; int n_frames;
  const float* cb[2]; const float* woT[2];   // woT [Dq][Cout]
  int levels[2]; int level_offset[2];
  float* out; long long ob, oc, ot;          // [B][Cout][n] via strides
  int Dq, Cout, bins;
  int* err;                                  // device error flags: a code outside [0, bins) decodes as the zero vector and
                                             // raises bit 2 (the reference indexes F.embedding: "dramatic CUDA crash", vq.py:144-145)
};
// grid (B * n_frames, ceil(Cout / 64)), 256 threads = 64 output channels x 4 slices of the Dq-long dot products: the
// dependent FMA chain per thread is Dq / 2 long instead of 2 * Dq, and a single session still spreads over 8 CTAs.
static __global__ void __launch_bounds__(256) rvq_decode_kernel(const RvqDecArgs a) {
  extern __shared__ float sm[];              // [2][Dq] summed code vectors, then [4][64] partial dot products
  const int b = blockIdx.x / a.n_frames, f = blockIdx.x % a.n_frames;
  const int tid = threadIdx.x;
  float* part = sm + 2 * a.Dq;
  for (int which = 0; which < 2; ++which) {
    for (int d = tid; d < a.Dq; d += blockDim.x) {
      float s = 0.f;
      for (int level = 0; level < a.levels[which]; ++level) {
        const long long idx = a.codes[b * a.cs_b + (a.level_offset[which] + level) * a.cs_k + f * a.cs_f];
        if (idx >= 0 && idx < a.bins) s += a.cb[which][((long long)level * a.bins + idx) * a.Dq + d];
        else if (a.err != nullptr && d == 0) atomicOr(a.err, 2);
      }
      sm[which * a.Dq + d] = s;
    }
  }
  __syncthreads();
  const int cl = tid & 63, slice = tid >> 6;
  const int c = blockIdx.y * 64 + cl;
  const int d0 = slice * (a.Dq / 4), d1 = slice == 3 ? a.Dq : d0 + a.Dq / 4;
  float acc0 = 0.f, acc1 = 0.f;
  if (c < a.Cout) {
    if (a.levels[0] > 0) {
#pragma unroll 8
      for (int d = d0; d < d1; ++d) acc0 = fmaf(a.woT[0][(long long)d * a.Cout + c], sm[d], acc0);
    }
    if (a.levels[1] > 0) {
#pragma unroll 8
      for (int d = d0; d < d1; ++d) acc1 = fmaf(a.woT[1][(long long)d * a.Cout + c], sm[a.Dq + d], acc1);
    }
  }
  part[slice * 64 + cl] = acc0 + acc1;
  __syncthreads();
  if (slice == 0 && c < a.Cout)               // slices in order: the sum does not depend on scheduling
    a.out[b * a.ob + c * a.oc + f * a.ot] = ((part[cl] + part[64 + cl]) + part[128 + cl]) + part[192 + cl];
}

// ---------------------------------------------------------------------------------------------
// load-time repacking
// ---------------------------------------------------------------------------------------------
static __global__ void transpose_kernel(const float* in /*[R][C]*/, float* out /*[C][R]*/, int R, int C) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)R * C) return;
  const int c = i % C; const int r = i / C;
  out[(long long)c * R + r] = in[i];
}
// centroids = embedding_sum / clamp(cluster_usage, 1e-5)  (core_vq.py:181-183) + transposed copy + norms
static __global__ void build_codebook_kernel(const float* esum, const float* usage, float* cb, float* cbT, float* cnorm,
                                      int bins, int Dq) {
  const int code = blockIdx.x;
  const float u = fmaxf(usage[code], 1e-5f);
  float s = 0.f;
  for (int d = threadIdx.x; d < Dq; d += blockDim.x) {
    const float v = esum[(long long)code * Dq + d] / u;
    cb[(long long)code * Dq + d] = v;
    cbT[(long long)d * bins + code] = v;
    s += v * v;
  }
  __shared__ float red[32];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < (blockDim.x + 31) / 32; ++w) t += red[w];
    cnorm[code] = t;
  }
}

}  // namespace mimi
}  // namespace b200
