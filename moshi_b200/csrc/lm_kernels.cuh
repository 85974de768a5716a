// bf16 kernels of the Moshi LM decode step (one 12.5 Hz frame for B concurrent sessions).
//
// Cast points follow the reference exactly (SURVEY.md appendix B): every nn.Linear output is a bf16
// tensor, RMSNorm / RoPE / softmax / SiLU are evaluated in fp32 on bf16 inputs and rounded once,
// residual adds and the 17-way embedding sum are bf16 adds.
#pragma once

#include <cmath>

#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include "common.cuh"

namespace b200 {
namespace lm {

typedef __nv_bfloat16 bf16;

// The GEMM that follows each of these kernels is launched with programmatic stream serialization
// (gemm_sk.cu): triggering at entry lets its CTAs take free SM resources and start streaming weights
// while this kernel runs; the GEMM itself waits (griddepcontrol.wait) before it touches activations.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ void unpack8(const uint4& v, float* f) {
  const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(p[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}

// ---------------------------------------------------------------------------------------------
// token ring (LMGen._step bookkeeping, lm.py:691-702 and :759-783)
// ---------------------------------------------------------------------------------------------
struct TokenRing {
  long long* cache;        // [B][Kc][CT]
  long long* offsets;      // [B]
  const uint8_t* exec_mask;
  const int* delays;       // [Kc]
  int Kc, CT, dep_q, n_q, card, text_card, max_delay;
  // classifier-free guidance (lm.py:596-604, 714-726): the model runs on 2B rows, rows [B, 2B) are the "null" copies
  int cfg;                          // 0 = off, 1 = on
  int cfg_is_no_text;               // null rows: text stream zeroed
  const long long* cfg_masked_until;   // [B] or null: null rows: every stream zeroed while offset <= delay + masked_until[b]
  int* err;                         // device error flags (ERR_*), may be null
};

// device error flags: raised instead of reading out of bounds; surfaced by b200_lm_error_flags / b200_mimi_error_flags and by
// the host-synchronising entry points
enum { ERR_TOKEN_RANGE = 1, ERR_CODE_RANGE = 2, ERR_KV_CAPACITY = 4, ERR_KV_POOL = 8 };

// One thread per (b, k): write the user's codes, then build the model input row(s) [MB][Kc].
static __global__ void lm_prepare_kernel(const TokenRing r, const long long* __restrict__ in_codes, int n_in,
                                  long long* __restrict__ input_tokens, int B) {
  pdl_trigger();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * r.Kc) return;
  const int b = i / r.Kc, k = i % r.Kc;
  const long long off = r.offsets[b];
  const bool exec = r.exec_mask[b] != 0;
  long long* row = r.cache + ((long long)b * r.Kc + k) * r.CT;
  if (k > r.dep_q && exec) {                                    // lm.py:691-696
    const int pos = (int)((off + r.delays[k]) % r.CT);
    row[pos] = in_codes[(long long)b * n_in + (k - r.dep_q - 1)];
  }
  const bool is_init = off <= r.delays[k] || !exec;             // lm.py:698-699
  const long long initial = k == 0 ? r.text_card : r.card;      // lm.py:297-311
  const long long tok = is_init ? initial : row[off % r.CT];
  input_tokens[i] = tok;
  if (r.cfg) {                                                  // lm.py:714-726
    long long t2 = tok;
    if (r.cfg_masked_until != nullptr && off <= r.delays[k] + r.cfg_masked_until[b] && !is_init) t2 = -1;
    if (r.cfg_is_no_text && k == 0 && !is_init) t2 = -1;
    input_tokens[(long long)B * r.Kc + i] = t2;
  }
}

// offsets += exec; store sampled tokens; gather the delay-aligned output (lm.py:759-783)
static __global__ void lm_finish_kernel(const TokenRing r, const long long* __restrict__ text_token,
                                 const long long* __restrict__ audio_tokens /*[dep_q][B]*/,
                                 long long* __restrict__ out /*[B][dep_q+1]*/, int B, unsigned long long* noise_ctr) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b == 0 && noise_ctr != nullptr) *noise_ctr += 1;        // the next step draws fresh Exp(1) noise (lm_noise_kernel)
  if (b >= B) return;
  const bool exec = r.exec_mask[b] != 0;
  long long off = r.offsets[b];
  if (exec) off += 1;
  r.offsets[b] = off;
  const int pos = (int)(off % r.CT);
  if (exec) {
    r.cache[((long long)b * r.Kc + 0) * r.CT + pos] = text_token[b];
    for (int k = 0; k < r.dep_q; ++k)
      r.cache[((long long)b * r.Kc + 1 + k) * r.CT + pos] = audio_tokens[(long long)k * B + b];
  }
  const bool not_ready = off <= r.max_delay || !exec;
  for (int k = 0; k <= r.dep_q; ++k) {
    long long idx = (off - r.max_delay + r.delays[k]) % r.CT;
    if (idx < 0) idx += r.CT;                                    // python modulo
    const long long v = r.cache[((long long)b * r.Kc + k) * r.CT + idx];
    out[(long long)b * (r.dep_q + 1) + k] = not_ready ? -2 : v;
  }
}

// ---------------------------------------------------------------------------------------------
// embeddings (lm.py:390-397; ScaledEmbedding: token -1 -> zero row, lm_utils.py:103-121)
// ---------------------------------------------------------------------------------------------
struct EmbedTables {
  const bf16* audio[32];   // [card+1][dim]
  const bf16* text;        // [text_card+1][dim]
  int n_q, card, text_card;
  const bf16* condition_sum;   // [rows][dim] or null: fuser.get_sum(condition_tensors), added last (lm.py:398-399)
  int* err;
};
// valid ids: [0, vocab] (vocab = the initial token) and -1 (zero row); anything else (-2 "ungenerated", ids past the table)
// would be a device assert in the reference (F.embedding); here it raises ERR_TOKEN_RANGE and embeds as the zero row
__device__ __forceinline__ bool embed_id_ok(long long id, int vocab, int* err) {
  if (id >= 0 && id <= vocab) return true;
  if (id != -1 && err != nullptr) atomicOr(err, ERR_TOKEN_RANGE);
  return false;
}
static __global__ void lm_embed_sum_kernel(const EmbedTables t, const long long* __restrict__ tokens /*[B][n_q+1]*/,
                                    bf16* __restrict__ x /*[B][dim]*/, int B, int dim) {
  pdl_trigger();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;   // (b, pair)
  const int half = dim / 2;
  if (i >= B * half) return;
  const int b = i / half, c = (i % half) * 2;
  const long long* tok = tokens + (long long)b * (t.n_q + 1);
  float s0 = 0.f, s1 = 0.f;
  for (int k = 0; k < t.n_q; ++k) {
    const long long id = tok[k + 1];
    float e0 = 0.f, e1 = 0.f;
    if (embed_id_ok(id, t.card, t.err)) {
      const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(t.audio[k] + id * dim + c);
      e0 = __low2float(v); e1 = __high2float(v);
    }
    if (k == 0) { s0 = e0; s1 = e1; }
    else { s0 = rbf(s0 + e0); s1 = rbf(s1 + e1); }       // bf16 add per table
  }
  {
    const long long id = tok[0];
    float e0 = 0.f, e1 = 0.f;
    if (embed_id_ok(id, t.text_card, t.err)) {
      const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(t.text + id * dim + c);
      e0 = __low2float(v); e1 = __high2float(v);
    }
    if (t.n_q == 0) { s0 = e0; s1 = e1; }
    else { s0 = rbf(s0 + e0); s1 = rbf(s1 + e1); }
  }
  if (t.condition_sum != nullptr) {
    const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(t.condition_sum + (long long)b * dim + c);
    s0 = rbf(s0 + __low2float(v)); s1 = rbf(s1 + __high2float(v));
  }
  *reinterpret_cast<__nv_bfloat162*>(x + (long long)b * dim + c) = __floats2bfloat162_rn(s0, s1);
}

// depformer input: x = depformer_in[k](transformer_out) + emb(prev)   (lm.py:475-486); with CFG the rows [Bt, 2*Bt) reuse the
// tokens of rows [0, Bt) (lm.py:824-826)
static __global__ void dep_input_kernel(const bf16* __restrict__ din /*[B][ld]*/, long long ld, int col0,
                                 const bf16* __restrict__ table /*[V][dd]*/, const long long* __restrict__ prev /*[Bt]*/,
                                 bf16* __restrict__ x /*[B][dd]*/, int B, int dd, int Bt, int vocab, int* err) {
  pdl_trigger();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * dd) return;
  const int b = i / dd, c = i % dd;
  const long long id = prev[b % Bt];
  const float e = embed_id_ok(id, vocab, err) ? bf2f(table[id * dd + c]) : 0.f;
  x[i] = f2bf(bf2f(din[(long long)b * ld + col0 + c]) + e);
}

// Load time, low-rank depformer embeddings (lm_utils.py:80-124): the full-rank table out[V][dd], row t = low[dd][r] . e_t for the
// factor rows e[V][r].  One CTA per row.  bf16 weights: fp32 sums in k order.  quantize (QLinear, utils/quantize.py:13-40, restated
// by oracle/quant.py): the row and each low-rank row are row-wise absmax int8 (the weight through fp16), summed in int32 and
// dequantised as acc * (sa * sw / 127^2).  Dynamic shared memory: r floats.
__device__ __forceinline__ int quant_i8_rn(float v, float inv) {       // round(v * 127 / absmax), ties to even, as the linears'
  const int q = __float2int_rn(v * inv);
  return q > 127 ? 127 : (q < -127 ? -127 : q);
}
static __global__ void lowrank_expand_kernel(const bf16* __restrict__ e, const bf16* __restrict__ low, bf16* __restrict__ out, int r,
                                             int dd, int quantize) {
  extern __shared__ float row[];
  __shared__ float red[32];
  const long long t = blockIdx.x;
  float mx = 0.f;
  for (int i = threadIdx.x; i < r; i += blockDim.x) {
    row[i] = bf2f(e[t * r + i]);
    mx = fmaxf(mx, fabsf(row[i]));
  }
  if (quantize) {
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    float sa = 0.f;
    for (int i = 0; i < (int)(blockDim.x + 31) / 32; ++i) sa = fmaxf(sa, red[i]);
    const float inv = sa > 0.f ? 127.f / sa : 0.f;
    for (int i = threadIdx.x; i < r; i += blockDim.x) row[i] = (float)quant_i8_rn(row[i], inv);
    __syncthreads();
    for (int j = threadIdx.x; j < dd; j += blockDim.x) {
      const bf16* w = low + (long long)j * r;
      float sw = 0.f;
      for (int i = 0; i < r; ++i) sw = fmaxf(sw, fabsf(__half2float(__float2half_rn(bf2f(w[i])))));
      const float winv = sw > 0.f ? 127.f / sw : 0.f;
      int acc = 0;
      for (int i = 0; i < r; ++i) acc += (int)row[i] * quant_i8_rn(__half2float(__float2half_rn(bf2f(w[i]))), winv);
      out[t * dd + j] = f2bf((float)acc * (sa * sw * (1.f / 16129.f)));
    }
    return;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < dd; j += blockDim.x) {
    const bf16* w = low + (long long)j * r;
    float acc = 0.f;
    for (int i = 0; i < r; ++i) acc = fmaf(row[i], bf2f(w[i]), acc);
    out[t * dd + j] = f2bf(acc);
  }
}

// classifier-free guidance on logits (lm.py:728-732, 828-833): out = null + (cond - null) * coef, every operation a bf16
// tensor op like the reference's; rows [0, B) = conditioned, [B, 2B) = null
static __global__ void cfg_combine_kernel(const bf16* __restrict__ logits /*[2B][card]*/, bf16* __restrict__ out /*[B][card]*/,
                                   int B, int card, float coef) {
  pdl_trigger();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * card) return;
  const float l = bf2f(logits[i]), n = bf2f(logits[(long long)B * card + i]);
  out[i] = f2bf(n + rbf(rbf(l - n) * coef));
}

// extra heads of the STT models (lm.py:224-226, 803-806): softmax(extra_head(transformer_out)) in the model dtype.
// One warp per (head, row); E <= 32 outputs per head.
static __global__ void extra_heads_kernel(const bf16* __restrict__ tout /*[B][dim]*/, const bf16* const* __restrict__ w /*[n][E][dim]*/,
                                   bf16* __restrict__ out /*[n][B][E]*/, int B, int dim, int E, int n_heads) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n_heads * B) return;
  const int hd = warp / B, b = warp - hd * B;
  const bf16* wh = w[hd];
  float mine = -INFINITY;                      // lane e keeps logit e
  for (int e = 0; e < E; ++e) {
    float acc = 0.f;
    for (int k = lane; k < dim; k += 32) acc = fmaf(bf2f(tout[(long long)b * dim + k]), bf2f(wh[(long long)e * dim + k]), acc);
    acc = rbf(warp_sum(acc));                  // nn.Linear output is a bf16 tensor
    if (lane == e) mine = acc;
  }
  const float mx = warp_max(mine);
  const float ex = lane < E ? expf(mine - mx) : 0.f;
  const float sum = warp_sum(ex);
  if (lane < E) out[((long long)hd * B + b) * E + lane] = f2bf(ex / sum);
}

// Exp(1) noise for one step's samplers (sampling.py:44: torch.empty_like(probs).exponential_(1)), drawn inside the step's graph:
// Philox4x32-10 keyed by the session seed, counter = (element / 4, step counter); element i is word i % 4 of block i / 4.
__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1, uint32_t* out) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}
// One Exp(1) draw from 32 random bits, as torch's exponential_ makes it on CUDA: u = (m + 1) 2^-24 in (0, 1] from the top
// 24 bits m, then -log(u) with the accurate logf (__logf's absolute error near 1 is about 2^-22, more than -log(u) itself).
// u >= 1 - 2^-24 (the top two patterns) gives 2^-24, torch's epsilon / 2: every draw is strictly positive, so no candidate's
// score p / q becomes -inf.
__device__ __forceinline__ float exp1_from_bits(uint32_t r) {
  const float u = ((float)(r >> 8) + 1.0f) * (1.0f / 16777216.0f);
  return u >= 1.0f - 0x1p-24f ? 0x1p-24f : -logf(u);
}
// exp1_from_bits on given words (test entry point b200_op_exp1)
static __global__ void exp1_kernel(const uint32_t* __restrict__ words, float* __restrict__ out, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = exp1_from_bits(words[i]);
}
static __global__ void lm_noise_kernel(float* __restrict__ noise, long long n, unsigned long long seed,
                                const unsigned long long* __restrict__ step_ctr) {
  pdl_trigger();
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;      // one Philox block = 4 values
  if (q * 4 >= n) return;
  const unsigned long long ctr = *step_ctr;
  uint32_t r[4];
  philox4x32_10((uint32_t)q, (uint32_t)(q >> 32), (uint32_t)ctr, (uint32_t)(ctr >> 32), (uint32_t)seed, (uint32_t)(seed >> 32), r);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const long long i = q * 4 + j;
    if (i < n) noise[i] = exp1_from_bits(r[j]);
  }
}

// ---------------------------------------------------------------------------------------------
// RMSNorm with fp32 math, eps 1e-8 (transformer.py:45-58): y = bf16(x * (alpha * rsqrt(eps + mean(x^2))))
// Optionally fuses the preceding residual add: x <- bf16(x + upd) first (transformer.py:769,777).
// ---------------------------------------------------------------------------------------------
static __global__ void __launch_bounds__(256) rmsnorm_kernel(const bf16* __restrict__ x, const bf16* __restrict__ alpha,
                                                      bf16* __restrict__ y, int dim, float eps) {
  pdl_trigger();
  const int row = blockIdx.x;
  const bf16* xr = x + (long long)row * dim;
  float ss = 0.f;
  for (int c = threadIdx.x * 2; c < dim; c += blockDim.x * 2) {
    const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(xr + c));
    ss += v.x * v.x + v.y * v.y;
  }
  __shared__ float red[32];
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    t = warp_sum(t);
    if (threadIdx.x == 0) red[0] = t;
  }
  __syncthreads();
  const float r = rsqrtf(eps + red[0] / (float)dim);
  for (int c = threadIdx.x * 2; c < dim; c += blockDim.x * 2) {
    const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(xr + c));
    const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(alpha + c));
    *reinterpret_cast<__nv_bfloat162*>(y + (long long)row * dim + c) =
        __floats2bfloat162_rn(v.x * (a.x * r), v.y * (a.y * r));
  }
}

// epilogues of the LM linears (gemm_sk.cu): plain store, residual add, gated SiLU (gating.py:18-20)
enum { LIN_STORE = 0, LIN_RESADD = 1, LIN_GATE = 2 };

constexpr int ATT_D = 128;
constexpr int ATT_THREADS = 128;
constexpr int ATT_GROUP = 4;                   // keys per half-warp per register buffer of the attention step

// split-KV so that B*H*nsplit CTAs cover the 132 SMs a few times over even at B = 1
inline int attn_pick_splits(int B, int H, int cap) {
  int ns = (148 * 4 + B * H - 1) / (B * H);
  if (ns < 1) ns = 1;
  if (ns > 16) ns = 16;
  const int max_by_len = (cap + 63) / 64;
  if (ns > max_by_len) ns = max_by_len;
  return ns;
}

// ---------------------------------------------------------------------------------------------
// Fused temporal attention step (T = 1, D = 128): RoPE(q, k) + ring append + split-KV attention +
// split combine in ONE launch (transformer.py:557-597).
//   grid = (B*H, nsplit), 128 threads.  qkv [B][3C] bf16 (rows q | k | v, each (h d)).
//   * the CTA whose key range holds the slot of the new key rotates k, writes K/V there, syncs, and then
//     reads it back like any other key; no other CTA touches that slot (ranges are disjoint), so the
//     append needs no separate kernel and the oldest key it replaces is never attended;
//   * q is rotated in registers (rounded to bf16 like the reference's apply_rope output);
//   * with nsplit > 1 the last CTA to arrive for a (b, h) merges the partials in split order.
// PAGED: kc / vc are page pools [n_pages + 1][H][page_slots][ATT_D] (b200_lm_set_kv_pool) and slot s of row b lives at
// page table[b * tab_ld + (s >> page_shift)], offset s & (page_slots - 1).  Only the key address changes: the split
// boundaries, the per-key arithmetic and the merge order are those of the contiguous ring, so the output is bit-identical.
// The table must map every slot the step reads or writes (kv_page_alloc_kernel does, with the sink page when the pool is dry).
// ---------------------------------------------------------------------------------------------
struct AttnStep {
  const bf16* qkv; bf16* kc; bf16* vc; bf16* out;
  float* part; int* counters;                  // [B*H][nsplit][ATT_D + 2], [B*H] (zero between launches)
  const long long* pos; const uint8_t* exec_mask;
  int H, cap, nsplit; float neg_log_period_2_over_d;
  const int* table; int tab_ld, page_shift;    // PAGED only: page table [B][tab_ld], log2(page_slots)
};

// Row of slot s of head h on page pg of a paged pool [n_pages + 1][H][1 << page_shift][row]
__device__ __forceinline__ long long kv_paged_row(int pg, int H, int h, int s, int page_shift) {
  return (((long long)pg * H + h) << page_shift) + (s & ((1 << page_shift) - 1));
}

// Split `split` of row b attends to ring slots [s0, s1) of the n_valid = min(pos + exec, cap) valid ones; the new key goes to
// slot_new = pos % cap, and owns_new (CTA-uniform) says whether this split appends it.
struct AttnRange {
  long long p;
  int s0, s1, slot_new;
  bool owns_new;
};
template <class Args>
__device__ __forceinline__ AttnRange attn_range(const Args& a, int b, int split) {
  AttnRange r;
  const bool exec = a.exec_mask[b] != 0;
  r.p = a.pos[b];
  long long n_valid = r.p + (exec ? 1 : 0);
  if (n_valid > a.cap) n_valid = a.cap;
  const int per = (int)((n_valid + a.nsplit - 1) / a.nsplit);
  r.s0 = split * per;
  r.s1 = (int)min((long long)(r.s0 + per), n_valid);
  r.slot_new = (int)(r.p % a.cap);
  r.owns_new = exec && r.slot_new >= r.s0 && r.slot_new < r.s1;
  return r;
}

// RoPE of the pair (re, im) at position pos (rope.py:45-82)
__device__ __forceinline__ void rope_pair(float re, float im, int pair, float pos, float neg_log_period_2_over_d, float* o0, float* o1) {
  const float freq = expf((float)pair * neg_log_period_2_over_d);
  float sn, cs;
  sincosf(freq * pos, &sn, &cs);
  *o0 = re * cs - im * sn;
  *o1 = re * sn + im * cs;
}

// Elements [8 * l16, 8 * l16 + 8) of the query q[ATT_D] at position pos, rotated, rounded to bf16 like apply_rope's output and
// times 1/sqrt(128), as store(j, element 2j, element 2j + 1) for j < 4
template <class Store>
__device__ __forceinline__ void attn_query(const bf16* q, int l16, float pos, float neg_log_period_2_over_d, Store store) {
  float raw[8];
  unpack8(*reinterpret_cast<const uint4*>(q + l16 * 8), raw);
  const float scale = 0.08838834764831845f;       // 1/sqrt(128)
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float o0, o1;
    rope_pair(raw[2 * j], raw[2 * j + 1], l16 * 4 + j, pos, neg_log_period_2_over_d, &o0, &o1);
    store(j, rbf(o0) * scale, rbf(o1) * scale);
  }
}

// Keys [s0, s1) in groups of ATT_GROUP keys per half-warp, double-buffered in registers: the loads of group i + 1 are in flight
// while group i is reduced.  load_group(first key of the CTA's group, Group&), reduce_group(same, const Group&).
template <class Group, class Load, class Reduce>
__device__ __forceinline__ void attn_key_loop(int s0, int s1, Load load_group, Reduce reduce_group) {
  constexpr int U = ATT_GROUP;
  Group ga, gb;
  if (s0 < s1) load_group(s0, ga);
  for (int kb0 = s0; kb0 < s1; kb0 += 16 * U) {     // CTA-uniform trip count and branches (shuffles inside reduce_group)
    const int k1 = kb0 + 8 * U, k2 = kb0 + 16 * U;
    if (k1 < s1) load_group(k1, gb);
    reduce_group(kb0, ga);
    if (k1 < s1) {
      if (k2 < s1) load_group(k2, ga);
      reduce_group(k1, gb);
    }
  }
}

// Merges the online-softmax states (m, l, acc[8] over this lane's 8 outputs) of the CTA's 8 half-warps and stores out[bh]; with
// nsplit > 1 each CTA stores its partial and the last to arrive for bh merges the splits in split order.
template <class Args>
__device__ __forceinline__ void attn_merge_store(const Args& a, int bh, int split, float m, float l, const float* acc) {
  const int tid = threadIdx.x, l16 = tid & 15, hw = tid >> 4;
  __shared__ float sm_m[8], sm_l[8], sm_acc[8][ATT_D];
  __shared__ int s_last;
  if (l16 == 0) { sm_m[hw] = m; sm_l[hw] = l; }
#pragma unroll
  for (int i = 0; i < 8; ++i) sm_acc[hw][l16 * 8 + i] = acc[i];
  __syncthreads();
  float M = -INFINITY;
#pragma unroll
  for (int w = 0; w < 8; ++w) M = fmaxf(M, sm_m[w]);
  float L = 0.f, A = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) {
    const float c = sm_m[w] == -INFINITY ? 0.f : __expf(sm_m[w] - M);
    L += sm_l[w] * c;
    A += sm_acc[w][tid] * c;
  }
  if (a.nsplit == 1) {
    a.out[(long long)bh * ATT_D + tid] = f2bf(L > 0.f ? A / L : 0.f);
    return;
  }
  float* o = a.part + ((long long)bh * a.nsplit + split) * (ATT_D + 2);
  __stcg(o + tid, A);
  if (tid == 0) { __stcg(o + ATT_D, M); __stcg(o + ATT_D + 1, L); }
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const int old = atomicAdd(a.counters + bh, 1);
    s_last = old == a.nsplit - 1;
    if (s_last) a.counters[bh] = 0;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const float* pp = a.part + (long long)bh * a.nsplit * (ATT_D + 2);
  float MM = -INFINITY;
  for (int s = 0; s < a.nsplit; ++s) MM = fmaxf(MM, __ldcg(pp + s * (ATT_D + 2) + ATT_D));
  float LL = 0.f, AA = 0.f;
  for (int s = 0; s < a.nsplit; ++s) {
    const float ms = __ldcg(pp + s * (ATT_D + 2) + ATT_D);
    const float c = ms == -INFINITY ? 0.f : __expf(ms - MM);
    LL += __ldcg(pp + s * (ATT_D + 2) + ATT_D + 1) * c;
    AA += __ldcg(pp + s * (ATT_D + 2) + tid) * c;
  }
  a.out[(long long)bh * ATT_D + tid] = f2bf(LL > 0.f ? AA / LL : 0.f);
}

template <bool PAGED>
static __global__ void __launch_bounds__(ATT_THREADS) attn_step_kernel(const AttnStep a) {
  pdl_trigger();
  const int bh = blockIdx.x, split = blockIdx.y;
  const int b = bh / a.H, h = bh - b * a.H;
  const int C = a.H * ATT_D;
  const int tid = threadIdx.x, l16 = tid & 15;
  const int hw = tid >> 4;                          // half-warp id 0..7
  const AttnRange r = attn_range(a, b, split);
  const bf16* base = a.qkv + (long long)b * 3 * C + h * ATT_D;
  const float fpos = (float)r.p;
  // PAGED: element offset of slot s of this (b, h) in the pool
  auto paged_off = [&](int s) -> long long {
    return kv_paged_row(__ldg(a.table + (long long)b * a.tab_ld + (s >> a.page_shift)), a.H, h, s, a.page_shift) * ATT_D;
  };

  if (r.owns_new) {
    if (tid < ATT_D / 2) {
      const int pr = tid;
      float k0, k1;
      rope_pair(bf2f(base[C + 2 * pr]), bf2f(base[C + 2 * pr + 1]), pr, fpos, a.neg_log_period_2_over_d, &k0, &k1);
      long long o;
      if constexpr (PAGED) o = paged_off(r.slot_new) + 2 * pr;
      else o = ((long long)bh * a.cap + r.slot_new) * ATT_D + 2 * pr;
      *reinterpret_cast<__nv_bfloat162*>(a.kc + o) = __floats2bfloat162_rn(k0, k1);
      *reinterpret_cast<__nv_bfloat162*>(a.vc + o) = *reinterpret_cast<const __nv_bfloat162*>(base + 2 * C + 2 * pr);
    }
    __syncthreads();
  }

  float qf[8];
  attn_query(base, l16, fpos, a.neg_log_period_2_over_d, [&](int j, float x0, float x1) { qf[2 * j] = x0; qf[2 * j + 1] = x1; });

  const long long row0 = PAGED ? 0 : (long long)bh * a.cap * ATT_D;
  const bf16* kb = a.kc + row0 + l16 * 8;
  const bf16* vb = a.vc + row0 + l16 * 8;
  float m = -INFINITY, l = 0.f, acc[8] = {};

  constexpr int U = ATT_GROUP;
  struct Group { uint4 k[U], v[U]; };
  auto load_group = [&](int kb0, Group& gp) {
    const int s = kb0 + hw * U;
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int ss = s + u < r.s1 ? s + u : r.s1 - 1;
      long long o;
      if constexpr (PAGED) o = paged_off(ss);
      else o = (long long)ss * ATT_D;
      gp.k[u] = *reinterpret_cast<const uint4*>(kb + o);
      gp.v[u] = *reinterpret_cast<const uint4*>(vb + o);
    }
  };
  auto reduce_group = [&](int kb0, const Group& gp) {
    const int s = kb0 + hw * U;
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float kf[8];
      unpack8(gp.k[u], kf);
      float d = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) d = fmaf(qf[i], kf[i], d);
      d += __shfl_xor_sync(0xffffffffu, d, 8);
      d += __shfl_xor_sync(0xffffffffu, d, 4);
      d += __shfl_xor_sync(0xffffffffu, d, 2);
      d += __shfl_xor_sync(0xffffffffu, d, 1);
      if (s + u < r.s1) {
        const float mn = fmaxf(m, d);
        const float corr = __expf(m - mn), pw = __expf(d - mn);
        float vf[8];
        unpack8(gp.v[u], vf);
        l = l * corr + pw;
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = fmaf(pw, vf[i], acc[i] * corr);
        m = mn;
      }
    }
  };
  attn_key_loop<Group>(r.s0, r.s1, load_group, reduce_group);
  attn_merge_store(a, bh, split, m, l, acc);
}

// ---------------------------------------------------------------------------------------------
// Opt-in 8-bit KV rings (SURVEY.md 8f item 3; NOT the reference's numerics): the same fused step as attn_step_kernel
// over rings of one byte per element with one fp32 scale per (session, head, slot).  Halves the ring (0.81 GB instead
// of 1.57 GB per session at context 3000), i.e. doubles the sessions a GPU can hold.  Two encodings of a row x[128]:
//   KV_E4M3: e4m3(x * 448 / absmax), scale = absmax / 448   (keeps relative precision under outlier channels)
//   KV_INT8: round(x * 127 / absmax) + 128, scale = absmax / 127   (4x smaller error on smooth rows, cheaper decode:
//            PRMT places the byte under the fp16 exponent 0x64 (= 1024 + u exactly) and one HADD2 removes 1152)
// Append: the rotated key (rounded to bf16 first, like the bf16 ring) and the value are scaled and rounded to nearest
// even.  Attention: a half-warp owns one key (16 lanes x 8 bytes); keys and values are decoded to packed fp16 (exact),
// the dot product and the per-group weighted value sums run as HFMA2, and everything that accumulates over the ring
// (softmax statistics, output accumulator) stays fp32; the online softmax is updated once per group of keys.
// Supported query range: |q| <= 256 per element of the rotated query.  Each fp16 lane partial sums four products
// (q / sqrt(128)) * key byte value, at most 4 * 22.6 * 448 = 40 544 for e4m3 (int8: 11 494) against the fp16 limit 65 504, so a
// query lined up with its key overflows to inf (and the row's output to NaN) only past |q| ~ 413 (e4m3) / ~1460 (int8).
// ---------------------------------------------------------------------------------------------
constexpr int KV_E4M3 = 1, KV_INT8 = 2;       // = B200_KV_FP8_E4M3, B200_KV_INT8

struct AttnStepQ8 {
  const bf16* qkv; uint8_t* kc; uint8_t* vc; float* ks; float* vs; bf16* out;
  float* part; int* counters;
  const long long* pos; const uint8_t* exec_mask;
  int H, cap, nsplit; float neg_log_period_2_over_d;
};

__device__ __forceinline__ __half2 e4m3x2_to_half2(uint32_t two) {
  const __half2_raw hr = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(two & 0xFFFFu), __NV_E4M3);    // exact
  __half2 h2;
  memcpy(&h2, &hr, sizeof(h2));
  return h2;
}
__device__ __forceinline__ __half2 u8x2_to_half2(uint32_t w, uint32_t selector) {
  const uint32_t bits = __byte_perm(w, 0x64646464u, selector);     // [b, 0x64, b', 0x64] = (1024 + b, 1024 + b')
  __half2 h;
  memcpy(&h, &bits, sizeof(h));
  return __hsub2(h, __floats2half2_rn(1152.f, 1152.f));            // exact: values in [-128, 127]
}
template <int FMT>
__device__ __forceinline__ void unpack8_q8(const uint2& v, __half2* h) {
  if (FMT == KV_INT8) {
    h[0] = u8x2_to_half2(v.x, 0x4140u);
    h[1] = u8x2_to_half2(v.x, 0x4342u);
    h[2] = u8x2_to_half2(v.y, 0x4140u);
    h[3] = u8x2_to_half2(v.y, 0x4342u);
  } else {
    h[0] = e4m3x2_to_half2(v.x);
    h[1] = e4m3x2_to_half2(v.x >> 16);
    h[2] = e4m3x2_to_half2(v.y);
    h[3] = e4m3x2_to_half2(v.y >> 16);
  }
}
// two scaled values -> two ring bytes
template <int FMT>
__device__ __forceinline__ uint16_t quant2_q8(float x0, float x1) {
  if (FMT == KV_INT8) {
    const float r0 = fminf(fmaxf(rintf(x0), -127.f), 127.f), r1 = fminf(fmaxf(rintf(x1), -127.f), 127.f);
    return (uint16_t)((uint32_t)((int)r0 + 128) | ((uint32_t)((int)r1 + 128) << 8));
  }
  return (uint16_t)__nv_cvt_float2_to_fp8x2(make_float2(x0, x1), __NV_SATFINITE, __NV_E4M3);
}

template <int FMT>
static __global__ void __launch_bounds__(ATT_THREADS) attn_step_q8_kernel(const AttnStepQ8 a) {
  pdl_trigger();
  const int bh = blockIdx.x, split = blockIdx.y;
  const int b = bh / a.H, h = bh - b * a.H;
  const int C = a.H * ATT_D;
  const int tid = threadIdx.x, lane = tid & 31, l16 = lane & 15;
  const int hw = tid >> 4;                          // half-warp id 0..7
  const AttnRange r = attn_range(a, b, split);
  const bf16* base = a.qkv + (long long)b * 3 * C + h * ATT_D;
  const float fpos = (float)r.p;

  if (r.owns_new) {
    __shared__ float s_amax[2][2];
    float k0 = 0.f, k1 = 0.f, v0 = 0.f, v1 = 0.f;
    if (tid < ATT_D / 2) {
      const int pr = tid;
      rope_pair(bf2f(base[C + 2 * pr]), bf2f(base[C + 2 * pr + 1]), pr, fpos, a.neg_log_period_2_over_d, &k0, &k1);
      k0 = rbf(k0);
      k1 = rbf(k1);
      v0 = bf2f(base[2 * C + 2 * pr]);
      v1 = bf2f(base[2 * C + 2 * pr + 1]);
    }
    const float ak = warp_max(fmaxf(fabsf(k0), fabsf(k1))), av = warp_max(fmaxf(fabsf(v0), fabsf(v1)));
    if (tid < ATT_D / 2 && lane == 0) { s_amax[tid >> 5][0] = ak; s_amax[tid >> 5][1] = av; }
    __syncthreads();
    if (tid < ATT_D / 2) {
      const float amk = fmaxf(s_amax[0][0], s_amax[1][0]), amv = fmaxf(s_amax[0][1], s_amax[1][1]);
      constexpr float QMAX = FMT == KV_INT8 ? 127.f : 448.f;
      const float ik = amk > 0.f ? QMAX / amk : 0.f, iv = amv > 0.f ? QMAX / amv : 0.f;
      const long long o = ((long long)bh * a.cap + r.slot_new) * ATT_D + 2 * tid;
      *reinterpret_cast<uint16_t*>(a.kc + o) = quant2_q8<FMT>(k0 * ik, k1 * ik);
      *reinterpret_cast<uint16_t*>(a.vc + o) = quant2_q8<FMT>(v0 * iv, v1 * iv);
      if (tid == 0) {
        a.ks[(long long)bh * a.cap + r.slot_new] = amk * (1.f / QMAX);
        a.vs[(long long)bh * a.cap + r.slot_new] = amv * (1.f / QMAX);
      }
    }
    __syncthreads();
  }

  __half2 qh[4];
  attn_query(base, l16, fpos, a.neg_log_period_2_over_d, [&](int j, float x0, float x1) { qh[j] = __floats2half2_rn(x0, x1); });

  const uint8_t* kb = a.kc + (long long)bh * a.cap * ATT_D + l16 * 8;
  const uint8_t* vb = a.vc + (long long)bh * a.cap * ATT_D + l16 * 8;
  const float* ksb = a.ks + (long long)bh * a.cap;
  const float* vsb = a.vs + (long long)bh * a.cap;
  float m = -INFINITY, l = 0.f, acc[8] = {};

  // Double buffering makes a warp's time per group max(memory latency, arithmetic) instead of their sum (the bf16 kernel could
  // afford the sum: it moves twice the bytes per key).
  constexpr int U = ATT_GROUP;
  struct Group { uint2 k[U], v[U]; float ks[U], vs[U]; };
  auto load_group = [&](int kb0, Group& gp) {
    const int s = kb0 + hw * U;
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int ss = s + u < r.s1 ? s + u : r.s1 - 1;
      gp.k[u] = *reinterpret_cast<const uint2*>(kb + (long long)ss * ATT_D);
      gp.v[u] = *reinterpret_cast<const uint2*>(vb + (long long)ss * ATT_D);
      gp.ks[u] = ksb[ss];
      gp.vs[u] = vsb[ss];
    }
  };
  auto reduce_group = [&](int kb0, const Group& gp) {
    const int s = kb0 + hw * U;
    float d[U];
    float mn = m;
#pragma unroll
    for (int u = 0; u < U; ++u) {
      __half2 kh[4];
      unpack8_q8<FMT>(gp.k[u], kh);
      __half2 t2 = __hmul2(qh[0], kh[0]);
      t2 = __hfma2(qh[1], kh[1], t2);
      t2 = __hfma2(qh[2], kh[2], t2);
      t2 = __hfma2(qh[3], kh[3], t2);
      const float2 tf = __half22float2(t2);
      float t = tf.x + tf.y;
      t += __shfl_xor_sync(0xffffffffu, t, 8);
      t += __shfl_xor_sync(0xffffffffu, t, 4);
      t += __shfl_xor_sync(0xffffffffu, t, 2);
      t += __shfl_xor_sync(0xffffffffu, t, 1);
      d[u] = s + u < r.s1 ? t * gp.ks[u] : -INFINITY;
      mn = fmaxf(mn, d[u]);
    }
    if (mn > -INFINITY) {                           // uniform over the half-warp; no shuffles inside
      const float corr = __expf(m - mn);            // m = -inf -> 0
      __half2 g[4];                                 // this group's weighted value sum, packed fp16
#pragma unroll
      for (int i = 0; i < 4; ++i) g[i] = __floats2half2_rn(0.f, 0.f);
      float lsum = 0.f;
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const float pw = __expf(d[u] - mn);         // padding keys: exp(-inf) = 0
        lsum += pw;
        const __half2 pv = __float2half2_rn(pw * gp.vs[u]);
        __half2 vh[4];
        unpack8_q8<FMT>(gp.v[u], vh);
#pragma unroll
        for (int i = 0; i < 4; ++i) g[i] = __hfma2(pv, vh[i], g[i]);
      }
      l = fmaf(l, corr, lsum);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 gf = __half22float2(g[i]);
        acc[2 * i] = fmaf(acc[2 * i], corr, gf.x);
        acc[2 * i + 1] = fmaf(acc[2 * i + 1], corr, gf.y);
      }
      m = mn;
    }
  };
  attn_key_loop<Group>(r.s0, r.s1, load_group, reduce_group);
  attn_merge_store(a, bh, split, m, l, acc);
}

// One layer's temporal K/V as the attention step reads them: bf16 rings [B][H][cap][ATT_D], or with a page table [B][tab_ld] the
// pools [n_pages + 1][H][1 << page_shift][ATT_D]; 8-bit rings: bytes [B][H][cap][ATT_D] and fp32 scales ks / vs [B][H][cap].
struct KvRings {
  void *k = nullptr, *v = nullptr;
  float *ks = nullptr, *vs = nullptr;
  const int* table = nullptr; int tab_ld = 0, page_shift = 0;
};

// One temporal attention step of B rows over rings stored as `storage` (0 = bf16, KV_E4M3, KV_INT8); nsplit >= 1 splits per
// (b, h), whose partials and arrival counters are part [B*H][nsplit][ATT_D + 2] and counters [B*H] (zero between launches).
// Defined in lm.cu, so the kernels are compiled once for the handle and the b200_op_attn_step* entry points.
void attn_step_launch(const bf16* qkv, const KvRings& r, bf16* out, float* part, int* counters, const long long* pos,
                      const uint8_t* exec_mask, int B, int H, int cap, int nsplit, float max_period, int storage, cudaStream_t st);

// ---------------------------------------------------------------------------------------------
// LayerNorm with weight and bias (the cross-attention layers' norm_cross, nn.LayerNorm(dim, eps=1e-5), transformer.py:727-732):
// bf16 in and out, fp32 statistics (the mean, then the mean of the squared deviations), y = bf16((x - mean) * rstd * w + b).
// One 256-thread CTA per row.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float block_sum_256(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();                                 // red is reused by consecutive calls
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) t += red[w];
  return t;
}

static __global__ void __launch_bounds__(256) layernorm_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w,
                                                        const bf16* __restrict__ bias, bf16* __restrict__ y, int dim, float eps) {
  pdl_trigger();
  __shared__ float red[8];
  const bf16* xr = x + (long long)blockIdx.x * dim;
  float s = 0.f;
  for (int c = threadIdx.x * 2; c < dim; c += 512) {
    const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(xr + c));
    s += v.x + v.y;
  }
  const float mean = block_sum_256(s, red) / (float)dim;
  float ss = 0.f;
  for (int c = threadIdx.x * 2; c < dim; c += 512) {
    const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(xr + c));
    ss += (v.x - mean) * (v.x - mean) + (v.y - mean) * (v.y - mean);
  }
  const float rstd = rsqrtf(block_sum_256(ss, red) / (float)dim + eps);
  for (int c = threadIdx.x * 2; c < dim; c += 512) {
    const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(xr + c));
    const float2 g = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(w + c));
    const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(bias + c));
    *reinterpret_cast<__nv_bfloat162*>(y + (long long)blockIdx.x * dim + c) =
        __floats2bfloat162_rn((v.x - mean) * rstd * g.x + b.x, (v.y - mean) * rstd * g.y + b.y);
  }
}

// ---------------------------------------------------------------------------------------------
// Cross-attention step of a temporal layer (transformer.py:544-597 with cross_attention=True): one query per (row, head)
// against all T keys of that row's condition memory k_cross / v_cross [B][H][T][ATT_D].  No RoPE, no mask, no append and no
// exec mask: every row computes, as in the reference.  The CTA layout, the key loop and the split merge are attn_step_kernel's
// (grid = (B*H, nsplit), 128 threads, a half-warp per key, partials merged in split order); only the query load (no rotation)
// and the key range [0, T) differ.  q [B][ldq] bf16, head h at columns [h * ATT_D, (h + 1) * ATT_D).
// ---------------------------------------------------------------------------------------------
struct CrossAttnStep {
  const bf16* q; long long ldq;
  const bf16* kc; const bf16* vc;              // [B][H][T][ATT_D]
  bf16* out;                                   // [B][H * ATT_D]
  float* part; int* counters;                  // [B*H][nsplit][ATT_D + 2], [B*H] (zero between launches)
  int H, T, nsplit;
};

static __global__ void __launch_bounds__(ATT_THREADS) cross_attn_step_kernel(const CrossAttnStep a) {
  pdl_trigger();
  const int bh = blockIdx.x, split = blockIdx.y;
  const int b = bh / a.H, h = bh - b * a.H;
  const int tid = threadIdx.x, l16 = tid & 15;
  const int hw = tid >> 4;                          // half-warp id 0..7
  const int per = (a.T + a.nsplit - 1) / a.nsplit;
  const int s0 = split * per, s1 = min(s0 + per, a.T);

  float qf[8];
  unpack8(*reinterpret_cast<const uint4*>(a.q + (long long)b * a.ldq + h * ATT_D + l16 * 8), qf);
  const float scale = 0.08838834764831845f;       // 1/sqrt(128)
#pragma unroll
  for (int i = 0; i < 8; ++i) qf[i] *= scale;

  const long long row0 = (long long)bh * a.T * ATT_D;
  const bf16* kb = a.kc + row0 + l16 * 8;
  const bf16* vb = a.vc + row0 + l16 * 8;
  float m = -INFINITY, l = 0.f, acc[8] = {};

  constexpr int U = ATT_GROUP;
  struct Group { uint4 k[U], v[U]; };
  auto load_group = [&](int kb0, Group& gp) {
    const int s = kb0 + hw * U;
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long o = (long long)(s + u < s1 ? s + u : s1 - 1) * ATT_D;
      gp.k[u] = *reinterpret_cast<const uint4*>(kb + o);
      gp.v[u] = *reinterpret_cast<const uint4*>(vb + o);
    }
  };
  auto reduce_group = [&](int kb0, const Group& gp) {
    const int s = kb0 + hw * U;
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float kf[8];
      unpack8(gp.k[u], kf);
      float d = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) d = fmaf(qf[i], kf[i], d);
      d += __shfl_xor_sync(0xffffffffu, d, 8);
      d += __shfl_xor_sync(0xffffffffu, d, 4);
      d += __shfl_xor_sync(0xffffffffu, d, 2);
      d += __shfl_xor_sync(0xffffffffu, d, 1);
      if (s + u < s1) {
        const float mn = fmaxf(m, d);
        const float corr = __expf(m - mn), pw = __expf(d - mn);
        float vf[8];
        unpack8(gp.v[u], vf);
        l = l * corr + pw;
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = fmaf(pw, vf[i], acc[i] * corr);
        m = mn;
      }
    }
  };
  attn_key_loop<Group>(s0, s1, load_group, reduce_group);
  attn_merge_store(a, bh, split, m, l, acc);
}

// The cross-attention K/V of condition rows (transformer.py:495-505: kv = src @ W[d:]^T, "b t (p h d) -> p b h t d") from a
// chunk of the projection, kv [n][2 * H * ATT_D] = flat rows [i0, i0 + n) of (condition row r, t), into the condition memory
// k_cross / v_cross [B][H][T][ATT_D] of model row rows[r].  One thread per 16 bytes.
static __global__ void cross_kv_scatter_kernel(const bf16* __restrict__ kv, long long i0, int n, const int* __restrict__ rows,
                                               bf16* __restrict__ kc, bf16* __restrict__ vc, int H, int T) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int per_row = 2 * H * (ATT_D / 8);
  if (i >= (long long)n * per_row) return;
  const int j = (int)(i / per_row), e = (int)(i - (long long)j * per_row);
  const int p = e / (H * (ATT_D / 8)), hh = (e / (ATT_D / 8)) % H, c = e % (ATT_D / 8);
  const long long g = i0 + j;
  const int r = (int)(g / T), t = (int)(g - (long long)r * T);
  bf16* dst = (p ? vc : kc) + (((long long)rows[r] * H + hh) * T + t) * ATT_D + c * 8;
  *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(kv + (long long)j * 2 * H * ATT_D + (long long)p * H * ATT_D + hh * ATT_D + c * 8);
}

// One cross-attention step of B rows over condition memories of T keys (defined in lm.cu next to attn_step_launch)
void cross_attn_launch(const bf16* q, long long ldq, const bf16* kc, const bf16* vc, bf16* out, float* part, int* counters, int B,
                       int H, int T, int nsplit, cudaStream_t st);

constexpr int DEP_MAX_Q = 16;              // dep_q of the largest family member (configs/moshi_dev_2b.json)
constexpr int DEP_LOW_RANK_MAX = 4096;     // rank of low-rank depformer embeddings: lowrank_expand_kernel keeps a row in shared memory

// Depformer attention step: the new key/value of sub-step `step` is appended to the per-frame cache and the query
// attends over step + 1 keys; no positional embedding (depformer_pos_emb = "none").  One warp per (b, h), D = 64.
static __global__ void dep_attn_step_kernel(const bf16* __restrict__ qkv /*[B][3*H*D]*/, bf16* __restrict__ kc,
                                     bf16* __restrict__ vc, bf16* __restrict__ out, int B, int H, int cap, int step) {
  pdl_trigger();
  constexpr int D = 64;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B * H) return;
  const int b = warp / H, h = warp - b * H;
  const int C = H * D;
  const bf16* base = qkv + (long long)b * 3 * C + h * D + 2 * lane;
  const long long row = (long long)warp * cap;
  *reinterpret_cast<__nv_bfloat162*>(kc + (row + step) * D + 2 * lane) = *reinterpret_cast<const __nv_bfloat162*>(base + C);
  *reinterpret_cast<__nv_bfloat162*>(vc + (row + step) * D + 2 * lane) = *reinterpret_cast<const __nv_bfloat162*>(base + 2 * C);
  __syncwarp();
  const float2 q = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(base));
  const float scale = 0.125f;                       // 1/sqrt(64)
  float sc[DEP_MAX_Q];
  float mx = -INFINITY;
  const int n_keys = step + 1;
  for (int j = 0; j < n_keys; ++j) {
    const float2 kk = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(kc + (row + j) * D + 2 * lane));
    const float d = warp_sum(q.x * kk.x + q.y * kk.y) * scale;
    sc[j] = d;
    mx = fmaxf(mx, d);
  }
  float sum = 0.f;
  for (int j = 0; j < n_keys; ++j) { sc[j] = expf(sc[j] - mx); sum += sc[j]; }
  const float inv = 1.f / sum;
  float a0 = 0.f, a1 = 0.f;
  for (int j = 0; j < n_keys; ++j) {
    const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(vc + (row + j) * D + 2 * lane));
    a0 = fmaf(sc[j] * inv, v.x, a0);
    a1 = fmaf(sc[j] * inv, v.y, a1);
  }
  *reinterpret_cast<__nv_bfloat162*>(out + (long long)warp * D + 2 * lane) = __floats2bfloat162_rn(a0, a1);
}

// _LMGenState.reset / _MHAState.reset / RingKVCache.reset / State.reset for the rows in `mask` (null = all)
// (with CFG the model rows b and B + b are reset together, lm.py:653-656)
static __global__ void lm_reset_kernel(long long* offsets, long long* pos, uint8_t* exec_mask, uint8_t* exec_mask_m, const uint8_t* mask,
                                int B, int cfg) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  if (mask != nullptr && !mask[b]) return;
  offsets[b] = 0;
  pos[b] = 0;
  exec_mask[b] = 1;
  exec_mask_m[b] = 1;
  if (cfg) { pos[B + b] = 0; exec_mask_m[B + b] = 1; }
}

// depformer_replace_tokens [B][dep_q] -> this frame's audio tokens [dep_q][B] (lm.py:751-755)
static __global__ void replace_audio_kernel(const long long* __restrict__ given, long long* __restrict__ audio_tokens, int B, int dep_q) {
  pdl_trigger();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * dep_q) return;
  const int b = i / dep_q, k = i - b * dep_q;
  audio_tokens[(long long)k * B + b] = given[i];
}

// rings shorter than the model's context (b200_lm_set_kv_capacity): a row about to write position >= cap would overwrite keys the
// reference still attends to -> ERR_KV_CAPACITY (the step still runs, as a ring of `cap` slots)
static __global__ void kv_capacity_check_kernel(const long long* __restrict__ pos, const uint8_t* __restrict__ exec_mask, int B, int cap,
                                                int* err) {
  pdl_trigger();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B && exec_mask[b] && pos[b] >= cap && err != nullptr) atomicOr(err, ERR_KV_CAPACITY);
}

// ---------------------------------------------------------------------------------------------
// Paged temporal KV pool (b200_lm_set_kv_pool): one page table [MB][tab_ld] shared by all layers (-1 = unmapped), a stack of
// free page ids and its top, all on the device.  A row holds its pages as a prefix of its table (held[b] of them); entries
// past that prefix are unmapped, or the sink page n_pages while the pool is dry.  One CTA of KV_PAGE_THREADS >= MB threads
// scans the rows in row order, so which row gets which page is deterministic.
// ---------------------------------------------------------------------------------------------
constexpr int KV_PAGE_THREADS = 256;

__device__ __forceinline__ int block_inclusive_scan(int v, int* s) {
  const int t = threadIdx.x;
  s[t] = v;
  __syncthreads();
  for (int o = 1; o < KV_PAGE_THREADS; o <<= 1) {
    const int w = t >= o ? s[t - o] : 0;
    __syncthreads();
    s[t] += w;
    __syncthreads();
  }
  return s[t];
}

// Before the first layer of a step: every executing row gets pages until slots [0, min(pos + 1, cap)) are mapped.  A row the
// pool cannot serve maps its missing entries to the sink page and raises ERR_KV_POOL; it keeps asking every step.
static __global__ void __launch_bounds__(KV_PAGE_THREADS) kv_page_alloc_kernel(int* __restrict__ table, int* __restrict__ held,
    const int* __restrict__ free_stack, int* __restrict__ top, const long long* __restrict__ pos, const uint8_t* __restrict__ exec_mask,
    int B, int tab_ld, int page_shift, int cap, int sink, int* err) {
  __shared__ int s[KV_PAGE_THREADS];
  pdl_trigger();
  const int b = threadIdx.x;
  int have = 0, need = 0;
  if (b < B && exec_mask[b]) {
    const long long n = min(pos[b] + 1, (long long)cap);
    const int want = (int)((n + (1 << page_shift) - 1) >> page_shift);
    have = held[b];
    need = max(want - have, 0);
  }
  const int end = block_inclusive_scan(need, s), start = end - need;
  const int avail = *top;
  const int total = s[KV_PAGE_THREADS - 1];
  __syncthreads();                     // every thread has read the top before it moves
  if (need > 0) {
    int* row = table + (long long)b * tab_ld;
    int got = 0;
    for (int i = 0; i < need; ++i) {
      const int k = start + i;         // this row's i-th page is the k-th pop of this step
      if (k < avail) { row[have + i] = free_stack[avail - 1 - k]; ++got; }
      else row[have + i] = sink;
    }
    held[b] = have + got;
    if (got < need && err != nullptr) atomicOr(err, ERR_KV_POOL);
  }
  if (b == 0) *top = avail - min(total, avail);
}

// b200_lm_reset: the masked sessions' rows (b and b + B under CFG, lm.py:653-656; null mask = all) push their pages back in row
// and table order and become unmapped.
static __global__ void __launch_bounds__(KV_PAGE_THREADS) kv_page_free_kernel(int* __restrict__ table, int* __restrict__ held,
    int* __restrict__ free_stack, int* __restrict__ top, const uint8_t* __restrict__ mask, int B, int MB, int tab_ld) {
  __shared__ int s[KV_PAGE_THREADS];
  const int r = threadIdx.x;
  const bool f = r < MB && (mask == nullptr || mask[r < B ? r : r - B]);
  const int n = f ? held[r] : 0;
  const int end = block_inclusive_scan(n, s), start = end - n;
  const int t0 = *top;
  const int total = s[KV_PAGE_THREADS - 1];
  __syncthreads();
  if (f) {
    int* row = table + (long long)r * tab_ld;
    for (int i = 0; i < n; ++i) free_stack[t0 + start + i] = row[i];
    for (int i = 0; i < tab_ld; ++i) row[i] = -1;
    held[r] = 0;
  }
  if (r == 0) *top = t0 + total;
}

// Temporal K/V rings <-> a flat buffer [array][k][H][n][slot] for model rows b = row0 + k * row_step, k < n_rows: the streaming
// state's view of a paged layer (one array, every row, n = cap) and a session record (every layer's K and V, the session's 1 or
// 2 rows, n = its fill).  `arrays` are the rings [MB][H][cap][slot] or, with a page table, the pools [n_pages + 1][H][page][slot].
// A slot is valid below the row's fill min(pos, cap) on a mapped, non-sink page: GATHER writes zeros for the others, the scatter
// leaves them alone.  blockIdx.y = (array, k, head); V units of type U per slot.
struct KvCopy {
  void* const* arrays;
  void* flat;
  const int* table;            // [MB][tab_ld], or nullptr: contiguous rings
  const long long* pos;
  int tab_ld, page_shift, sink;
  int row0, n_rows, row_step, H, cap, n;
};
template <bool GATHER, typename U, int V>
static __global__ void kv_copy_kernel(KvCopy a) {
  const int seg = blockIdx.y;
  const int h = seg % a.H, k = (seg / a.H) % a.n_rows, arr = seg / (a.H * a.n_rows);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n * V) return;
  const int s = i / V, c = i - s * V;
  const int b = a.row0 + k * a.row_step;
  bool valid = s < min(a.pos[b], (long long)a.cap);
  long long r;
  if (a.table != nullptr) {
    const int pg = a.table[(long long)b * a.tab_ld + (s >> a.page_shift)];
    valid = valid && pg >= 0 && pg < a.sink;
    r = kv_paged_row(pg, a.H, h, s, a.page_shift) * V + c;
  } else {
    r = (((long long)b * a.H + h) * a.cap + s) * V + c;
  }
  U* ring = static_cast<U*>(a.arrays[arr]);
  U* fv = static_cast<U*>(a.flat) + (long long)seg * a.n * V + i;
  if (GATHER) *fv = valid ? ring[r] : U{};
  else if (valid) ring[r] = *fv;
}

static __global__ void advance_pos_kernel(long long* pos, const uint8_t* exec_mask, int B) {
  pdl_trigger();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B && exec_mask[b]) pos[b] += 1;
}

// ---------------------------------------------------------------------------------------------
// sample_token (sampling.py:86-106): softmax(logits/temp) -> top-k -> argmax(p / Exp(1) noise).
// Candidates are ranked by (logit desc, index asc); the noise is indexed by rank like the
// reference indexes it by the position in torch.topk's sorted output.
// ---------------------------------------------------------------------------------------------
constexpr int SAMPLE_THREADS = 256;
constexpr int SAMPLE_MAX_K = 1024;

__device__ __forceinline__ unsigned sample_key(const bf16* logits, int i) {
  const unsigned short raw = __bfloat16_as_ushort(logits[i]);
  const unsigned short mono = (raw & 0x8000u) ? (unsigned short)~raw : (unsigned short)(raw | 0x8000u);
  return ((unsigned)mono << 16) | (unsigned)(0xFFFFu - (unsigned)i);
}

// Per-session sampling settings of one row (b200_lm_set_row_sampling), all fp32 so that the row is one state entry row.
// own = 0: the row follows the handle-wide temperatures and top-k, with no pad bias and no repetition penalty.
struct RowSampling { float temp_text, temp, top_k_text, top_k, pad_mult, context, penalty, own; };
constexpr int TEXT_PAD_ID = 3;               // existing_text_padding_id: the token pad_mult biases, skipped by the history

// the temperature and top-k row b samples with: its own where it has them, else the handle's (*temp, *top_k on entry).  The own
// top-k is clamped to [1, the handle's] here, at every step, and not only where the settings are set: settings that arrive
// through a session record or a state snapshot of a handle with a larger top-k must still draw within the row's noise block.
__device__ __forceinline__ void row_sampling(const RowSampling* rs, int b, bool text, float* temp, int* top_k) {
  if (rs != nullptr && rs[b].own != 0.f) {
    const float k = text ? rs[b].top_k_text : rs[b].top_k;
    *temp = text ? rs[b].temp_text : rs[b].temp;
    *top_k = k >= 1.f ? (int)fminf(k, (float)*top_k) : 1;
  }
}

// Where the sampler's scores come from.  bf16 logits: the score is logit / temp, the key (monotone bf16 bits, 0xFFFF - index)
// in 32 bits, four radix passes.  fp32 scores (text_adjust_kernel: penalised logits, already / temp with the pad bias on
// sampling rows): the score as it is, the key (monotone fp32 bits, 0xFFFF - index) in the low 48 bits of a 64-bit word, six
// passes.  On an unadjusted row the fp32 scores are the bf16 path's logit / temp, so both pick the same token.
template <typename T> struct SampleSrc;
template <> struct SampleSrc<bf16> {
  typedef unsigned Key;
  static constexpr int PASSES = 4;
  static __device__ __forceinline__ float score(const bf16* p, int i, float temp) { return bf2f(p[i]) / temp; }
  static __device__ __forceinline__ Key key(const bf16* p, int i) { return sample_key(p, i); }
};
template <> struct SampleSrc<float> {
  typedef unsigned long long Key;
  static constexpr int PASSES = 6;
  static __device__ __forceinline__ float score(const float* p, int i, float) { return p[i]; }
  static __device__ __forceinline__ Key key(const float* p, int i) {
    const unsigned raw = __float_as_uint(p[i]);
    const unsigned mono = (raw & 0x80000000u) ? ~raw : (raw | 0x80000000u);
    return ((Key)mono << 16) | (Key)(0xFFFFu - (unsigned)i);
  }
};

static __device__ float block_reduce(float v, bool is_max, float* red) {
  v = is_max ? warp_max(v) : warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = is_max ? -INFINITY : 0.f;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t = is_max ? fmaxf(t, red[w]) : t + red[w];
  return t;
}

// One row per call; every thread of a SAMPLE_THREADS-wide CTA must call it (block-wide barriers inside).  T: bf16 logits or
// fp32 scores (SampleSrc).  Thread 0 writes *out.
template <typename T>
static __device__ void sample_row(const T* __restrict__ logits, const float* __restrict__ noise, long long* __restrict__ out,
                                  int card, int use_sampling, float temp, int top_k) {
  typedef SampleSrc<T> S;
  typedef typename S::Key Key;
  __shared__ float red[SAMPLE_THREADS / 32];
  __shared__ unsigned hist[256];
  __shared__ Key s_prefix;
  __shared__ unsigned s_remaining, s_count;
  __shared__ Key sel[SAMPLE_MAX_K];
  __shared__ float s_best[SAMPLE_THREADS / 32];
  __shared__ int s_brank[SAMPLE_THREADS / 32];
  const int tid = threadIdx.x;

  if (!(use_sampling && temp > 0.f)) {        // greedy: argmax, first maximum (sampling.py:102-103)
    Key best = 0;
    for (int i = tid; i < card; i += SAMPLE_THREADS) best = max(best, S::key(logits, i));
    for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
    if ((tid & 31) == 0) sel[tid >> 5] = best;
    __syncthreads();
    if (tid == 0) {
      Key bb = 0;
      for (int w = 0; w < SAMPLE_THREADS / 32; ++w) bb = max(bb, sel[w]);
      *out = 0xFFFFu - (unsigned)(bb & 0xFFFFu);
    }
    return;
  }
  const int k = min(min(top_k, card), SAMPLE_MAX_K);
  // softmax statistics in fp32 on the scores (logits / temp)
  float mx = -INFINITY;
  for (int i = tid; i < card; i += SAMPLE_THREADS) mx = fmaxf(mx, S::score(logits, i, temp));
  mx = block_reduce(mx, true, red);
  float sum = 0.f;
  for (int i = tid; i < card; i += SAMPLE_THREADS) sum += expf(S::score(logits, i, temp) - mx);
  sum = block_reduce(sum, false, red);

  // radix select of the k-th largest key (keys are unique)
  if (tid == 0) { s_prefix = 0; s_remaining = (unsigned)k; }
  __syncthreads();
  for (int pass = S::PASSES - 1; pass >= 0; --pass) {
    hist[tid] = 0;
    __syncthreads();
    const Key prefix = s_prefix;
    const Key mask = pass == S::PASSES - 1 ? (Key)0 : (~(Key)0 << ((pass + 1) * 8));
    for (int i = tid; i < card; i += SAMPLE_THREADS) {
      const Key key = S::key(logits, i);
      if ((key & mask) == prefix) atomicAdd(&hist[(unsigned)(key >> (pass * 8)) & 0xFFu], 1u);
    }
    __syncthreads();
    if (tid < 32) {
      // the bin of the rem-th largest key, scanning the 256 counts from the top: lane l owns bins 8l .. 8l+7, a suffix sum over
      // the lanes finds the one lane whose bins contain it (the serial scan by one thread cost ~4 us per pass)
      const unsigned rem = s_remaining;
      unsigned h8[8], own = 0;
#pragma unroll
      for (int i = 0; i < 8; ++i) { h8[i] = hist[tid * 8 + i]; own += h8[i]; }
      unsigned incl = own;                         // counts in this lane's bins and every higher lane's
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned v = __shfl_down_sync(0xffffffffu, incl, o);
        if (tid + o < 32) incl += v;
      }
      unsigned cum = incl - own;                   // counts in bins above this lane's
      if (cum < rem && rem <= incl) {
        int bin = tid * 8;
#pragma unroll
        for (int i = 7; i >= 0; --i) {
          if (cum + h8[i] >= rem) { bin = tid * 8 + i; break; }
          cum += h8[i];
        }
        s_remaining = rem - cum;
        s_prefix = prefix | ((Key)bin << (pass * 8));
      }
    }
    __syncthreads();
  }
  const Key thr = s_prefix;                    // exactly k keys are >= thr
  if (tid == 0) s_count = 0;
  // pad the sort buffer
  int p2 = 1;
  while (p2 < k) p2 <<= 1;
  for (int i = tid; i < p2; i += SAMPLE_THREADS) sel[i] = 0;
  __syncthreads();
  for (int i = tid; i < card; i += SAMPLE_THREADS) {
    const Key key = S::key(logits, i);
    if (key >= thr) {
      const unsigned slot = atomicAdd(&s_count, 1u);
      if (slot < (unsigned)p2) sel[slot] = key;
    }
  }
  __syncthreads();
  // bitonic sort, descending
  for (int size = 2; size <= p2; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = tid; i < p2 / 2; i += SAMPLE_THREADS) {
        const int lo = 2 * i - (i & (stride - 1));
        const int hi = lo + stride;
        const bool desc = ((lo & size) == 0);
        const Key a = sel[lo], b = sel[hi];
        if ((a < b) == desc) { sel[lo] = b; sel[hi] = a; }
      }
      __syncthreads();
    }
  }
  // argmax over ranks of p / q (first maximum wins, like torch.argmax)
  float best = -INFINITY;
  int brank = 0x7fffffff;
  for (int j = tid; j < k; j += SAMPLE_THREADS) {
    const int idx = 0xFFFF - (int)(sel[j] & 0xFFFFu);
    const float p = expf(S::score(logits, idx, temp) - mx) / sum;
    const float s = p / noise[j];
    if (s > best || (s == best && j < brank)) { best = s; brank = j; }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oj = __shfl_xor_sync(0xffffffffu, brank, o);
    if (ob > best || (ob == best && oj < brank)) { best = ob; brank = oj; }
  }
  if ((tid & 31) == 0) { s_best[tid >> 5] = best; s_brank[tid >> 5] = brank; }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < SAMPLE_THREADS / 32; ++w)
      if (s_best[w] > best || (s_best[w] == best && s_brank[w] < brank)) { best = s_best[w]; brank = s_brank[w]; }
    if (brank == 0x7fffffff) brank = 0;
    *out = 0xFFFF - (int)(sel[brank] & 0xFFFFu);
  }
}

// rs: per-row settings (null, or rows without their own: temp / top_k); text: rs's text or audio fields
static __global__ void __launch_bounds__(SAMPLE_THREADS) sample_kernel(const bf16* __restrict__ logits_all, long long ld,
                                                                const float* __restrict__ noise, long long noise_ld,
                                                                long long* __restrict__ out, int card, int use_sampling,
                                                                float temp, int top_k, const RowSampling* rs, int text) {
  pdl_trigger();
  const int row = blockIdx.x;
  row_sampling(rs, row, text != 0, &temp, &top_k);
  sample_row(logits_all + (long long)row * ld, noise + (long long)row * noise_ld, out + row, card, use_sampling, temp, top_k);
}

// ---------------------------------------------------------------------------------------------
// Per-session text sampling (lm_generate_multistream.rs:142-175, 247-255): repetition penalty over the row's recent text,
// temperature and pad bias, into fp32 scores; then the shared sampler on them, and the row's history ring.
// ---------------------------------------------------------------------------------------------
struct TextHistory {
  int* ring;                 // [B][N] the row's generated text tokens, the special ids left out; slot count % N is the next
  int* count;                // [B] tokens appended since the last reset
  int N;
};

__device__ __forceinline__ bool text_special(int t, int text_card) { return t == 0 || t == TEXT_PAD_ID || t == text_card; }

// One CTA per row.  The penalty window: the newest `context` entries of the ring that are not special ids, each distinct id
// penalised once (a bitmap of card bits in shared memory, 8 KB at 65 535 ids).  Greedy rows get the penalised logits.
static __global__ void __launch_bounds__(SAMPLE_THREADS) text_adjust_kernel(const bf16* __restrict__ logits, float* __restrict__ scores,
                                                                     int card, int use_sampling, float temp,
                                                                     const RowSampling* __restrict__ rs, TextHistory th) {
  __shared__ unsigned bits[2048];
  __shared__ int s_warp[SAMPLE_THREADS / 32];
  const int b = blockIdx.x, tid = threadIdx.x;
  const RowSampling r = rs[b];
  float pen = 1.f, pad = 0.f;
  int ctx = 0;
  if (r.own != 0.f) { temp = r.temp_text; pen = r.penalty; pad = r.pad_mult; ctx = (int)r.context; }
  const bool sampling = use_sampling && temp > 0.f;
  const int cnt = th.count[b];
  const int n = min(cnt, th.N);
  const bool penal = pen != 1.f && ctx > 0 && n > 0;
  if (penal) {
    const int words = (card + 31) >> 5;
    for (int i = tid; i < words; i += SAMPLE_THREADS) bits[i] = 0u;
    __syncthreads();
    int taken = 0;                                      // window entries before this chunk (same value in every thread)
    for (int base = 0; base < n && taken < ctx; base += SAMPLE_THREADS) {
      const int j = base + tid;                         // the j-th newest entry
      int t = -1;
      if (j < n) t = th.ring[(long long)b * th.N + ((cnt - 1 - j) % th.N + th.N) % th.N];
      const bool keep = j < n && t >= 0 && t < card && !text_special(t, card);
      const unsigned bal = __ballot_sync(0xffffffffu, keep);
      if ((tid & 31) == 0) s_warp[tid >> 5] = __popc(bal);
      __syncthreads();
      int before = taken;
      for (int w = 0; w < (tid >> 5); ++w) before += s_warp[w];
      before += __popc(bal & ((1u << (tid & 31)) - 1u));
      if (keep && before < ctx) atomicOr(&bits[t >> 5], 1u << (t & 31));
      for (int w = 0; w < SAMPLE_THREADS / 32; ++w) taken += s_warp[w];
      __syncthreads();
    }
  }
  const bf16* lg = logits + (long long)b * card;
  float* sc = scores + (long long)b * card;
  for (int i = tid; i < card; i += SAMPLE_THREADS) {
    float l = bf2f(lg[i]);
    if (penal && (bits[i >> 5] >> (i & 31)) & 1u) l = l >= 0.f ? l / pen : l * pen;
    if (sampling) {
      l = l / temp;
      if (i == TEXT_PAD_ID && pad != 0.f) l += pad;
    }
    sc[i] = l;
  }
}

// The text sampler on the adjusted scores, then the row's history: the token is appended when the row executed this step
// (exec_mask null: every row did) and it is not a special id.
static __global__ void __launch_bounds__(SAMPLE_THREADS) sample_text_kernel(const float* __restrict__ scores, const float* __restrict__ noise,
                                                                     long long noise_ld, long long* __restrict__ out, int card,
                                                                     int use_sampling, float temp, int top_k, const RowSampling* rs,
                                                                     TextHistory th, const uint8_t* exec_mask) {
  const int row = blockIdx.x;
  row_sampling(rs, row, true, &temp, &top_k);
  sample_row(scores + (long long)row * card, noise + (long long)row * noise_ld, out + row, card, use_sampling, temp, top_k);
  if (threadIdx.x == 0 && (exec_mask == nullptr || exec_mask[row])) {
    const int t = (int)out[row];
    if (!text_special(t, card)) {
      const int c = max(th.count[row], 0);           // a count from a state snapshot is not trusted to be in range
      th.ring[(long long)row * th.N + c % th.N] = t;
      th.count[row] = c + 1;
    }
  }
}

// b200_lm_reset: the masked rows' histories are emptied (null mask: all); their settings stay
static __global__ void text_history_clear_kernel(int* count, const uint8_t* mask, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B && (mask == nullptr || mask[b])) count[b] = 0;
}

// Host: b200_row_sampling -> the row's device settings; B200_ERR_INVALID outside the ranges of moshi_b200.h (top-k capped by
// the handle's, whose top-k lays out the noise rows)
inline int row_sampling_check(const b200_row_sampling& p, int top_k, int top_k_text, RowSampling* out, const char* what) {
  const bool temps = std::isfinite(p.temp) && std::isfinite(p.temp_text) && p.temp >= 0.f && p.temp_text >= 0.f;
  if (!temps) B200_FAIL(B200_ERR_INVALID, "%s: temperatures %g / %g (finite, >= 0)", what, p.temp_text, p.temp);
  if (p.top_k < 1 || p.top_k > top_k || p.top_k_text < 1 || p.top_k_text > top_k_text)
    B200_FAIL(B200_ERR_INVALID, "%s: top_k %d / top_k_text %d outside [1, %d] / [1, %d] (the handle's)", what, p.top_k, p.top_k_text,
              top_k, top_k_text);
  if (!std::isfinite(p.pad_mult)) B200_FAIL(B200_ERR_INVALID, "%s: pad_mult %g", what, p.pad_mult);
  if (p.repetition_context < 0 || p.repetition_context > 1024)
    B200_FAIL(B200_ERR_INVALID, "%s: repetition_context %d outside [0, 1024]", what, p.repetition_context);
  if (!(p.repetition_penalty > 0.f && p.repetition_penalty <= 1000.f))
    B200_FAIL(B200_ERR_INVALID, "%s: repetition_penalty %g outside (0, 1000]", what, p.repetition_penalty);
  *out = RowSampling{p.temp_text, p.temp, (float)p.top_k_text, (float)p.top_k, p.pad_mult, (float)p.repetition_context,
                     p.repetition_penalty, 1.f};
  return B200_OK;
}

// Host: the text path of a session-sampling step on B rows: adjusted scores, then the sampler and the history
inline void text_rows_launch(const bf16* logits, float* scores, const float* noise, long long noise_ld, long long* out, int B, int card,
                             int use_sampling, float temp, int top_k, const RowSampling* rs, const TextHistory& th,
                             const uint8_t* exec_mask, cudaStream_t st) {
  B200_LAUNCH(text_adjust_kernel, B, SAMPLE_THREADS, 0, st, logits, scores, card, use_sampling, temp, rs, th);
  B200_LAUNCH(sample_text_kernel, B, SAMPLE_THREADS, 0, st, scores, noise, noise_ld, out, card, use_sampling, temp, top_k, rs, th,
              exec_mask);
}

}  // namespace lm
}  // namespace b200
