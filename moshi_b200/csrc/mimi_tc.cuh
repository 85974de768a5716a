// Mimi's contractions on the Hopper tensor cores: every StreamingConv1d / StreamingConvTranspose1d of the SEANet
// (conv.py:245-274, 340-362; seanet.py:90-93) and every nn.Linear of the two bottleneck transformers (transformer.py:752-777)
// is one launch of mimi_tc_kernel, a persistent TMA + wgmma (tf32) implicit GEMM with fp32-equivalent accuracy:
//
//     out[token][n] = epi( sum_{tap, ci} act[session][row0 + t * stride + tap * dil][ci] * w[n][tap][ci] )
//
//   * Activations are TOKEN-MAJOR: act[session][row][channel], channel fastest.  A layer's input lives in its own extended
//     buffer ext[b][carried rows | frame rows][Cin] (the producing layer's epilogue writes the consumer's activation, ELU
//     applied, straight behind the consumer's carried left context, so `cat(previous, x)` (conv.py:261) is an address).  A
//     tile of 128 GEMM rows = bb sessions x tt consecutive output steps, fetched per tap by ONE 3-D TMA box
//     (32 channels, tt rows with element stride = conv stride, bb sessions) into a K-major SWIZZLE_128B tile: the im2col
//     matrix never exists and strided convolutions cost no gather instructions.
//   * ConvTranspose1d with K = 2 S is the same kernel: out[b][t*S + r][co] = x[t] . W[:, co, r] + x[t-1] . W[:, co, S + r], i.e.
//     two taps over [x[t-1], x[t]], N = S * Cout ordered (r, co), whose row-major result IS the token-major output; the
//     overlap-add carry of conv.py:349-361 becomes one carried input row (x[-1] of the next frame).
//   * 3xTF32: a = a_hi + a_lo with a_hi = tf32(a) and a_lo = tf32(a - a_hi) (both round-to-nearest, written by the producing
//     epilogue), likewise for the weights at load; the product is a_hi*w_hi + a_hi*w_lo + a_lo*w_hi with fp32 accumulation
//     in registers (dropped terms <= 2^-22 relative).  The RVQ indices downstream stay exact up to the margin the parity tests
//     define (tests/util.py).
//   * Warp roles (288 threads): warp 8 = TMA producer (A hi + A lo boxes, one contiguous bulk copy of the pre-tiled weight
//     pair per k-block), warps 0-7 = two consumer warpgroups, each owning 64 GEMM rows (tokens) of the tile: wgmma into
//     register accumulators, then the epilogue straight from the fragments (bias, residual, ELU / GELU / layer-scale, hi/lo
//     split).  Persistent grid; the producer runs ahead through the stage ring while the consumers finish a tile.
//     Deep-and-skinny layers are cut along K into fp32 partials reduced in split order by mimi_tc_reduce_kernel
//     (deterministic).
#pragma once

#include <cuda.h>

#include "common.cuh"

namespace b200 {
namespace mtc {

constexpr int TC_ROWS = 128;            // GEMM rows (tokens) per tile: 64 per consumer warpgroup
constexpr int TC_KB = 32;               // fp32 elements per k-block row: 128 bytes = one SWIZZLE_128B row
constexpr int TC_MAX_NT = 128;          // output features per tile = wgmma N (<= 128: 64 KB per stage, 3 stages)
constexpr int TC_THREADS = 288;         // warps 0-7: two consumer warpgroups (MMA + epilogue), warp 8: producer
constexpr int TC_PRODUCER_WARP = 8;
constexpr int TC_CONSUMERS = 256;
constexpr int TC_MAX_STAGES = 6;

enum { TC_EPI_CONV = 0, TC_EPI_GELU = 1, TC_EPI_RES_SCALE = 2 };
enum { TC_ACT_NONE = 0, TC_ACT_SPLIT = 1, TC_ACT_FULL = 2 };      // how the consumer wants its input: hi/lo pair or plain fp32

struct TcParams {
  // ---- geometry of the A operand (tensor maps are kernel arguments)
  int tt, bb;                 // tile = bb sessions x tt steps, tt * bb == 128
  int T;                      // output steps per session (tt divides T, or T < tt == 128 for the flat linear case)
  int n_sessions;             // B (rows beyond it are zero-filled by TMA and masked in the epilogue)
  int n_taps, dil, stride, row0, Cin;
  // ---- B operand: pre-tiled weights [n_tile][kb][hi | lo][NT rows][32] (SWIZZLE_128B), kb = tap * (Cin / 32) + ci_block
  const uint8_t* wt; int NT, n_tiles_n, num_kb, N;
  // ---- schedule
  int m_tiles, ksplit, kb_per_split;
  float* ws;                  // split-K partials [split][rows_total][N] (rows_total = m_tiles * 128)
  // ---- epilogue
  int epi;
  const float* bias; int bias_mod;                 // bias[n % bias_mod] (conv: bias_mod = N; convtr: Cout)
  float* y; long long y_sb, y_row;                 // raw output: y[b * y_sb + t * y_row + n] (null = not stored)
  const float* res; long long r_sb, r_row;         // residual source (conv: same indexing; lin: res[token * r_row + n])
  const float* scale;                              // lin RES_SCALE: per-feature layer scale
  int act_mode, act_elu;
  float *a_hi, *a_lo; long long a_sb, a_row;       // activated copy for the consumer: a[b * a_sb + t * a_row + n]
  uint32_t stage_bytes; int stages;
};

// y = hi + lo with hi = tf32(y) and lo = tf32(y - hi), both round-to-nearest (cvt.rna): |y - hi - lo| <= 2^-23 |y|
__device__ __forceinline__ void split_tf32(float v, float& hi, float& lo) {
  uint32_t h, l;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(h) : "f"(v));
  hi = __uint_as_float(h);
  const float r = v - hi;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(l) : "f"(r));
  lo = __uint_as_float(l);
}

// ---- host side ---------------------------------------------------------------------------------------------------------
enum { TC_CONV = 0, TC_CONVTR = 1, TC_LINEAR = 2, TC_LINEAR_ROWS = 3 };   // TC_LINEAR_ROWS: M flat rows as one session
constexpr size_t TC_SPLIT_BYTES = (size_t)64 << 20;   // split-K partials budget of one layer

// what the weights fix: N output features over n_taps * Cin inputs and their tiling NT / n_tiles_n / num_kb
struct TcShape {
  int kind = TC_CONV;
  int Cin = 0, N = 0, n_taps = 1, dil = 1, stride = 1;
  int bias_mod = 0;           // bias[n % bias_mod]
  int NT = 0, n_tiles_n = 0, num_kb = 0;
};

// what one launch runs for n_sessions sessions of T GEMM rows each (plan_tc)
struct TcSchedule {
  int tt = 0, bb = 0, T = 0, n_sessions = 0;
  int m_tiles = 0, ksplit = 0, kb_per_split = 0, stages = 0;
  uint32_t stage_bytes = 0;
  int grid = 0; size_t smem = 0;
};

// a layer bound to its weights, input and schedule: what tc_launch launches
struct TcLayer {
  TcShape s;
  uint8_t* wt = nullptr;      // packed hi/lo tiles
  const float* bias = nullptr;
  CUtensorMap map_hi, map_lo;
  TcParams p;
  int grid = 0; size_t smem = 0;
};

// bias_mod 0: N
TcShape tc_shape(int kind, int N, int Cin, int n_taps, int dil = 1, int stride = 1, int bias_mod = 0);
// The schedule of a layer on a device of `sms` multiprocessors whose split-K partials fit ws_bytes; no CUDA call.  Tile:
// bb = 128 / tt sessions of tt steps, tt the largest power of two (<= 128) that divides T and keeps the TMA box (tt * stride
// rows) within 256; TC_LINEAR_ROWS: one session of T rows on 128 x 1 tiles, the last one partial.
int plan_tc(const TcShape& s, int n_sessions, int T, int sms, size_t ws_bytes, TcSchedule* out);
size_t tc_packed_bytes(const TcShape& s);
// w: fp32 [N][n_taps * Cin] (k = tap * Cin + ci) -> tiles
int tc_pack_weights(const float* w_dev, void* out_dev, const TcShape& s, cudaStream_t st);
int tc_init();
// Binds L (shape, weights and bias set) to schedule q: the launch parameters are `epi` (epilogue fields) completed from shape,
// schedule and the split-K workspace ws; the A maps cover in_hi / in_lo, token-major [q.n_sessions][rows_per_session][Cin].
int tc_bind(TcLayer& L, const TcSchedule& q, const TcParams& epi, const float* in_hi, const float* in_lo, long long rows_per_session,
            float* ws);
int tc_launch(const TcLayer& L, cudaStream_t st);

}  // namespace mtc
}  // namespace b200
