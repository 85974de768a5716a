// wgmma / TMA weight-streaming GEMM for the LM linears:  y[M][N] = epi(x[M][K] . w[N][K]^T)
//
// Skinny-M decode GEMMs are HBM-bound on the weights, so the kernel is organised around streaming
// each weight row exactly once ("swap-AB"): the 128-row weight tile is the MMA A operand (two m64
// halves, one per consumer warpgroup), the sessions are the MMA N dimension, and the fp32 accumulator
// lives in registers.  Both operands are K-major in HBM, which is the native TMA / wgmma SWIZZLE_128B
// layout, so no repacking of the reference's [out, in] weight layout is needed.
#pragma once

#include <cuda.h>

#include "tc_host.cuh"

namespace b200 {
namespace lm { struct RowSampling; }
namespace tc {

struct MapKey {
  const void* ptr; long long ld; int rows, cols, box_rows;
  bool operator<(const MapKey& o) const {
    if (ptr != o.ptr) return ptr < o.ptr;
    if (ld != o.ld) return ld < o.ld;
    if (rows != o.rows) return rows < o.rows;
    if (cols != o.cols) return cols < o.cols;
    return box_rows < o.box_rows;
  }
};

// activation tensor maps of the linears, encoded once per (buffer, shape, box)
struct TensorMapCache {
  std::map<MapKey, CUtensorMap> maps;
  void clear() { maps.clear(); }
};

// shared-memory attributes of the swap-AB / cluster kernels (linear_init) and of those and the non-swapped kernels
// (linear_prepare; call before capturing a graph).  Setting an attribute loads the kernel's code into device memory, which
// moves the buffers allocated after it: the LM calls linear_init when a batch starts streaming, before its depformer buffers.
int linear_init();
int linear_prepare();

// ---- the plan of one linear:  y[M][N] = epi(x[M][K] . w[N][K]^T) over packed weight tiles ---------------------------
//   GEMV (gemm_sk.cu): one to gemv_max_m rows, plain loads on the CUDA cores;
//   NS   (gemm_ns.cu): 33..256 rows, activations as the wgmma A operand, two weight tiles as B;
//   CK   (gemm_sk.cu): more than 32 rows over few row tiles, K cut over a cluster and reduced over DSMEM;
//   SK   (gemm_sk.cu): swap-AB stream-K, up to 128 rows per launch (64 gated).
enum LinearKernel { LK_GEMV = 1, LK_NS = 2, LK_CK = 3, LK_SK = 4 };

// Forces for tests and tools (the b200_op_* entry points); all zero = the LM's own choice
struct LinearForce {
  int kernel = 0;         // LK_NS: the non-swapped kernel at any M; LK_SK: never the non-swapped kernel
  int sk_grid = 0;        // stream-K with this many CTAs, tiles cut at every M
  int ck_cluster = 0;     // cluster split-K with this many CTAs per tile
  int ns_splits = 0;      // NS: K-splits over a cluster
  int ns_unit_tiles = 0;  // NS: weight tiles per CTA (1 = N 128, 2 = N 256)
  int stage_budget = 0;   // SK: bytes of pipeline stages per CTA (0 = 200 KB)
  int stream_only = 0;    // diagnostics: SK runs the copy pipeline without MMAs / stores
};

// One launch over rows [m0, m0 + rows); fields a kernel does not use are 0
struct LinearBlock {
  int kernel, m0, rows;
  int grid, cluster, smem, stages, stage_bytes;   // cluster: CK / NS K-splits
  int np, Mpad, kb_per;                           // np: activation box rows (SK / CK: the wgmma width, NS: 128)
  int S, kbps;                                    // GEMV splits and k-blocks per split
  int unit_tiles, ldw;                            // NS
  int Wc;                                         // CK
  int whole_rounds, sk_tile0, sk_items;           // SK schedule
};
constexpr int LINEAR_MAX_BLOCKS = 4;
struct LinearPlan {
  int M, N, K, epi, gate_rows, i8;
  int norm_folded;        // the RMSNorm asked for is folded into the GEMV's activation staging
  int stream_only;        // LinearForce::stream_only
  int n_blocks;
  LinearBlock blocks[LINEAR_MAX_BLOCKS];
};
// Pure host function (no CUDA call).  ld_aligned: the output and residual row strides are multiples of 8.
int plan_linear(int M, int N, int K, int epi, int gate_rows, bool i8, bool norm, bool ld_aligned, int sms, int gemv_max_m,
                const LinearForce& force, LinearPlan* plan);

struct LinearArgs {
  const __nv_bfloat16* x; long long ldx;     // bf16 activations (the residual stream when the norm is folded)
  const void* w;                             // packed tiles
  __nv_bfloat16* y; long long ldy;
  const __nv_bfloat16* res; long long ldr;
  float* ws; int* counters;                  // sk_workspace_bytes(M) and SK_MAX_TILES ints, zeroed once
  // int8 path (QLinear): row-wise absmax int8 activations [M][K] + their scales, and the weight-row scales [N]
  const void* xq; const float* sa; const float* sw;
  const __nv_bfloat16* norm_alpha;           // a folded RMSNorm's alpha (plan.norm_folded)
  int pdl;
};
int run_linear(TensorMapCache& maps, const LinearPlan& plan, const LinearArgs& a, cudaStream_t stream);
// the non-swapped kernel (gemm_ns.cu): shared-memory attributes, and the launch of one block of an NS plan
constexpr int NS_MAX_STAGES = 8, NS_MAX_CS = 8;
constexpr int NS_A_BYTES = 128 * 64 * 2;   // one activation box: 128 session rows x 64 k
int ns_init();
int ns_launch(const CUtensorMap& mx, const LinearPlan& plan, const LinearBlock& b, const LinearArgs& a, cudaStream_t stream);

int sk_gemv_max_m();
int sk_set_gemv_max_m(int max_m);      // rows up to which the GEMV path is taken (0..4); returns the previous value
bool sk_supported(int M, int N, int K, int epi);
size_t sk_packed_bytes(int N, int K, int epi, int gate_rows);
int sk_pack_weights(const __nv_bfloat16* w, void* out, int N, int K, int epi, int gate_rows, cudaStream_t stream);
size_t sk_workspace_bytes(int max_M);
// int8 (QLinear, utils/quantize.py:13-40): weights -> row-wise absmax int8 tiles + scales; activations -> int8 rows + scales
size_t sk_packed_bytes_i8(int N, int K, int epi, int gate_rows);
int sk_quant_pack_weights(const __nv_bfloat16* w, void* out_tiles, float* out_scales, int N, int K, int epi, int gate_rows,
                          cudaStream_t stream);
// weights that arrive already quantised (QLinear CB int8 [N][K] of a q8 checkpoint): tiled as they are
int sk_pack_weights_i8(const int8_t* q, void* out_tiles, int N, int K, int epi, int gate_rows, cudaStream_t stream);
int sk_quantize_rows(const __nv_bfloat16* x, long long ldx, void* xq, float* sa, int M, int K, cudaStream_t stream, int pdl = 0);
constexpr int SK_MAX_GRID = 304;     // 2 CTAs per SM at most
constexpr int SK_MAX_TILES = 1024;   // ints in the arrival-counter array

// ---- the depformer of one frame: its plan and the persistent kernel (dep_fused.cu) ---------------------------
struct Gemm {                                      // one GEMM phase of the persistent kernel
  const uint8_t* wt;                               // packed tiles [n_tile][kb][A][16 KB] (filled per sub-step and layer)
  int n_tiles, num_kb, kbps, S, A, N;              // S splits of kbps k-blocks; N = output columns per accumulator
};
enum DepPath { DEP_NONE = 0, DEP_CHAIN = 1, DEP_FUSED = 2 };
struct DepformerPlan {
  int path;                                        // DEP_NONE: dep_q = 0; DEP_CHAIN: one launch per kernel; DEP_FUSED
  Gemm g_in, g_out, g_lin_in, g_lin_out, g_head;   // DEP_FUSED: the five GEMM phases
  long long part_floats;                           // floats of each of the two split-partial buffers
  int stages, stage_bytes, smem, grid;
};
// Pure host function (no CUDA call).  mode: B200_DEPFORMER_AUTO / _CHAIN / _FUSED; B sessions (2B model rows under cfg).
int plan_depformer(int dep_q, int dd, int H, int F, int card, int B, bool cfg, bool i8, int sms, int gemv_max_m, int mode,
                   DepformerPlan* plan);

struct DepLayerW { const uint8_t *in_w, *out_w, *lin_in, *lin_out; };
struct DepParams {
  int B, Mpad, dd, H, F, card, text_card, dep_q, L, n_tables;
  int* err;                                                  // device error flags (lm::ERR_*)
  int stages; uint32_t stage_bytes;
  Gemm g_in, g_out, g_lin_in, g_lin_out, g_head;              // shapes (wt filled per (k, l) from the tables below)
  const DepLayerW* w;                                        // [dep_q][L] packed weight pointers (device)
  const uint8_t* const* heads;                               // [dep_q]
  const __nv_bfloat16* const* tables;                        // [dep_q] embedding tables ([0] = text)
  const __nv_bfloat16* const* n1; const __nv_bfloat16* const* n2;   // [L] RMSNorm alphas
  const __nv_bfloat16* din; long long din_ld;                // depformer_in_all output [B][n_sets*dd]
  const int* din_col;                                        // [dep_q] first column of sub-step k's block (its weight set * dd)
  const long long* text_token;                               // [B]
  __nv_bfloat16 *x, *xn, *ao, *hbuf;                         // [B][dd] x3, [B][F]
  __nv_bfloat16* const* kc; __nv_bfloat16* const* vc;        // [L] per-frame KV [B][H][dep_q][64]
  float *part0, *part1;                                      // split partials [S][B][Nmax]
  __nv_bfloat16* logits;                                     // [dep_q][B][card]
  long long* audio_tokens;                                   // [dep_q][B]
  const float* noise; long long noise_ld; int noise_off, ka; // Exp(1) noise, row stride, offset of sub-step 0, per-step width
  int use_sampling, top_k; float temp;
  const lm::RowSampling* rows;                               // [B] per-session settings (their temp / top_k), or null
  unsigned* bar;                                             // grid barrier counter (zero at launch)
  unsigned long long* trace;                                 // optional [DEP_TRACE_SLOTS]: %globaltimer of CTA 0 after every grid barrier
};
constexpr int DEP_TRACE_SLOTS = 512;
struct DepFused;
// p: every field but the plan's, its pointer tables (w .. n2, kc, vc) and din_col on the host; they are copied to the device
int dep_fused_create(const DepformerPlan& plan, const DepParams& p, DepFused** out);
void dep_fused_set_sampling(DepFused* d, int use_sampling, float temp, int top_k);
void dep_fused_destroy(DepFused* d);
int dep_fused_launch(DepFused* d, cudaStream_t stream);


}  // namespace tc
}  // namespace b200
