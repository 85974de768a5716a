// wgmma / TMA weight-streaming GEMM for the LM linears:  y[M][N] = epi(x[M][K] . w[N][K]^T)
//
// Skinny-M decode GEMMs are HBM-bound on the weights, so the kernel is organised around streaming
// each weight row exactly once ("swap-AB"): the 128-row weight tile is the MMA A operand (two m64
// halves, one per consumer warpgroup), the sessions are the MMA N dimension, and the fp32 accumulator
// lives in registers.  Both operands are K-major in HBM, which is the native TMA / wgmma SWIZZLE_128B
// layout, so no repacking of the reference's [out, in] weight layout is needed.
#pragma once

#include <cuda.h>

#include "common.cuh"

namespace b200 {
namespace tc {

struct PlanKey {
  const void* ptr; long long ld; int rows, cols, box_rows;
  bool operator<(const PlanKey& o) const {
    if (ptr != o.ptr) return ptr < o.ptr;
    if (ld != o.ld) return ld < o.ld;
    if (rows != o.rows) return rows < o.rows;
    if (cols != o.cols) return cols < o.cols;
    return box_rows < o.box_rows;
  }
};

struct GemmPlanCache {
  std::map<PlanKey, CUtensorMap> maps;
  void clear() { maps.clear(); }
};

// resolves cuTensorMapEncodeTiled and sets the kernels' shared-memory attributes (call before capturing a graph)
int prepare_plans(GemmPlanCache& cache);

// ---- stream-K kernel over pre-tiled weights (gemm_sk.cu) --------------------------------------
struct SkTuning {
  int grid = 0;          // CTAs (0 = one per SM)
  int smem_budget = 0;   // bytes of pipeline stages per CTA (0 = 200 KB)
  int stream_only = 0;   // diagnostics: run the copy pipeline without MMAs / stores
  int no_split = 0;      // never cut a tile across CTAs (whole tiles only)
  int force_split = 0;   // tests: cut tiles even where the default policy keeps them whole
  int no_cluster = 0;    // never use the cluster split-K kernel
  int cluster = 0;       // force a cluster size (tests)
  // int8 path (QLinear): row-wise absmax int8 activations [M][K] + their scales, and the weight-row scales [N]
  const void* xq = nullptr; const float* sa = nullptr; const float* sw = nullptr;
  int pdl = 0;           // launch with programmatic stream serialization (the kernel waits on its own)
  int ns = 0;            // 33..256 sessions: 0 = the non-swapped kernel (gemm_ns.cu) unless B200_GEMM_NS=0, -1 = never, 1 = always (tests)
  // GEMV path only (M <= sk_gemv_max_m()): x is the residual stream and the linear's input is rmsnorm(x, norm_alpha)
  const __nv_bfloat16* norm_alpha = nullptr;
};
int sk_num_sms();
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
int sk_linear(GemmPlanCache& cache, const __nv_bfloat16* x, long long ldx, const void* w_tiles, __nv_bfloat16* y,
              long long ldy, const __nv_bfloat16* res, long long ldr, int M, int N, int K, int epi, int gate_rows,
              float* ws, int* counters, const SkTuning& tune, cudaStream_t stream);

// ---- non-swapped kernel for 33..256 sessions (gemm_ns.cu): A = activations, B = two weight tiles (N = 256) ------------
bool ns_supported(int M, int N, int K, int epi);
int ns_prepare();
// cluster: K-splits (0 = the default plan for the shape); same packed weights and epilogues as sk_linear
// unit_tiles: weight tiles per CTA as the B operand (2 = N 256; 1 = N 128: twice the units for few-tile shapes; 0 = the LM's choice)
int ns_linear(GemmPlanCache& cache, const __nv_bfloat16* x, long long ldx, const void* w_tiles, __nv_bfloat16* y, long long ldy,
              const __nv_bfloat16* res, long long ldr, int M, int N, int K, int epi, int gate_rows, int cluster, int pdl,
              cudaStream_t stream, int unit_tiles = 0);

// ---- the depformer of one frame as one persistent kernel (dep_fused.cu) ---------------------------
struct DepFusedConfig {
  int B, dd, H, F, card, text_card, dep_q, L;
  int* err;                                        // device error flags (lm::ERR_*), may be null
  const void* const* in_w; const void* const* out_w; const void* const* lin_in; const void* const* lin_out;   // [dep_q*L] packed tiles
  const void* const* heads;        // [dep_q] packed tiles
  const void* const* tables;       // [dep_q] embedding tables (bf16 [V][dd]); [0] = text
  const void* const* n1; const void* const* n2;   // [L] RMSNorm alphas (bf16 [dd])
  void* const* kc; void* const* vc;               // [L] KV [B][H][dep_q][64] bf16
  const void* din; long long din_ld;              // depformer_in_all output, bf16 [B][dep_q*dd]
  const long long* text_token;
  void *x, *xn, *ao, *hbuf;                       // bf16 [B][dd] x3, [B][F]
  float *part0, *part1;                           // dep_fused_partial_floats() floats each
  void* logits; long long* audio_tokens;          // bf16 [dep_q][B][card], i64 [dep_q][B]
  const float* noise; long long noise_ld; int noise_off, ka;
  int use_sampling, top_k; float temp;
  unsigned* bar;
  unsigned long long* trace;                       // optional [DEP_TRACE_SLOTS] barrier timestamps of CTA 0 (diagnostics), may be null
};
constexpr int DEP_TRACE_SLOTS = 512;
struct DepFused;
size_t dep_fused_partial_floats(const DepFusedConfig& c);
int dep_fused_create(const DepFusedConfig& c, DepFused** out);
void dep_fused_set_sampling(DepFused* d, int use_sampling, float temp, int top_k);
void dep_fused_destroy(DepFused* d);
int dep_fused_launch(DepFused* d, cudaStream_t stream);


}  // namespace tc
}  // namespace b200
