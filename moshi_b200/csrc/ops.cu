// Kernel-level C entry points used by the parity tests (same kernels the handles launch).
#include "gemm_sk.cuh"
#include "lm_kernels.cuh"
#include "mimi_kernels.cuh"
#include "mimi_tc.cuh"
#include "mimi_tm_kernels.cuh"

using namespace b200;

extern "C" {

// split-K workspace + arrival counters of the kernel-level entry points (a handle owns its own); separate sets for the bf16 and
// the int8 kernels, like the handles keep them
static int sk_scratch(float** ws, int** counters, int which = 0) {
  static float* g_ws[2] = {nullptr, nullptr};
  static int* g_counters[2] = {nullptr, nullptr};
  if (!g_ws[which]) {
    B200_CUDA(cudaMalloc(&g_ws[which], tc::sk_workspace_bytes(256)));
    B200_CUDA(cudaMalloc(&g_counters[which], tc::SK_MAX_TILES * sizeof(int)));
    B200_CUDA(cudaMemset(g_counters[which], 0, tc::SK_MAX_TILES * sizeof(int)));
  }
  *ws = g_ws[which]; *counters = g_counters[which];
  return B200_OK;
}

// split-KV partials + merge counters of the attention entry points, grown on demand; separate sets for the bf16 and the 8-bit rings
static int attn_scratch(int B, int H, int nsplit, float** part, int** counters, int which) {
  static float* g_part[2] = {nullptr, nullptr};
  static int* g_counters[2] = {nullptr, nullptr};
  static size_t part_n[2] = {0, 0}, cnt_n[2] = {0, 0};
  const size_t need = (size_t)B * H * nsplit * (lm::ATT_D + 2);
  if (need > part_n[which]) {
    if (g_part[which]) cudaFree(g_part[which]);
    B200_CUDA(cudaMalloc(&g_part[which], need * sizeof(float)));
    part_n[which] = need;
  }
  if ((size_t)B * H > cnt_n[which]) {
    if (g_counters[which]) cudaFree(g_counters[which]);
    B200_CUDA(cudaMalloc(&g_counters[which], (size_t)B * H * sizeof(int)));
    B200_CUDA(cudaMemset(g_counters[which], 0, (size_t)B * H * sizeof(int)));
    cnt_n[which] = (size_t)B * H;
  }
  *part = g_part[which]; *counters = g_counters[which];
  return B200_OK;
}

// The LM's linear as the kernel-level entry points run it: rows of x, y and res are contiguous (ldx = K, ldy = ldr = output
// columns); `which` picks the bf16 or the int8 scratch and tensor-map cache
static int op_linear(const void* x, const void* w, void* y, const void* res, int M, int N, int K, int epi, int gate_rows,
                     const tc::LinearForce& force, const void* xq, const float* sa, const float* sw, const void* norm_alpha, int which,
                     cudaStream_t st) {
  static tc::TensorMapCache caches[2];
  float* ws = nullptr; int* counters = nullptr;
  B200_TRY(sk_scratch(&ws, &counters, which));
  const int out_cols = epi == 2 ? gate_rows : N;
  tc::LinearPlan plan;
  B200_TRY(tc::plan_linear(M, N, K, epi, gate_rows, xq != nullptr, norm_alpha != nullptr, out_cols % 8 == 0, num_sms(), tc::sk_gemv_max_m(),
                           force, &plan));
  const tc::LinearArgs a{static_cast<const __nv_bfloat16*>(x), K, w, static_cast<__nv_bfloat16*>(y), out_cols,
                         static_cast<const __nv_bfloat16*>(res), out_cols, ws, counters, xq, sa, sw,
                         static_cast<const __nv_bfloat16*>(norm_alpha), 0};
  return tc::run_linear(caches[which], plan, a, st);
}

int b200_op_linear_bf16(const void* x_dev, const void* w_dev, void* y_dev, int M, int N, int K, void* stream) {
  if (!x_dev || !w_dev || !y_dev || M < 1 || N < 1 || K < 8 || K % 8) B200_FAIL(B200_ERR_SHAPE, "op_linear_bf16: bad shape");
  if (!tc::sk_supported(M, N, K, 0)) B200_FAIL(B200_ERR_SHAPE, "op_linear_bf16: unsupported shape");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  void* tiles = nullptr;
  B200_CUDA(cudaMalloc(&tiles, tc::sk_packed_bytes(N, K, 0, 0)));
  int rc = tc::sk_pack_weights(static_cast<const __nv_bfloat16*>(w_dev), tiles, N, K, 0, 0, st);
  if (rc == B200_OK) rc = op_linear(x_dev, tiles, y_dev, nullptr, M, N, K, 0, 0, tc::LinearForce(), nullptr, nullptr, nullptr, nullptr, 0, st);
  cudaStreamSynchronize(st);
  cudaFree(tiles);
  return rc;
}

int64_t b200_op_packed_bytes(int N, int K, int epi, int gate_rows) { return (int64_t)tc::sk_packed_bytes(N, K, epi, gate_rows); }

int b200_op_pack_tiles(const void* w_dev, void* out_dev, int N, int K, int epi, int gate_rows, void* stream) {
  if (!w_dev || !out_dev) B200_FAIL(B200_ERR_INVALID, "op_pack_tiles: null pointer");
  return tc::sk_pack_weights(static_cast<const __nv_bfloat16*>(w_dev), out_dev, N, K, epi, gate_rows,
                             static_cast<cudaStream_t>(stream));
}

int b200_op_linear_sk(const void* x_dev, const void* w_tiles_dev, void* y_dev, const void* res_dev, int M, int N, int K,
                      int epi, int gate_rows, int grid, int smem_budget, int stream_only, void* stream) {
  if (!x_dev || !w_tiles_dev || !y_dev) B200_FAIL(B200_ERR_INVALID, "op_linear_sk: null pointer");
  if (!tc::sk_supported(M, N, K, epi)) B200_FAIL(B200_ERR_SHAPE, "op_linear_sk: unsupported shape");
  tc::LinearForce f;
  // grid > 0: stream-K with that many CTAs (tiles cut at every M); grid < 0: cluster split-K with |grid| CTAs per tile; 0: the LM's own choice
  f.sk_grid = grid > 0 ? grid : 0; f.ck_cluster = grid < 0 ? -grid : 0; f.stream_only = stream_only;
  // smem_budget > 0: the stage ring's bytes; -1: never the non-swapped kernel (the swap-AB comparison row of tools/kbench.py)
  f.stage_budget = smem_budget > 0 ? smem_budget : 0;
  f.kernel = smem_budget == -1 ? tc::LK_SK : 0;
  return op_linear(x_dev, w_tiles_dev, y_dev, res_dev, M, N, K, epi, gate_rows, f, nullptr, nullptr, nullptr, nullptr, 0,
                   static_cast<cudaStream_t>(stream));
}

// the non-swapped kernel (33..256 sessions in the LM) at any M <= 256; cluster = K-splits (0 = the LM's own choice)
int b200_op_linear_ns(const void* x_dev, const void* w_tiles_dev, void* y_dev, const void* res_dev, int M, int N, int K, int epi,
                      int gate_rows, int cluster, void* stream) {
  if (!x_dev || !w_tiles_dev || !y_dev) B200_FAIL(B200_ERR_INVALID, "op_linear_ns: null pointer");
  if (!tc::sk_supported(M, N, K, epi)) B200_FAIL(B200_ERR_SHAPE, "op_linear_ns: unsupported shape");
  tc::LinearForce f;
  f.kernel = tc::LK_NS;
  // cluster >= 100: single-tile units (N = 128 per instruction) with cluster - 100 K-splits
  f.ns_unit_tiles = cluster >= 100 ? 1 : (cluster > 0 ? 2 : 0);
  f.ns_splits = cluster >= 100 ? cluster - 100 : cluster;
  return op_linear(x_dev, w_tiles_dev, y_dev, res_dev, M, N, K, epi, gate_rows, f, nullptr, nullptr, nullptr, nullptr, 0,
                   static_cast<cudaStream_t>(stream));
}

// y = epi(rmsnorm(x, alpha) . W^T) with the norm folded into the GEMV's activation staging (norm_linear at one or two
// sessions); every other path refuses a norm input with B200_ERR_STATE
int b200_op_linear_sk_norm(const void* x_dev, const void* alpha_dev, const void* w_tiles_dev, void* y_dev, const void* res_dev, int M,
                           int N, int K, int epi, int gate_rows, void* stream) {
  if (!x_dev || !alpha_dev || !w_tiles_dev || !y_dev) B200_FAIL(B200_ERR_INVALID, "op_linear_sk_norm: null pointer");
  if (!tc::sk_supported(M, N, K, epi)) B200_FAIL(B200_ERR_SHAPE, "op_linear_sk_norm: unsupported shape");
  return op_linear(x_dev, w_tiles_dev, y_dev, res_dev, M, N, K, epi, gate_rows, tc::LinearForce(), nullptr, nullptr, nullptr, alpha_dev,
                   0, static_cast<cudaStream_t>(stream));
}

int b200_op_set_gemv_max_rows(int max_rows) { return tc::sk_set_gemv_max_m(max_rows); }

int b200_op_linear_plan(int M, int N, int K, int epi, int gate_rows, int int8, int norm, int sms, int gemv_max_rows, int64_t* out,
                        int capacity) {
  if (!out || capacity < 2) B200_FAIL(B200_ERR_INVALID, "op_linear_plan: no room for the plan");
  tc::LinearPlan plan;
  B200_TRY(tc::plan_linear(M, N, K, epi, gate_rows, int8 != 0, norm != 0, (epi == 2 ? gate_rows : N) % 8 == 0, sms, gemv_max_rows,
                           tc::LinearForce(), &plan));
  constexpr int F = 19;
  if (capacity < 2 + F * plan.n_blocks) B200_FAIL(B200_ERR_INVALID, "op_linear_plan: %d launches need %d slots", plan.n_blocks, 2 + F * plan.n_blocks);
  out[0] = plan.n_blocks; out[1] = plan.norm_folded;
  for (int i = 0; i < plan.n_blocks; ++i) {
    const tc::LinearBlock& b = plan.blocks[i];
    const int v[F] = {b.kernel, b.m0, b.rows, b.grid, b.cluster, b.smem, b.stages, b.stage_bytes, b.np, b.Mpad, b.kb_per, b.S, b.kbps,
                      b.unit_tiles, b.ldw, b.Wc, b.whole_rounds, b.sk_tile0, b.sk_items};
    for (int j = 0; j < F; ++j) out[2 + F * i + j] = v[j];
  }
  return B200_OK;
}

int b200_op_depformer_plan(int dep_q, int depformer_dim, int depformer_num_heads, int depformer_ffn_hidden, int card, int batch,
                           int cfg, int int8, int mode, int sms, int gemv_max_rows, int64_t* out, int capacity) {
  constexpr int F = 6 + 5 * 6;
  if (!out || capacity < F) B200_FAIL(B200_ERR_INVALID, "op_depformer_plan: %d slots, the plan needs %d", capacity, F);
  tc::DepformerPlan P;
  B200_TRY(tc::plan_depformer(dep_q, depformer_dim, depformer_num_heads, depformer_ffn_hidden, card, batch, cfg != 0, int8 != 0, sms,
                              gemv_max_rows, mode, &P));
  const long long v[6] = {P.path, P.part_floats, P.stages, P.stage_bytes, P.smem, P.grid};
  int i = 0;
  for (long long x : v) out[i++] = x;
  for (const tc::Gemm& g : {P.g_in, P.g_out, P.g_lin_in, P.g_lin_out, P.g_head})
    for (int x : {g.n_tiles, g.num_kb, g.kbps, g.S, g.A, g.N}) out[i++] = x;
  return B200_OK;
}

// rmsnorm_kernel as the LM launches it (lm.cu norm_linear and the output norm): one 256-thread CTA per row, eps 1e-8
int b200_op_rmsnorm(const void* x_dev, const void* alpha_dev, void* y_dev, int M, int dim, void* stream) {
  using namespace b200::lm;
  if (!x_dev || !alpha_dev || !y_dev) B200_FAIL(B200_ERR_INVALID, "op_rmsnorm: null pointer");
  if (M < 1 || dim < 2 || dim % 2) B200_FAIL(B200_ERR_SHAPE, "op_rmsnorm: bad shape M=%d dim=%d", M, dim);
  B200_LAUNCH(rmsnorm_kernel, M, 256, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(x_dev),
              static_cast<const bf16*>(alpha_dev), static_cast<bf16*>(y_dev), dim, 1e-8f);
  return check_launch("op_rmsnorm");
}

int b200_op_layernorm(const void* x_dev, const void* w_dev, const void* b_dev, void* y_dev, int M, int dim, void* stream) {
  using namespace b200::lm;
  if (!x_dev || !w_dev || !b_dev || !y_dev) B200_FAIL(B200_ERR_INVALID, "op_layernorm: null pointer");
  if (M < 1 || dim < 2 || dim % 2) B200_FAIL(B200_ERR_SHAPE, "op_layernorm: bad shape M=%d dim=%d", M, dim);
  B200_LAUNCH(layernorm_kernel, M, 256, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(x_dev),
              static_cast<const bf16*>(w_dev), static_cast<const bf16*>(b_dev), static_cast<bf16*>(y_dev), dim, 1e-5f);
  return check_launch("op_layernorm");
}

int b200_op_cross_attn_step(const void* q_dev, const void* k_dev, const void* v_dev, void* out_dev, int B, int H, int T, int nsplit,
                            void* stream) {
  using namespace b200::lm;
  if (!q_dev || !k_dev || !v_dev || !out_dev) B200_FAIL(B200_ERR_INVALID, "op_cross_attn_step: null pointer");
  if (B < 1 || H < 1 || T < 1) B200_FAIL(B200_ERR_SHAPE, "op_cross_attn_step: bad shape");
  if (nsplit <= 0) nsplit = attn_pick_splits(B, H, T);
  float* part = nullptr;
  int* counters = nullptr;
  B200_TRY(attn_scratch(B, H, nsplit, &part, &counters, 0));
  cross_attn_launch(static_cast<const bf16*>(q_dev), (long long)H * ATT_D, static_cast<const bf16*>(k_dev), static_cast<const bf16*>(v_dev),
                    static_cast<bf16*>(out_dev), part, counters, B, H, T, nsplit, static_cast<cudaStream_t>(stream));
  return check_launch("op_cross_attn_step");
}

int64_t b200_op_packed_bytes_i8(int N, int K, int epi, int gate_rows) { return (int64_t)tc::sk_packed_bytes_i8(N, K, epi, gate_rows); }

int b200_op_quant_pack_tiles(const void* w_dev, void* tiles_dev, float* scales_dev, int N, int K, int epi, int gate_rows,
                             void* stream) {
  if (!w_dev || !tiles_dev || !scales_dev) B200_FAIL(B200_ERR_INVALID, "op_quant_pack_tiles: null pointer");
  return tc::sk_quant_pack_weights(static_cast<const __nv_bfloat16*>(w_dev), tiles_dev, scales_dev, N, K, epi, gate_rows,
                                   static_cast<cudaStream_t>(stream));
}

int b200_op_quantize_rows(const void* x_dev, void* xq_dev, float* sa_dev, int M, int K, void* stream) {
  if (!x_dev || !xq_dev || !sa_dev) B200_FAIL(B200_ERR_INVALID, "op_quantize_rows: null pointer");
  return tc::sk_quantize_rows(static_cast<const __nv_bfloat16*>(x_dev), K, xq_dev, sa_dev, M, K, static_cast<cudaStream_t>(stream));
}

int b200_op_linear_i8(const void* xq_dev, const float* sa_dev, const void* w_tiles_dev, const float* sw_dev, void* y_dev,
                      const void* res_dev, int M, int N, int K, int epi, int gate_rows, void* stream) {
  if (!xq_dev || !sa_dev || !w_tiles_dev || !sw_dev || !y_dev) B200_FAIL(B200_ERR_INVALID, "op_linear_i8: null pointer");
  if (!tc::sk_supported(M, N, K, epi)) B200_FAIL(B200_ERR_SHAPE, "op_linear_i8: unsupported shape");
  // int32 partials of cut tiles in their own scratch
  return op_linear(nullptr, w_tiles_dev, y_dev, res_dev, M, N, K, epi, gate_rows, tc::LinearForce(), xq_dev, sa_dev, sw_dev, nullptr, 1,
                   static_cast<cudaStream_t>(stream));
}

int b200_op_attn_step(const void* qkv_dev, void* k_dev, void* v_dev, void* out_dev, const int64_t* pos_dev,
                      const uint8_t* exec_mask_dev, int B, int H, int cap, int nsplit, float max_period, void* stream) {
  using namespace b200::lm;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (B < 1 || H < 1 || cap < 1) B200_FAIL(B200_ERR_SHAPE, "op_attn_step: bad shape");
  if (nsplit <= 0) nsplit = attn_pick_splits(B, H, cap);
  float* part = nullptr;
  int* counters = nullptr;
  B200_TRY(attn_scratch(B, H, nsplit, &part, &counters, 0));
  attn_step_launch(static_cast<const bf16*>(qkv_dev), KvRings{k_dev, v_dev}, static_cast<bf16*>(out_dev), part, counters,
                   reinterpret_cast<const long long*>(pos_dev), exec_mask_dev, B, H, cap, nsplit, max_period, 0, st);
  return check_launch("op_attn_step");
}

int b200_op_attn_step_paged(const void* qkv_dev, void* k_pool_dev, void* v_pool_dev, const int32_t* page_table_dev, void* out_dev,
                            const int64_t* pos_dev, const uint8_t* exec_mask_dev, int B, int H, int cap, int page_slots, int nsplit,
                            float max_period, void* stream) {
  using namespace b200::lm;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (B < 1 || H < 1 || cap < 1) B200_FAIL(B200_ERR_SHAPE, "op_attn_step_paged: bad shape");
  if (page_slots < 4 || page_slots > 256 || (page_slots & (page_slots - 1)))
    B200_FAIL(B200_ERR_INVALID, "op_attn_step_paged: page_slots %d (a power of two in [4, 256])", page_slots);
  if (!page_table_dev) B200_FAIL(B200_ERR_INVALID, "op_attn_step_paged: null page table");
  if (nsplit <= 0) nsplit = attn_pick_splits(B, H, cap);
  float* part = nullptr;
  int* counters = nullptr;
  B200_TRY(attn_scratch(B, H, nsplit, &part, &counters, 0));
  const KvRings r{k_pool_dev, v_pool_dev, nullptr, nullptr, page_table_dev, (cap + page_slots - 1) / page_slots, __builtin_ctz(page_slots)};
  attn_step_launch(static_cast<const bf16*>(qkv_dev), r, static_cast<bf16*>(out_dev), part, counters,
                   reinterpret_cast<const long long*>(pos_dev), exec_mask_dev, B, H, cap, nsplit, max_period, 0, st);
  return check_launch("op_attn_step_paged");
}

int b200_op_attn_step_q8(const void* qkv_dev, void* k8_dev, void* v8_dev, float* ks_dev, float* vs_dev, void* out_dev,
                         const int64_t* pos_dev, const uint8_t* exec_mask_dev, int B, int H, int cap, int nsplit, float max_period,
                         int kv_dtype, void* stream) {
  using namespace b200::lm;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (B < 1 || H < 1 || cap < 1) B200_FAIL(B200_ERR_SHAPE, "op_attn_step_q8: bad shape");
  if (kv_dtype != B200_KV_FP8_E4M3 && kv_dtype != B200_KV_INT8) B200_FAIL(B200_ERR_INVALID, "op_attn_step_q8: kv_dtype %d", kv_dtype);
  if (nsplit <= 0) nsplit = attn_pick_splits(B, H, cap);
  float* part = nullptr;
  int* counters = nullptr;
  B200_TRY(attn_scratch(B, H, nsplit, &part, &counters, 1));
  attn_step_launch(static_cast<const bf16*>(qkv_dev), KvRings{k8_dev, v8_dev, ks_dev, vs_dev}, static_cast<bf16*>(out_dev), part, counters,
                   reinterpret_cast<const long long*>(pos_dev), exec_mask_dev, B, H, cap, nsplit, max_period, kv_dtype, st);
  return check_launch("op_attn_step_q8");
}

// dep_attn_step_kernel with the LM's launch shape (lm.cu, depformer layers): one warp per (b, h), 128 threads per CTA
int b200_op_dep_attn_step(const void* qkv_dev, void* k_dev, void* v_dev, void* out_dev, int B, int H, int cap, int step, void* stream) {
  using namespace b200::lm;
  if (!qkv_dev || !k_dev || !v_dev || !out_dev) B200_FAIL(B200_ERR_INVALID, "op_dep_attn_step: null pointer");
  if (B < 1 || H < 1 || cap < 1 || cap > DEP_MAX_Q || step < 0 || step >= cap)
    B200_FAIL(B200_ERR_SHAPE, "op_dep_attn_step: B=%d H=%d cap=%d step=%d (cap <= %d, step < cap)", B, H, cap, step, DEP_MAX_Q);
  B200_LAUNCH(dep_attn_step_kernel, ceil_div(B * H * 32, 128), 128, 0, static_cast<cudaStream_t>(stream),
              static_cast<const bf16*>(qkv_dev), static_cast<bf16*>(k_dev), static_cast<bf16*>(v_dev), static_cast<bf16*>(out_dev), B, H, cap,
              step);
  return check_launch("op_dep_attn_step");
}

// ring_attn_step_kernel<64> with the Mimi handle's launch shape (mimi.cu run_transformer): one 128-thread CTA per (b, h)
int b200_op_mimi_ring_attn(const float* qkv_dev, float* k_dev, float* v_dev, float* out_hi_dev, float* out_lo_dev, const int64_t* offset_dev,
                           const uint8_t* exec_mask_dev, int B, int H, int T, int cap, int context, float max_period, void* stream) {
  using namespace b200::mimi;
  constexpr int D = 64;
  if (!qkv_dev || !k_dev || !v_dev || !out_hi_dev || !out_lo_dev || !offset_dev || !exec_mask_dev)
    B200_FAIL(B200_ERR_INVALID, "op_mimi_ring_attn: null pointer");
  // one warp per query does the softmax and the kernel has 4 warps; the scores of all T queries over the ring sit in shared memory
  const size_t smem = (size_t)(T * D + T * cap) * sizeof(float);
  if (B < 1 || H < 1 || T < 1 || T > 4 || cap < 1 || context < 1 || smem > 48 * 1024)
    B200_FAIL(B200_ERR_SHAPE, "op_mimi_ring_attn: B=%d H=%d T=%d cap=%d context=%d (T <= 4, %zu bytes of shared memory <= 48 KB)", B, H,
              T, cap, context, smem);
  const float nl = -logf(max_period) * 2.f / (float)D;
  B200_LAUNCH((ring_attn_step_kernel<D>), B * H, 128, smem, static_cast<cudaStream_t>(stream), qkv_dev, k_dev, v_dev, out_hi_dev,
              out_lo_dev, reinterpret_cast<const long long*>(offset_dev), exec_mask_dev, T, H, cap, context, nl);
  return check_launch("op_mimi_ring_attn");
}

}  // extern "C"

// ---- Mimi's conv kernels on the reference's [B, C, T] layout (test scaffolding: the handle keeps everything token-major) ----
namespace {

// ext[b][j][ci] (hi / lo) = cat(previous, act(x))[b][ci][j]  for j < P + T
__global__ void tm_pack_in_kernel(const float* __restrict__ x, const float* __restrict__ prev, float* __restrict__ hi, float* __restrict__ lo,
                                  int B, int Cin, int T, int P, int elu) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long E = P + T;
  if (i >= (long long)B * E * Cin) return;
  const int ci = (int)(i % Cin);
  const long long r = i / Cin;
  const int j = (int)(r % E), b = (int)(r / E);
  float v;
  if (j < P) v = prev ? prev[((long long)b * Cin + ci) * P + j] : 0.f;
  else { v = x[((long long)b * Cin + ci) * T + (j - P)]; v = elu ? elu1(v) : v; }
  float h, l;
  b200::mtc::split_tf32(v, h, l);
  hi[i] = h; lo[i] = l;
}
// previous[b][ci][j] <- (hi + lo)[b][T + j][ci] for rows with exec_mask (conv.py:263-267)
__global__ void tm_commit_bct_kernel(const float* __restrict__ hi, const float* __restrict__ lo, float* __restrict__ prev,
                                     const uint8_t* __restrict__ exec_mask, int B, int Cin, int T, int P) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * Cin * P) return;
  const int j = (int)(i % P);
  const long long r = i / P;
  const int ci = (int)(r % Cin), b = (int)(r / Cin);
  if (exec_mask && !exec_mask[b]) return;
  const long long o = ((long long)b * (P + T) + T + j) * Cin + ci;
  prev[i] = hi[o] + lo[o];
}
struct DevBufs {
  std::vector<void*> p;
  ~DevBufs() { for (void* q : p) cudaFree(q); }
  template <class T> int get(T** out, size_t n) {
    void* q = nullptr;
    B200_CUDA(cudaMalloc(&q, n ? n : 1));
    p.push_back(q);
    *out = static_cast<T*>(q);
    return B200_OK;
  }
};

}  // namespace

extern "C" {

// StreamingConv1d on the down-sampling conv's kernels: weight re-layout, split-K GEMM + in-order reduction, state commit
int b200_op_conv1d(const float* x_dev, const float* w_dev, const float* bias_dev, float* prev_dev,
                   const uint8_t* exec_mask_dev, float* y_dev, int B, int Cin, int Cout, int T, int K, int stride,
                   int dilation, int elu_in, void* stream) {
  using namespace b200::mimi;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int keff = (K - 1) * dilation + 1, P = keff - stride;
  if (T % stride || P < 0) B200_FAIL(B200_ERR_SHAPE, "op_conv1d: T %% stride != 0");
  ConvSplitK p;
  p.x = x_dev; p.xb = (long long)Cin * T; p.xc = T; p.xt = 1; p.Tin = T;
  p.st = prev_dev; p.P = P; p.first = nullptr; p.bias = bias_dev;
  p.y = y_dev; p.yb = (long long)Cout * (T / stride); p.yc = T / stride; p.yt = 1;
  p.Cin = Cin; p.stride = stride; p.dil = dilation; p.Tout = T / stride; p.elu_in = elu_in;
  p.M = Cout; p.N = B * (T / stride); p.Kd = Cin * K;
  const int KS = ds_splits(p.Kd);
  DevBufs d;
  float *wp, *part;
  B200_TRY(d.get(&wp, (size_t)Cout * Cin * K * 4));
  B200_TRY(d.get(&part, (size_t)KS * p.N * p.M * 4));
  p.w = wp;
  const long long n = (long long)Cout * Cin * K;
  B200_LAUNCH(tm_weight_conv_kernel, (unsigned)ceil_div64(n, 256), 256, 0, st, w_dev, wp, Cout, Cin, K);
  B200_LAUNCH(conv_splitk_kernel, dim3(ceil_div(p.M, DS_CO), KS), 256, 0, st, p, part, KS);
  B200_LAUNCH(conv_splitk_reduce_kernel, (unsigned)ceil_div64((long long)p.N * p.M, 256), 256, 0, st, p, part, KS);
  if (P > 0) B200_LAUNCH(conv_commit_kernel, B, 128, 0, st, p, exec_mask_dev);
  B200_CUDA(cudaStreamSynchronize(st));
  return check_launch("op_conv1d");
}

int b200_op_tc_linear_f32(const float* x_dev, const float* w_dev, float* y_dev, int M, int N, int K, void* stream) {
  using namespace b200::mtc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!x_dev || !w_dev || !y_dev || M < 1 || K % 32 || N % 16) B200_FAIL(B200_ERR_SHAPE, "op_tc_linear_f32: bad shape");
  B200_TRY(tc_init());
  TcLayer L;
  L.s = tc_shape(TC_LINEAR_ROWS, N, K, 1);
  TcSchedule q;
  B200_TRY(plan_tc(L.s, 1, M, num_sms(), TC_SPLIT_BYTES, &q));
  DevBufs d;
  float *hi, *lo, *ws; uint8_t* wt;
  B200_TRY(d.get(&hi, (size_t)M * K * 4));
  B200_TRY(d.get(&lo, (size_t)M * K * 4));
  B200_TRY(d.get(&wt, tc_packed_bytes(L.s)));
  B200_TRY(d.get(&ws, TC_SPLIT_BYTES));
  const long long n = (long long)M * K;
  // x is already [M][K] token-major: a flat hi/lo split is tm_pack_in with B = M "sessions" of Cin = K, T = 1, P = 0
  B200_LAUNCH(tm_pack_in_kernel, (unsigned)ceil_div64(n, 256), 256, 0, st, x_dev, (const float*)nullptr, hi, lo, M, K, 1, 0, 0);
  B200_TRY(tc_pack_weights(w_dev, wt, L.s, st));
  L.wt = wt;
  TcParams e{};
  e.epi = TC_EPI_CONV; e.y = y_dev; e.y_sb = 0; e.y_row = N;
  B200_TRY(tc_bind(L, q, e, hi, lo, M, ws));
  B200_TRY(tc_launch(L, st));
  B200_CUDA(cudaStreamSynchronize(st));
  return B200_OK;
}

int b200_op_tc_conv1d(const float* x_dev, const float* w_dev, const float* bias_dev, float* prev_dev, const uint8_t* exec_mask_dev,
                      float* y_dev, int B, int Cin, int Cout, int T, int K, int stride, int dilation, int elu_in, int transposed,
                      void* stream) {
  using namespace b200::mtc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  B200_TRY(tc_init());
  // transposed: ConvTranspose1d with K == 2 * stride as two taps over [x[t-1], x[t]] (P = 1 carried input row, N = S * Cout)
  const int n_taps = transposed ? 2 : K, S = stride;
  const int P = transposed ? 1 : (K - 1) * dilation + 1 - stride;
  const int Tout = transposed ? T : T / stride;               // GEMM rows per session
  const int N = transposed ? S * Cout : Cout;
  if (Cin % 32 || N % 16 || (N > 128 && N % 128) || P < 0 || (!transposed && T % stride) || (transposed && K != 2 * S))
    B200_FAIL(B200_ERR_SHAPE, "op_tc_conv1d: unsupported shape");
  TcLayer L;
  L.s = transposed ? tc_shape(TC_CONVTR, N, Cin, 2, 1, 1, Cout) : tc_shape(TC_CONV, N, Cin, K, dilation, stride, Cout);
  L.bias = bias_dev;
  TcSchedule q;
  B200_TRY(plan_tc(L.s, B, Tout, num_sms(), TC_SPLIT_BYTES, &q));
  DevBufs d;
  float *hi, *lo, *ws, *wk, *ytm; uint8_t* wt;
  const size_t E = (size_t)P + T;
  B200_TRY(d.get(&hi, (size_t)B * E * Cin * 4));
  B200_TRY(d.get(&lo, (size_t)B * E * Cin * 4));
  B200_TRY(d.get(&wk, (size_t)N * n_taps * Cin * 4));
  B200_TRY(d.get(&wt, tc_packed_bytes(L.s)));
  B200_TRY(d.get(&ytm, (size_t)B * Tout * N * 4));
  B200_TRY(d.get(&ws, TC_SPLIT_BYTES));
  const long long n_in = (long long)B * E * Cin, n_w = (long long)N * n_taps * Cin;
  B200_LAUNCH(tm_pack_in_kernel, (unsigned)ceil_div64(n_in, 256), 256, 0, st, x_dev, (const float*)prev_dev, hi, lo, B, Cin, T, P, elu_in);
  if (transposed) B200_LAUNCH(mimi::tm_weight_convtr_kernel, (unsigned)ceil_div64(n_w, 256), 256, 0, st, w_dev, wk, Cin, Cout, S);
  else B200_LAUNCH(mimi::tm_weight_conv_kernel, (unsigned)ceil_div64(n_w, 256), 256, 0, st, w_dev, wk, Cout, Cin, K);
  B200_TRY(tc_pack_weights(wk, wt, L.s, st));
  L.wt = wt;
  TcParams e{};
  e.epi = TC_EPI_CONV; e.y = ytm; e.y_sb = (long long)Tout * N; e.y_row = N;
  B200_TRY(tc_bind(L, q, e, hi, lo, (long long)E, ws));
  B200_TRY(tc_launch(L, st));
  // token-major [B][Tout][N] -> the reference layout: conv [B][Cout][Tout]; convtr [B][Cout][Tout * S] (row t holds S steps of Cout)
  const int Tr = transposed ? Tout * S : Tout;
  B200_LAUNCH(mimi::tm_to_bct_kernel, (unsigned)ceil_div64((long long)B * Cout * Tr, 256), 256, 0, st, ytm, y_dev, B, Cout, Tr);
  if (P > 0 && prev_dev)
    B200_LAUNCH(tm_commit_bct_kernel, (unsigned)ceil_div64((long long)B * Cin * P, 256), 256, 0, st, hi, lo, prev_dev, exec_mask_dev, B, Cin, T, P);
  B200_CUDA(cudaStreamSynchronize(st));
  return check_launch("op_tc_conv1d");
}

// lm_noise_kernel with the LM's launch shape (lm.cu step_body), the step counter in a device word like the handle's
int b200_op_lm_noise(float* out_dev, int64_t n, uint64_t seed, uint64_t ctr, void* stream) {
  using namespace b200::lm;
  static unsigned long long* g_ctr = nullptr;
  if (!out_dev || n < 1) B200_FAIL(B200_ERR_INVALID, "op_lm_noise: null output or n < 1");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!g_ctr) B200_CUDA(cudaMalloc(&g_ctr, sizeof(unsigned long long)));
  const unsigned long long c = ctr;
  B200_CUDA(cudaMemcpyAsync(g_ctr, &c, sizeof(c), cudaMemcpyHostToDevice, st));
  B200_CUDA(cudaStreamSynchronize(st));          // `c` lives on this stack frame
  B200_LAUNCH(lm_noise_kernel, (unsigned)ceil_div64(ceil_div64(n, 4), 256), 256, 0, st, out_dev, (long long)n,
              (unsigned long long)seed, g_ctr);
  return check_launch("op_lm_noise");
}

int b200_op_exp1(const uint32_t* words_dev, float* out_dev, int64_t n, void* stream) {
  using namespace b200::lm;
  if (!words_dev || !out_dev || n < 1) B200_FAIL(B200_ERR_INVALID, "op_exp1: null pointer or n < 1");
  B200_LAUNCH(exp1_kernel, (unsigned)ceil_div64(n, 256), 256, 0, static_cast<cudaStream_t>(stream), words_dev, out_dev, (long long)n);
  return check_launch("op_exp1");
}

int b200_op_sample(const void* logits_bf16_dev, const float* noise_dev, int64_t* out_dev, int B, int card,
                   int use_sampling, float temp, int top_k, void* stream) {
  using namespace b200::lm;
  if (card + 1 > 65535 || top_k < 1 || top_k > SAMPLE_MAX_K) B200_FAIL(B200_ERR_SHAPE, "op_sample: bad card/top_k");
  const int k = top_k < card ? top_k : card;
  B200_LAUNCH(sample_kernel, B, SAMPLE_THREADS, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(logits_bf16_dev),
              (long long)card, noise_dev, (long long)k, reinterpret_cast<long long*>(out_dev), card, use_sampling, temp, top_k,
              nullptr, 0);
  return check_launch("op_sample");
}

int b200_op_sample_text_rows(const void* logits_bf16_dev, const float* noise_dev, int64_t noise_ld, int64_t* out_dev, int B, int card,
                             int use_sampling, float temp, int top_k, const b200_row_sampling* p, int32_t* history_dev,
                             int32_t* count_dev, int history, void* stream) {
  using namespace b200::lm;
  const char* what = "op_sample_text_rows";
  if (!logits_bf16_dev || !noise_dev || !out_dev || !history_dev || !count_dev || B < 1)
    B200_FAIL(B200_ERR_INVALID, "%s: null pointer or B < 1", what);
  if (card < 4 || card + 1 > 65535 || top_k < 1 || top_k > SAMPLE_MAX_K || history < 1 || history > 1024 || noise_ld < 1)
    B200_FAIL(B200_ERR_SHAPE, "%s: bad card / top_k / history / noise_ld", what);
  std::vector<RowSampling> rs(B, RowSampling{});
  for (int b = 0; p && b < B; ++b) B200_TRY(row_sampling_check(p[b], top_k, top_k, &rs[b], what));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RowSampling* rs_dev = nullptr;
  float* scores = nullptr;
  B200_CUDA(cudaMalloc(&rs_dev, (size_t)B * sizeof(RowSampling)));
  if (cudaMalloc(&scores, (size_t)B * card * 4) != cudaSuccess) {
    cudaFree(rs_dev);
    B200_FAIL(B200_ERR_CUDA, "%s: out of device memory", what);
  }
  cudaMemcpyAsync(rs_dev, rs.data(), rs.size() * sizeof(RowSampling), cudaMemcpyHostToDevice, st);
  text_rows_launch(static_cast<const bf16*>(logits_bf16_dev), scores, noise_dev, noise_ld, reinterpret_cast<long long*>(out_dev), B, card,
                   use_sampling, temp, top_k, rs_dev, TextHistory{history_dev, count_dev, history}, nullptr, st);
  const int rc = check_launch(what);
  cudaStreamSynchronize(st);
  cudaFree(scores);
  cudaFree(rs_dev);
  return rc;
}

}  // extern "C"
