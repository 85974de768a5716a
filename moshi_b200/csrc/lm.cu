// Moshi LM handle: weights (reference state-dict names), streaming state, and the per-frame decode
// step (LMGen._step, lm.py:668-783): token ring -> Temporal transformer -> text sample ->
// Depformer (dep_q dependent sub-steps) -> token ring.
#include "gemm_sk.cuh"
#include "lm_kernels.cuh"

using namespace b200;
using namespace b200::lm;

namespace {

struct TLayer {
  const bf16 *in_w, *out_w, *n1, *n2, *lin_in, *lin_out;
  const float *in_s = nullptr, *out_s = nullptr, *lin_in_s = nullptr, *lin_out_s = nullptr;   // int8 path: weight-row scales
};

}  // namespace

void b200::lm::attn_step_launch(const bf16* qkv, const KvRings& r, bf16* out, float* part, int* counters, const long long* pos,
                                const uint8_t* exec_mask, int B, int H, int cap, int nsplit, float max_period, int storage,
                                cudaStream_t st) {
  const dim3 grid(B * H, nsplit);
  const float nl = -logf(max_period) * 2.f / (float)ATT_D;
  if (storage) {
    const AttnStepQ8 a{qkv, static_cast<uint8_t*>(r.k), static_cast<uint8_t*>(r.v), r.ks, r.vs, out, part, counters, pos, exec_mask,
                       H, cap, nsplit, nl};
    if (storage == KV_INT8) B200_LAUNCH(attn_step_q8_kernel<KV_INT8>, grid, ATT_THREADS, 0, st, a);
    else B200_LAUNCH(attn_step_q8_kernel<KV_E4M3>, grid, ATT_THREADS, 0, st, a);
    return;
  }
  const AttnStep a{qkv, static_cast<bf16*>(r.k), static_cast<bf16*>(r.v), out, part, counters, pos, exec_mask, H, cap, nsplit, nl,
                   r.table, r.tab_ld, r.page_shift};
  if (r.table) B200_LAUNCH(attn_step_kernel<true>, grid, ATT_THREADS, 0, st, a);
  else B200_LAUNCH(attn_step_kernel<false>, grid, ATT_THREADS, 0, st, a);
}

void b200::lm::cross_attn_launch(const bf16* q, long long ldq, const bf16* kc, const bf16* vc, bf16* out, float* part, int* counters,
                                 int B, int H, int T, int nsplit, cudaStream_t st) {
  const CrossAttnStep a{q, ldq, kc, vc, out, part, counters, H, T, nsplit};
  B200_LAUNCH(cross_attn_step_kernel, dim3(B * H, nsplit), ATT_THREADS, 0, st, a);
}

// ---- temporal K/V storage -----------------------------------------------------------------------------------------------------
// The temporal K/V of one LM handle, in one of four forms: bf16 rings of the model's context (the reference's RingKVCache), rings
// shortened to kv_capacity slots, 8-bit rings (kv_dtype), or one pool of pages shared by all rows (kv_pool_frames).  Only this
// unit knows which: the handle asks it for the step's prologue and each layer's rings, position writes, the state entries, the K/V
// section of a session record and the meaning of error flags 4 and 8.
namespace {

struct TemporalKv {
  // configuration, before streaming_begin
  int kind = B200_KV_BF16;                     // B200_KV_BF16, or 8-bit rings B200_KV_FP8_E4M3 / B200_KV_INT8 (= KV_E4M3 / KV_INT8)
  int capacity = 0;                            // slots per ring when shorter than the context, else 0
  int64_t pool_frames = 0;                     // > 0: the bf16 rings live in pages of page_slots slots
  int page_slots = 64;
  int context = 0, H = 0;                      // the model's
  // geometry, from streaming_begin
  int MB = 0, cap = 0;                         // model rows, slots per ring
  int n_pages = 0, tab_ld = 0, page_shift = 0;   // n_pages = 0: no pool
  // per layer K and V: bf16 rings [MB][H][cap][ATT_D] or pools [n_pages + 1][H][page_slots][ATT_D] (the last page a sink), or
  // 8-bit rings [MB][H][cap][ATT_D] and their fp32 scales ks / vs [MB][H][cap]
  struct Layer { void *k = nullptr, *v = nullptr; float *ks = nullptr, *vs = nullptr; };
  std::vector<Layer> layers;
  int *table = nullptr, *held = nullptr;             // [MB][tab_ld] (-1 = unmapped), pages held per row [MB]
  int *free_stack = nullptr, *free_top = nullptr;    // [n_pages], [1]
  void** arrays = nullptr;                     // what kv_copy_kernel reads: [layer][k|v], then for 8-bit rings [layer][ks|vs]
  const long long* pos = nullptr;              // the handle's model.offset [MB]

  // bytes of one head's K (or V) in one slot: ATT_D bf16, or ATT_D 8-bit codes and their fp32 scale
  int64_t slot_bytes() const { return kind ? ATT_D + 4 : ATT_D * 2; }
  size_t ring_slots() const { return n_pages ? (size_t)(n_pages + 1) * page_slots : (size_t)MB * cap; }   // per layer and head
  size_t bytes() const { return layers.size() * 2 * ring_slots() * H * slot_bytes(); }

  int pool_conflict(int64_t frames, const char* what) const {
    if (frames > 0 && (kind || capacity > 0))
      B200_FAIL(B200_ERR_INVALID, "%s: the KV pool holds bf16 rings of the model's context (no kv_dtype or kv_capacity)", what);
    return B200_OK;
  }
  int set_dtype(int dtype) {
    if (dtype != B200_KV_BF16 && dtype != B200_KV_FP8_E4M3 && dtype != B200_KV_INT8)
      B200_FAIL(B200_ERR_INVALID, "lm_set_kv_dtype: unknown dtype %d", dtype);
    kind = dtype;
    return B200_OK;
  }
  int set_capacity(int slots) {
    if (slots < 0) B200_FAIL(B200_ERR_INVALID, "lm_set_kv_capacity: negative capacity");
    capacity = slots >= context ? 0 : slots;
    return B200_OK;
  }
  int set_pool(int64_t frames, int slots) {
    if (frames < 0) B200_FAIL(B200_ERR_INVALID, "lm_set_kv_pool: negative size");
    if (frames > 0) {
      if (slots < 4 || slots > 256 || (slots & (slots - 1)))
        B200_FAIL(B200_ERR_INVALID, "lm_set_kv_pool: page_slots %d (a power of two in [4, 256])", slots);
      B200_TRY(pool_conflict(frames, "lm_set_kv_pool"));
      page_slots = slots;
    }
    pool_frames = frames;
    return B200_OK;
  }

  // streaming_begin, before it allocates: the geometry of `rows` model rows and `n_layers` layers
  int plan(int rows, int n_layers) {
    B200_TRY(pool_conflict(pool_frames, "lm_streaming_begin"));
    MB = rows;
    cap = capacity > 0 ? capacity : context;
    n_pages = tab_ld = page_shift = 0;
    if (pool_frames > 0) {
      tab_ld = ceil_div(context, page_slots);
      page_shift = __builtin_ctz(page_slots);
      n_pages = (int)std::min(ceil_div64(pool_frames, page_slots), (int64_t)MB * tab_ld);
    }
    layers.assign(n_layers, Layer{});
    return B200_OK;
  }
  // layer l's K and V, where streaming_begin allocates that layer's state
  int alloc_layer(Arena& A, int l) {
    Layer& L = layers[l];
    const size_t n = ring_slots() * H;         // (head, slot) pairs
    B200_TRY(A.alloc(&L.k, n * (kind ? ATT_D : ATT_D * 2)));
    B200_TRY(A.alloc(&L.v, n * (kind ? ATT_D : ATT_D * 2)));
    if (kind) {
      B200_TRY(A.alloc_t(&L.ks, n));
      B200_TRY(A.alloc_t(&L.vs, n));
    }
    return B200_OK;
  }
  // the page table, page counts and free stack (nothing without a pool)
  int alloc_pages(Arena& A) {
    if (!n_pages) return B200_OK;
    B200_TRY(A.alloc_t(&table, (size_t)MB * tab_ld, false));
    B200_CUDA(cudaMemset(table, 0xFF, (size_t)MB * tab_ld * 4));      // -1: unmapped
    B200_TRY(A.alloc_t(&held, MB));
    B200_TRY(A.alloc_t(&free_stack, n_pages, false));
    B200_TRY(A.alloc_t(&free_top, 1, false));
    std::vector<int> stack(n_pages);
    for (int i = 0; i < n_pages; ++i) stack[i] = n_pages - 1 - i;        // page 0 is popped first
    B200_CUDA(cudaMemcpy(free_stack, stack.data(), stack.size() * 4, cudaMemcpyHostToDevice));
    B200_CUDA(cudaMemcpy(free_top, &n_pages, 4, cudaMemcpyHostToDevice));
    return B200_OK;
  }
  // The state entries layers.<l>.k / .v [MB][H][cap][ATT_D] bf16 (a paged layer's in that ring layout too, see copy_entry), or
  // .k8 / .v8 and .k_scale / .v_scale; then the device list of the arrays.
  int mark_state(Arena& A) {
    const int D = ATT_D;
    const size_t n = (size_t)MB * H * cap;
    std::vector<void*> list;
    for (size_t l = 0; l < layers.size(); ++l) {
      const Layer& L = layers[l];
      const std::string p = "layers." + std::to_string(l);
      if (kind) {
        A.mark_state(L.k, n * D, p + ".k8", B200_U8, {MB, H, cap, D});
        A.mark_state(L.v, n * D, p + ".v8", B200_U8, {MB, H, cap, D});
        A.mark_state(L.ks, n * 4, p + ".k_scale", B200_F32, {MB, H, cap});
        A.mark_state(L.vs, n * 4, p + ".v_scale", B200_F32, {MB, H, cap});
      } else {
        A.mark_state(L.k, n * D * 2, p + ".k", B200_BF16, {MB, H, cap, D});
        A.mark_state(L.v, n * D * 2, p + ".v", B200_BF16, {MB, H, cap, D});
      }
      list.insert(list.end(), {L.k, L.v});
    }
    for (auto& L : layers)
      if (kind) list.insert(list.end(), {L.ks, L.vs});
    B200_TRY(A.alloc_t(&arrays, list.size(), false));
    B200_CUDA(cudaMemcpy(arrays, list.data(), list.size() * sizeof(void*), cudaMemcpyHostToDevice));
    return B200_OK;
  }
  void end() {
    MB = cap = n_pages = tab_ld = page_shift = 0;
    layers.clear();
    table = held = free_stack = free_top = nullptr;
    arrays = nullptr; pos = nullptr;
  }

  // Before the step's first layer: a shortened ring serves a session only until it is full, so a row about to overwrite a live key
  // raises flag 4 instead of silently forgetting; a pool maps the page of this step's slot (all layers share the table).
  void prologue(const uint8_t* exec_mask, int* err, cudaStream_t st) const {
    if (cap < context) B200_LAUNCH(kv_capacity_check_kernel, ceil_div(MB, 128), 128, 0, st, pos, exec_mask, MB, cap, err);
    if (n_pages)
      B200_LAUNCH(kv_page_alloc_kernel, 1, KV_PAGE_THREADS, 0, st, table, held, free_stack, free_top, pos, exec_mask, MB, tab_ld,
                  page_shift, context, n_pages, err);
  }
  KvRings rings(int l) const { return {layers[l].k, layers[l].v, layers[l].ks, layers[l].vs, table, tab_ld, page_shift}; }
  // b200_lm_reset: the masked sessions' rows (b and b + B under CFG; null mask = all) return their pages to the pool
  void release(const uint8_t* mask, int B, cudaStream_t st) const {
    if (n_pages)
      B200_LAUNCH(kv_page_free_kernel, 1, KV_PAGE_THREADS, 0, st, table, held, free_stack, free_top, mask, B, MB, tab_ld);
  }

  // Model rows row0 + k * row_step are about to hold positions at[k], in ascending row order.  A pool gives each exactly the pages of
  // slots [0, min(at[k], context)) (synchronises): excess pages are pushed back first (row and table order), then missing ones
  // are popped (row order); B200_ERR_STATE, changing nothing, when the free pages do not cover them.  Rings need nothing.
  int hold(int row0, int row_step, const std::vector<long long>& at, const char* what, cudaStream_t st) {
    if (!n_pages) return B200_OK;
    auto pages_for = [&](long long p) { return (int)((std::min(std::max(p, 0LL), (long long)context) + page_slots - 1) / page_slots); };
    const int T = tab_ld, n_rows = (int)at.size();
    std::vector<int> tab((size_t)MB * T), got(MB), stack(n_pages);
    int top = 0;
    const struct { int* dev; int* host; size_t n; } io[4] = {{table, tab.data(), tab.size()}, {held, got.data(), got.size()},
                                                            {free_stack, stack.data(), stack.size()}, {free_top, &top, 1}};
    B200_CUDA(cudaStreamSynchronize(st));
    for (auto& x : io) B200_CUDA(cudaMemcpy(x.host, x.dev, x.n * 4, cudaMemcpyDeviceToHost));
    int more = 0;
    for (int k = 0; k < n_rows; ++k) more += pages_for(at[k]) - got[row0 + k * row_step];
    if (more > top) B200_FAIL(B200_ERR_STATE, "%s: the rows need %d more KV pages, the pool has %d free", what, more, top);
    for (int k = 0; k < n_rows; ++k) {
      const int b = row0 + k * row_step, want = pages_for(at[k]);
      int* row = tab.data() + (size_t)b * T;
      for (int i = want; i < T; ++i) {
        if (i < got[b]) stack[top++] = row[i];
        row[i] = -1;
      }
      got[b] = std::min(got[b], want);
    }
    for (int k = 0; k < n_rows; ++k) {
      const int b = row0 + k * row_step, want = pages_for(at[k]);
      for (int i = got[b]; i < want; ++i) tab[(size_t)b * T + i] = stack[--top];
      got[b] = want;
    }
    for (auto& x : io) B200_CUDA(cudaMemcpy(x.dev, x.host, x.n * 4, cudaMemcpyHostToDevice));
    return B200_OK;
  }
  // the same for every model row, the positions being a model.offset [MB] on the device about to be written
  int hold_dev(const void* at_dev, const char* what, cudaStream_t st) {
    if (!n_pages) return B200_OK;
    std::vector<long long> at(MB);
    B200_CUDA(cudaStreamSynchronize(st));
    B200_CUDA(cudaMemcpy(at.data(), at_dev, (size_t)MB * 8, cudaMemcpyDeviceToHost));
    return hold(0, 1, at, what, st);
  }
  // a shortened ring holds a session's history until position cap: B200_ERR_STATE past it
  int check_history(int64_t top, const char* what) const {
    if (cap < context && top > cap)
      B200_FAIL(B200_ERR_STATE, "%s: the session is at position %lld, past its %d-slot KV ring: the ring no longer holds its history", what,
                (long long)top, cap);
    return B200_OK;
  }

  // K / V of n_arrays arrays from arrays[first] on, model rows row0 + k * row_step (k < n_rows), slots [0, n), to or from the flat
  // buffer [array][k][H][n][slot] (kv_copy_kernel).  scales: the arrays are 8-bit rings' fp32 scales.
  template <typename U, int V>
  static void launch_copy(bool gather, dim3 grid, const KvCopy& a, cudaStream_t st) {
    if (gather) B200_LAUNCH((kv_copy_kernel<true, U, V>), grid, 256, 0, st, a);
    else B200_LAUNCH((kv_copy_kernel<false, U, V>), grid, 256, 0, st, a);
  }
  int copy(int first, int n_arrays, int row0, int n_rows, int row_step, int n, void* flat, bool gather, bool scales,
           cudaStream_t st) const {
    if (n <= 0) return B200_OK;
    KvCopy a;
    a.arrays = arrays + first; a.flat = flat; a.pos = pos;
    a.table = table; a.tab_ld = tab_ld; a.page_shift = page_shift; a.sink = n_pages;
    a.row0 = row0; a.n_rows = n_rows; a.row_step = row_step; a.H = H; a.cap = cap; a.n = n;
    const long long segs = (long long)n_arrays * n_rows * H;
    if (segs > 65535) B200_FAIL(B200_ERR_INVALID, "kv_copy: %lld ring segments in one launch", segs);
    const int V = scales ? 1 : kind ? ATT_D / 16 : ATT_D / 8;     // 4-byte scales, 16-byte vectors of bytes or bf16
    const dim3 grid((unsigned)ceil_div(n * V, 256), (unsigned)segs);
    if (scales) launch_copy<uint32_t, 1>(gather, grid, a, st);
    else if (kind) launch_copy<uint4, ATT_D / 16>(gather, grid, a, st);
    else launch_copy<uint4, ATT_D / 8>(gather, grid, a, st);
    return check_launch("kv_copy");
  }
  // A paged layer's K / V state entry keeps the ring layout: its index in `arrays`, or -1 (another entry, or no pool) ...
  int paged_array(const void* p) const {
    for (size_t l = 0; n_pages && l < layers.size(); ++l) {
      if (p == layers[l].k) return 2 * (int)l;
      if (p == layers[l].v) return 2 * (int)l + 1;
    }
    return -1;
  }
  // ... gathered from the pool into dst, or scattered from src into it
  int copy_entry(int arr, void* dst, const void* src, cudaStream_t st) const {
    return copy(arr, 1, 0, MB, 1, cap, dst ? dst : const_cast<void*>(src), dst != nullptr, false, st);
  }

  // The K/V section of a session record: slots [0, n) of `rows` model rows (row, row + row_step) as
  // [layer][k|v][model row][head][n][ATT_D], 8-bit rings' bytes followed by their fp32 scales [layer][k|v][model row][head][n]
  int64_t record_bytes(int rows, int64_t n) const { return (int64_t)layers.size() * 2 * H * slot_bytes() * rows * n; }
  int check_record(uint32_t record_kind, const char* what) const {
    if (record_kind != (uint32_t)kind)
      B200_FAIL(B200_ERR_INVALID, "%s: the record's KV storage type %u differs from the handle's %d", what, record_kind, kind);
    return B200_OK;
  }
  int record(int row, int rows, int row_step, int n, char* rec, bool gather, cudaStream_t st) const {
    const int L2 = 2 * (int)layers.size();
    B200_TRY(copy(0, L2, row, rows, row_step, n, rec, gather, false, st));
    if (kind) B200_TRY(copy(L2, L2, row, rows, row_step, n, rec + (int64_t)L2 * rows * H * n * ATT_D, gather, true, st));
    return B200_OK;
  }

  // error flags 4 (a row stepped past its shortened ring) and 8 (a row's ring did not get a page) as B200_ERR_STATE
  int flag_error(int flags, const char* what) const {
    if (flags & ERR_KV_CAPACITY)
      B200_FAIL(B200_ERR_STATE, "%s: a session stepped past its %d-slot KV ring (b200_lm_set_kv_capacity; flags %d)", what, cap, flags);
    if (flags & ERR_KV_POOL)
      B200_FAIL(B200_ERR_STATE, "%s: a session's KV ring did not get a page: the KV pool of %d pages is full (flags %d)", what, n_pages,
                flags);
    return B200_OK;
  }
  // flag 8 alone, read and cleared on the device (synchronises); the other flags stay
  int check_pool_flag(int* err, const char* what, cudaStream_t st) const {
    if (!n_pages) return B200_OK;
    int v = 0;
    B200_CUDA(cudaMemcpyAsync(&v, err, 4, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    if (!(v & ERR_KV_POOL)) return B200_OK;
    const int rest = v & ~ERR_KV_POOL;
    B200_CUDA(cudaMemcpyAsync(err, &rest, 4, cudaMemcpyHostToDevice, st));
    B200_CUDA(cudaStreamSynchronize(st));
    return flag_error(v, what);
  }
  int usage(int* used, int* total, cudaStream_t st) const {
    int top = 0;
    if (n_pages) {
      B200_CUDA(cudaMemcpyAsync(&top, free_top, 4, cudaMemcpyDeviceToHost, st));
      B200_CUDA(cudaStreamSynchronize(st));
    }
    if (used) *used = n_pages - top;
    if (total) *total = n_pages;
    return B200_OK;
  }
};

}  // namespace

// ---- depformer ----------------------------------------------------------------------------------------------------------------
// The depformer (lm.py:450-493, 809-850): weights, per-batch buffers, the path a batch takes (tc::plan_depformer: none, the launch
// chain or the persistent kernel of dep_fused.cu) and where each sub-step's Exp(1) draws start in a noise row.  Its allocations
// keep their place in streaming_begin's order (begin, alloc_guided, alloc_activations, and alloc_fused after linear_init).
namespace {

struct Depformer {
  // sub-step k of layer l: packed tiles, and under int8 their weight-row scales
  struct Step { const bf16 *in_w, *out_w, *lin_in, *lin_out; const float *in_s, *out_s, *lin_in_s, *lin_out_s; };
  // configuration
  int dep_q = 0, dd = 0, H = 0, F = 0, L = 0, card = 0, text_card = 0;
  int mode = B200_DEPFORMER_AUTO;              // b200_lm_set_depformer, before streaming_begin
  // b200_lm_set_depformer_schedule / _low_rank, before the first tensor: sub-step k runs weight set sched[k] of n_sets
  // (lm.py:172-181, transformer.py:399-401); low_rank > 0: the embedding tables arrive as [V][low_rank] factors
  std::vector<int> sched;
  int n_sets = 0, low_rank = 0;
  int kt = 0, ka = 0;                          // Exp(1) draws per noise row of the text sampler, and of each sub-step's
  // weights
  const bf16* in_all = nullptr;                // depformer_in.{j} stacked: all n_sets projections of transformer_out are one GEMM
  const float* in_s = nullptr;
  std::vector<Step> w;                         // [dep_q][L], sub-step k pointing at the tiles of set sched[k]
  std::vector<const bf16*> n1, n2;             // [L]
  std::vector<const bf16*> tables;             // [0] = depformer_text_emb, [k] = depformer_emb[k-1]
  std::vector<const bf16*> heads; std::vector<const float*> heads_s;    // linears[k]
  // per batch
  tc::DepformerPlan plan{};
  int B = 0, MB = 0;
  bf16 *din = nullptr, *dx = nullptr, *dxn = nullptr, *dqkv = nullptr, *dao = nullptr, *dh = nullptr;
  bf16 *logits = nullptr, *logits_cfg = nullptr;       // [dep_q][MB][card], under CFG the guided [dep_q][B][card]
  std::vector<bf16*> kc, vc;                   // [L] the frame's K / V [MB][H][dep_q][64]
  float *part0 = nullptr, *part1 = nullptr;    // the persistent kernel's split partials, its grid barrier ...
  unsigned* bar = nullptr;
  unsigned long long* trace = nullptr;         // ... and (B200_DEP_TRACE=1, diagnostics) its barrier timestamps
  tc::DepFused* fused = nullptr;

  void configure(const b200_lm_config& c) {
    dep_q = c.dep_q; dd = c.depformer_dim; H = c.depformer_num_heads; F = c.depformer_ffn_hidden;
    L = c.dep_q > 0 ? c.depformer_num_layers : 0; card = c.card; text_card = c.text_card;
    set_schedule(nullptr, 0);
  }
  // n = 0: one weight set per sub-step
  void set_schedule(const int* s, int n) {
    sched.resize(dep_q);
    n_sets = n ? 0 : dep_q;
    for (int k = 0; k < dep_q; ++k) {
      sched[k] = n ? s[k] : k;
      n_sets = std::max(n_sets, sched[k] + 1);
    }
  }
  // the first column of sub-step k's block of din, and din's row stride
  int din_col(int k) const { return sched[k] * dd; }
  long long din_ld() const { return (long long)n_sets * dd; }
  // where sub-step k's draws start in a noise row (k = dep_q: the row's length)
  long long noise_at(int k) const { return kt + (long long)k * ka; }
  void set_sampling(int use_sampling, float temp, int top_k, int top_k_text) {
    kt = std::min(top_k_text, text_card);
    ka = std::min(top_k, card);
    tc::dep_fused_set_sampling(fused, use_sampling, temp, top_k);
  }
  // streaming_begin: the plan of `batch` sessions, and the frame's K / V
  int begin(Arena& A, int batch, bool cfg, bool i8) {
    B = batch;
    MB = cfg ? 2 * batch : batch;
    B200_TRY(tc::plan_depformer(dep_q, dd, H, F, card, B, cfg, i8, num_sms(), tc::sk_gemv_max_m(), mode, &plan));
    kc = vc = std::vector<bf16*>(L);
    for (int l = 0; l < L; ++l) {
      B200_TRY(A.alloc_t(&kc[l], (size_t)MB * dd * dep_q));
      B200_TRY(A.alloc_t(&vc[l], (size_t)MB * dd * dep_q));
    }
    return B200_OK;
  }
  int alloc_guided(Arena& A) { return A.alloc_t(&logits_cfg, (size_t)B * std::max(dep_q, 1) * card); }
  int alloc_activations(Arena& A) {
    const size_t q1 = std::max(dep_q, 1);
    B200_TRY(A.alloc_t(&din, (size_t)MB * q1 * dd));
    B200_TRY(A.alloc_t(&dx, (size_t)MB * dd));
    B200_TRY(A.alloc_t(&dxn, (size_t)MB * dd));
    B200_TRY(A.alloc_t(&dqkv, (size_t)MB * 3 * dd));
    B200_TRY(A.alloc_t(&dao, (size_t)MB * dd));
    B200_TRY(A.alloc_t(&dh, (size_t)MB * F));
    return A.alloc_t(&logits, (size_t)MB * q1 * card);
  }
  int alloc_fused(b200_lm* h);
  int load(b200_lm* h);
  int run(b200_lm* h, bool replace);
  void end() {
    tc::dep_fused_destroy(fused);
    fused = nullptr; plan = tc::DepformerPlan{}; B = MB = 0; kc.clear(); vc.clear();
    din = dx = dxn = dqkv = dao = dh = logits = logits_cfg = nullptr; part0 = part1 = nullptr; bar = nullptr; trace = nullptr;
  }

  // b200_lm_read_buffer's depformer entries; false for any other name
  bool buffer(const std::string& n, bool cfg, const void** src, int64_t* sz) const {
    // with CFG "dep_logits" are what the samplers read (the guided rows, lm.py:828-833), "model_dep_logits" the model's 2B rows
    if (n == "dep_logits") { *src = cfg ? logits_cfg : logits; *sz = (int64_t)dep_q * B * card * 2; }
    else if (n == "model_dep_logits") { *src = logits; *sz = (int64_t)dep_q * MB * card * 2; }
    else if (n == "dep_trace") { *src = trace; *sz = trace ? (int64_t)tc::DEP_TRACE_SLOTS * 8 : 0; }
    else if (n == "dep_in" && dep_q > 0) { *src = din; *sz = (int64_t)MB * din_ld() * 2; }
    else if (n.rfind("depformer.tables.", 0) == 0 && dep_q > 0) {
      const std::string idx = n.substr(17);
      const bool digits = !idx.empty() && idx.size() <= 2 && idx.find_first_not_of("0123456789") == std::string::npos;
      const int k = digits ? atoi(idx.c_str()) : -1;
      if (k < 0 || k >= dep_q) return false;
      *src = tables[k];
      *sz = (int64_t)((k == 0 ? text_card : card) + 1) * dd * 2;
    }
    else if (n.rfind("depformer.layers.", 0) == 0 && dep_q > 0) {
      // the per-frame cache of one layer: after a frame it holds every sub-step's k / v
      const std::string rest = n.substr(17);
      const size_t dot = rest.find('.');
      const std::string idx = rest.substr(0, dot), kind = dot == std::string::npos ? "" : rest.substr(dot + 1);
      const bool digits = !idx.empty() && idx.size() <= 4 && idx.find_first_not_of("0123456789") == std::string::npos;
      const int l = digits ? atoi(idx.c_str()) : -1;
      if (l < 0 || l >= L || (kind != "k" && kind != "v")) return false;
      *src = kind == "k" ? kc[l] : vc[l];
      *sz = (int64_t)MB * dd * dep_q * 2;
    } else {
      return false;
    }
    return true;
  }
};

}  // namespace

// ---- cross-attention conditioning ---------------------------------------------------------------------------------------------
// The TTS models' conditioning (transformer.py:727-732, 779-798): every temporal layer attends to its row's condition memory
// k_cross / v_cross [MB][H][T][ATT_D] bf16.  Only this unit knows the key count T, the layers' weights, the memory's size and
// buffers, its fill, the step's block, the state entries and the record section; the handle asks only whether it is on (taps).
namespace {

// condition rows (x T keys) per K/V projection GEMM of the fill: the LM GEMMs take at most 256 rows
constexpr int CROSS_CHUNK = 256;

struct CrossAttention {
  // configuration: b200_lm_set_cross_attention before finalize, b200_lm_set_cross_len before streaming_begin
  bool on = false;
  int T = 0;                                   // keys per condition memory
  int d = 0, H = 0;                            // the model's
  // per layer (when on): norm_cross weight and bias, the query / K|V / output linears in packed tiles, and the memory's K and V
  struct Layer { const bf16 *nw = nullptr, *nb = nullptr, *q_w = nullptr, *kv_w = nullptr, *out_w = nullptr; bf16 *k = nullptr, *v = nullptr; };
  std::vector<Layer> layers;
  // per batch
  int MB = 0, nsplit = 1;                      // model rows, splits of the attention
  bf16 *chunk = nullptr, *chunk_kv = nullptr;  // fill staging: [CROSS_CHUNK][d] rows of the condition, their K|V
  int* rows_dev = nullptr;                     // [MB] model rows of the condition rows being filled

  int set(int enable, const b200_lm_config& c) {
    if (enable && c.quantize)      // the reference's _compute_cross_attention asserts an nn.Linear in_proj
      B200_FAIL(B200_ERR_INVALID, "lm_set_cross_attention: cross-attention layers with quantize=True (int8 linears) are not supported");
    on = enable != 0;
    d = c.dim; H = c.num_heads;
    layers.assign(on ? c.num_layers : 0, Layer{});
    return B200_OK;
  }
  int set_len(int keys, bool streaming) {
    if (!on) B200_FAIL(B200_ERR_INVALID, "lm_set_cross_len: the model has no cross-attention layers");
    if (streaming) B200_FAIL(B200_ERR_STATE, "lm_set_cross_len: the condition memory is allocated at streaming_begin; set it before");
    if (keys < 1 || keys > (1 << 20)) B200_FAIL(B200_ERR_INVALID, "lm_set_cross_len: %d keys", keys);
    T = keys;
    return B200_OK;
  }

  // bytes of one model row's memory in one layer, K or V
  int64_t row_bytes() const { return (int64_t)H * T * ATT_D * 2; }
  // bytes of the memory of `rows` model rows, K and V of every layer (0 when off)
  int64_t bytes(int64_t rows) const { return (int64_t)layers.size() * 2 * rows * row_bytes(); }
  // the largest M of its linears (the fill's chunks; the step's run MB), 0 when off
  int max_m() const { return on ? CROSS_CHUNK : 0; }

  // streaming_begin, before it allocates: `rows` model rows, and the splits of the attention (its partials share attn_part)
  int plan(int rows) {
    if (on && T < 1) B200_FAIL(B200_ERR_STATE, "lm_streaming_begin: set the condition memory's length (b200_lm_set_cross_len) first");
    MB = rows;
    nsplit = on ? attn_pick_splits(MB, H, T) : 1;
    return B200_OK;
  }
  // layer l's memory, where streaming_begin allocates that layer's state
  int alloc_layer(Arena& A, int l) {
    if (!on) return B200_OK;
    B200_TRY(A.alloc_t(&layers[l].k, (size_t)MB * H * T * ATT_D));
    return A.alloc_t(&layers[l].v, (size_t)MB * H * T * ATT_D);
  }
  int alloc_fill(Arena& A) {
    if (!on) return B200_OK;
    B200_TRY(A.alloc_t(&chunk, (size_t)CROSS_CHUNK * d, false));
    B200_TRY(A.alloc_t(&chunk_kv, (size_t)CROSS_CHUNK * 2 * d, false));
    return A.alloc_t(&rows_dev, MB, false);
  }
  // the state entries layers.<l>.k_cross / .v_cross (_MHAState, transformer.py:321-327)
  void mark_state(Arena& A) const {
    for (size_t l = 0; l < layers.size(); ++l) {
      const std::string p = "layers." + std::to_string(l);
      A.mark_state(layers[l].k, (size_t)(MB * row_bytes()), p + ".k_cross", B200_BF16, {MB, H, T, ATT_D});
      A.mark_state(layers[l].v, (size_t)(MB * row_bytes()), p + ".v_cross", B200_BF16, {MB, H, T, ATT_D});
    }
  }
  void end() {
    MB = 0; nsplit = 1;
    chunk = chunk_kv = nullptr; rows_dev = nullptr;
    for (Layer& L : layers) L.k = L.v = nullptr;
  }
  int load(b200_lm* h, int l);
  int fill(b200_lm* h, const void* src, const int32_t* rows_host, int n_rows) const;
  int step(b200_lm* h, int l) const;

  // The condition-memory section of a session record: from the first 256-byte boundary at or after `end` (*off), the memory of
  // the session's `rows` model rows as [layer][k|v][model row][H][T][ATT_D] bf16.  Returns the record's end (`end` when off).
  int64_t record_section(int64_t end, int rows, int64_t* off) const {
    *off = (end + 255) / 256 * 256;
    return on ? *off + bytes(rows) : end;
  }
  // model rows row + k * row_step (k < rows) to or from that section at `at`, each row's memory a contiguous [H][T][ATT_D]
  int record(int row, int rows, int row_step, char* at, bool gather, cudaStream_t st) const {
    const int64_t rb = row_bytes();
    for (const Layer& L : layers)
      for (bf16* m : {L.k, L.v})
        for (int k = 0; k < rows; ++k, at += rb) {
          char* mem = reinterpret_cast<char*>(m) + (int64_t)(row + k * row_step) * rb;
          B200_CUDA(cudaMemcpyAsync(gather ? at : mem, gather ? mem : at, (size_t)rb, cudaMemcpyDeviceToDevice, st));
        }
    return B200_OK;
  }
  // export: SESSION_CROSS, and T in the header's first reserved bytes
  void stamp(SessionHeader* s) const {
    if (!on) return;
    s->flags |= SESSION_CROSS;
    memcpy(s->reserved, &T, sizeof(int32_t));
  }
  // import: a record whose flag or T differs from the handle's is refused
  int check_record(const SessionHeader& s, const char* what) const {
    if (((s.flags & SESSION_CROSS) != 0) != on) B200_FAIL(B200_ERR_INVALID, "%s: cross-attention conditioning on one side only", what);
    int32_t keys = 0;
    memcpy(&keys, s.reserved, sizeof(keys));
    if (on && keys != T)
      B200_FAIL(B200_ERR_INVALID, "%s: the record's condition memory has %d keys, the handle's %d", what, keys, T);
    return B200_OK;
  }

  // its part of b200_lm_algorithmic_bytes for `rows` model rows: the query, K|V and output linears of every layer, once per step,
  // and each row's read of its memory
  int64_t algorithmic_bytes(int64_t rows) const { return on ? (int64_t)layers.size() * 4 * d * d * 2 + bytes(1) * rows : 0; }
};

}  // namespace

// ---- per-session sampling ----------------------------------------------------------------------------------------------------
// Each session's own temperatures, top-k, pad bias and text repetition penalty (b200_lm_set_session_sampling / _row_sampling).
// Only this unit knows whether it is on, the history length N, the device settings and history, the text path of the step
// (text_adjust_kernel, then the fp32-score sampler that appends to the history), the clear on reset, the state entries and the
// record section; the rest of the handle asks it whether it is on and for the per-row settings the audio samplers read.
namespace {

struct SessionSampling {
  int N = 0;                                   // history ring length; 0 = off (before streaming_begin)
  int B = 0, card = 0;
  RowSampling* params = nullptr;               // [B] (own = 0: the row follows the handle-wide values)
  int *ring = nullptr, *count = nullptr;       // [B][N], [B]
  float* scores = nullptr;                     // [B][text_card] the adjusted text scores of the step

  bool on() const { return N > 0; }
  int set(int history, bool streaming) {
    if (streaming) B200_FAIL(B200_ERR_STATE, "lm_set_session_sampling: the settings and histories are allocated at streaming_begin; set it before");
    if (history < 0 || history > 1024) B200_FAIL(B200_ERR_INVALID, "lm_set_session_sampling: history %d outside [0, 1024]", history);
    N = history;
    return B200_OK;
  }
  int alloc(Arena& A, int batch, int text_card) {
    if (!on()) return B200_OK;
    B = batch; card = text_card;
    B200_TRY(A.alloc_t(&params, B));
    B200_TRY(A.alloc_t(&ring, (size_t)B * N));
    B200_TRY(A.alloc_t(&count, B));
    return A.alloc_t(&scores, (size_t)B * card, false);
  }
  // the state entries session_sampling.params [B][8] (RowSampling's fields), .history [B][N], .count [B]
  void mark_state(Arena& A) const {
    if (!on()) return;
    A.mark_state(params, (size_t)B * sizeof(RowSampling), "session_sampling.params", B200_F32, {B, 8});
    A.mark_state(ring, (size_t)B * N * 4, "session_sampling.history", B200_I32, {B, N});
    A.mark_state(count, (size_t)B * 4, "session_sampling.count", B200_I32, {B});
  }
  void end() { B = card = 0; params = nullptr; ring = count = nullptr; scores = nullptr; }

  const RowSampling* rows() const { return on() ? params : nullptr; }
  TextHistory history() const { return TextHistory{ring, count, N}; }
  // b200_lm_set_row_sampling: every row and setting checked before anything is written
  int set_rows(const int32_t* rows, int n, const b200_row_sampling* p, int top_k, int top_k_text, cudaStream_t st) const {
    const char* what = "lm_set_row_sampling";
    if (!on()) B200_FAIL(B200_ERR_STATE, "%s: per-session sampling is off (b200_lm_set_session_sampling before streaming_begin)", what);
    if (n < 0 || (n > 0 && !rows)) B200_FAIL(B200_ERR_INVALID, "%s: %d rows", what, n);
    std::vector<RowSampling> v(n, RowSampling{});
    for (int k = 0; k < n; ++k) {
      if (rows[k] < 0 || rows[k] >= B) B200_FAIL(B200_ERR_INVALID, "%s: row %d outside [0, %d)", what, rows[k], B);
      if (p) B200_TRY(row_sampling_check(p[k], top_k, top_k_text, &v[k], what));
    }
    for (int k = 0; k < n; ++k)
      B200_CUDA(cudaMemcpyAsync(params + rows[k], &v[k], sizeof(RowSampling), cudaMemcpyHostToDevice, st));
    return B200_OK;
  }
  // b200_lm_reset: the masked rows' histories (null: all)
  void clear(const uint8_t* mask, cudaStream_t st) const {
    if (on()) B200_LAUNCH(text_history_clear_kernel, ceil_div(B, 128), 128, 0, st, count, mask, B);
  }

  // The session-record section: from the first 256-byte boundary at or after `end` (*off), the row's settings (32 bytes), its
  // count (4 bytes, then 12 of padding) and its history ring (N int32).  Returns the record's end (`end` when off).
  int64_t record_section(int64_t end, int64_t* off) const {
    *off = (end + 255) / 256 * 256;
    return on() ? *off + 48 + (int64_t)N * 4 : end;
  }
  int record(int row, char* at, bool gather, cudaStream_t st) const {
    if (!on()) return B200_OK;
    const struct { void* dev; char* rec; size_t n; } part[3] = {{params + row, at, sizeof(RowSampling)}, {count + row, at + 32, 4},
                                                              {ring + (size_t)row * N, at + 48, (size_t)N * 4}};
    for (const auto& x : part)
      B200_CUDA(cudaMemcpyAsync(gather ? x.rec : x.dev, gather ? x.dev : x.rec, x.n, cudaMemcpyDeviceToDevice, st));
    return B200_OK;
  }
  // export: SESSION_SAMPLING, and N in the header's reserved bytes after the condition memory's keys
  void stamp(SessionHeader* s) const {
    if (!on()) return;
    s->flags |= SESSION_SAMPLING;
    memcpy(s->reserved + 4, &N, sizeof(int32_t));
  }
  // import: a record whose flag or N differs from the handle's is refused
  int check_record(const SessionHeader& s, const char* what) const {
    if (((s.flags & SESSION_SAMPLING) != 0) != on()) B200_FAIL(B200_ERR_INVALID, "%s: per-session sampling on one side only", what);
    int32_t n = 0;
    memcpy(&n, s.reserved + 4, sizeof(n));
    if (on() && n != N) B200_FAIL(B200_ERR_INVALID, "%s: the record's text history holds %d tokens, the handle's %d", what, n, N);
    return B200_OK;
  }
};

}  // namespace

struct b200_lm : StreamCore {       // batch: sessions (LMGen batch); graphs[0]: the step
  b200_lm_config cfg;
  TensorStore store;
  Arena weights;
  int MB = 0;                          // rows the model runs on: batch, or 2 * batch under classifier-free guidance (lm.py:646-647)
  int Kc = 0, max_delay = 0, CT = 0;
  // sampling (LMGen defaults, lm.py:556-571)
  int use_sampling = 1, top_k = 250, top_k_text = 25;
  float temp = 0.8f, temp_text = 0.7f;
  int pdl = 1;                                 // programmatic dependent launch of the GEMMs (B200_PDL=0 disables)
  float* sk_ws = nullptr;                      // stream-K partial-accumulator slots (L2-resident)
  int* sk_counters = nullptr;                  // per-tile arrival counters (zero between launches)
  // weights
  EmbedTables emb;
  std::vector<TLayer> layers;
  const bf16 *out_norm = nullptr, *text_linear = nullptr;
  const float* text_linear_s = nullptr;
  int8_t* xq = nullptr; float* xq_scale = nullptr;     // int8 path: the current GEMM's quantised activations [B][max K] and row scales
  int* delays_dev = nullptr;
  // state
  long long *cache = nullptr, *offsets = nullptr, *pos = nullptr;
  uint8_t* exec_mask = nullptr;                // [batch] LMGen's mask
  uint8_t* exec_mask_m = nullptr;              // [MB] the model's mask (= exec_mask, or exec_mask.repeat(2) with CFG, lm.py:658-661)
  long long offset_cpu = 0;
  // classifier-free guidance (lm.py:596-604, 714-732, 820-833) and conditioning by sum (lm.py:398-399, 616-626)
  float cfg_coef = 1.f; int cfg_is_no_text = 0;
  std::vector<long long> cfg_until_host; long long* cfg_until = nullptr;
  bf16* text_logits_cfg = nullptr;             // guided logits [batch][text_card]
  bf16* cond_sum = nullptr; int cond_on = 0;                          // [MB][dim]
  // extra heads of the STT models (lm.py:224-226, 793-807)
  std::vector<const bf16*> extra_w; const bf16** extra_w_dev = nullptr; bf16* extra_out = nullptr;
  // Exp(1) noise drawn inside the step (when the caller passes none): Philox keyed by (seed, step counter)
  unsigned long long noise_seed = 0x9E3779B97F4A7C15ull; unsigned long long* noise_ctr = nullptr; int noise_internal = 0;
  // activations
  long long *in_codes = nullptr, *input_tokens = nullptr, *text_token = nullptr, *audio_tokens = nullptr, *out_tokens = nullptr;
  float* noise = nullptr;
  bf16 *x = nullptr, *xn = nullptr, *qkv = nullptr, *ao = nullptr, *hbuf = nullptr, *tout = nullptr;
  bf16* text_logits = nullptr;
  float* attn_part = nullptr;
  int* attn_counters = nullptr;                // split arrival counters [B*H]
  Depformer dep;                               // the depformer: weights, buffers and the path it runs on
  TemporalKv kv;                               // the temporal K/V: rings or pool, their state entries and record section
  CrossAttention cross;                        // cross-attention conditioning: weights, condition memory, fill and record section
  SessionSampling ss;                          // per-session sampling settings, text histories and their record section
  // session records: the per-session slices of the small state entries; the condition_sum rows come last and travel while it is on
  RowSlice* slices_dev = nullptr;
  int n_slices = 0, n_slices_cond = 0;
  long long slices_end = 0, slices_end_cond = 0, slices_max = 0;
  int nsplit = 1;
  // b200_lm_set_taps: the step copies the temporal stack's activations into taps (see tap_slot), allocated on first enable
  int taps_on = 0;
  bf16* taps = nullptr;
  int n_in_static = 0;
  int noise_static = 0;                        // 1: the captured step draws its own noise
  int replace_static = 0;                      // 1: this step's audio tokens are given (depformer_replace_tokens, lm.py:751-755)
  long long* replace_tokens = nullptr;         // [B][dep_q] staging of those tokens
  // pinned host staging
  long long *pin_in = nullptr, *pin_out = nullptr;
  float* pin_noise = nullptr;
  int64_t weight_bytes = 0;
  tc::TensorMapCache maps;
  // a paged handle gathers its K / V entries into ring layout and scatters them back (TemporalKv::copy_entry)
  int copy_entry(const StateEntry& e, void* dst, const void* src) override;
};

namespace {

int get_bf16(b200_lm* h, const std::string& name, std::vector<int64_t> shape, const bf16** out) {
  const Tensor* t = h->store.find(name);
  if (!t) B200_FAIL(B200_ERR_MISSING, "lm finalize: tensor '%s' was not loaded", name.c_str());
  if (t->dtype != B200_BF16) B200_FAIL(B200_ERR_SHAPE, "lm tensor '%s' must be bfloat16", name.c_str());
  if (t->shape != shape) {
    std::string got;
    for (auto s : t->shape) got += std::to_string(s) + ",";
    B200_FAIL(B200_ERR_SHAPE, "lm tensor '%s' has shape [%s]", name.c_str(), got.c_str());
  }
  *out = static_cast<const bf16*>(t->data);
  h->weight_bytes += t->numel() * 2;
  return B200_OK;
}

bool cfg_on(const b200_lm* h) { return h->cfg_coef != 1.f; }

int noise_per_row(const b200_lm* h) { return (int)h->dep.noise_at(h->cfg.dep_q); }

// The plan of y[M][N] = epi(x[M][K] . w[N][K]^T) on this device; norm: an RMSNorm in front that may fold into the GEMV.
int plan(const b200_lm* h, int M, int N, int K, int epi, int gate_rows, long long ldy, long long ldr, bool norm, tc::LinearPlan* out) {
  return tc::plan_linear(M, N, K, epi, gate_rows, h->cfg.quantize != 0, norm, ldy % 8 == 0 && ldr % 8 == 0, num_sms(), tc::sk_gemv_max_m(),
                         tc::LinearForce(), out);
}

// Runs a plan; `w` is the packed-tile form of gemm_sk.cu.
int run(b200_lm* h, const tc::LinearPlan& p, const bf16* x, long long ldx, const bf16* w, bf16* y, long long ldy, const bf16* res,
        long long ldr, const float* w_scales, const bf16* norm_alpha = nullptr) {
  tc::LinearArgs a{x, ldx, w, y, ldy, res, ldr, h->sk_ws, h->sk_counters, nullptr, nullptr, nullptr, norm_alpha, h->pdl};
  if (h->cfg.quantize) {       // QLinear.forward (utils/quantize.py:22-40): row-wise int8 activations, int8 x int8 -> int32
    if (!w_scales) B200_FAIL(B200_ERR_STATE, "quantised LM: linear without weight scales");
    B200_TRY(tc::sk_quantize_rows(x, ldx, h->xq, h->xq_scale, p.M, p.K, h->body, h->pdl));
    a.xq = h->xq; a.sa = h->xq_scale; a.sw = w_scales;
  }
  return tc::run_linear(h->maps, p, a, h->body);
}

// y[M][N] = epi(x[M][K] . w[N][K]^T)
int linear(b200_lm* h, const bf16* x, long long ldx, const bf16* w, bf16* y, long long ldy, const bf16* res,
           long long ldr, int M, int N, int K, int epi, int gate_rows, const float* w_scales = nullptr) {
  tc::LinearPlan p;
  B200_TRY(plan(h, M, N, K, epi, gate_rows, ldy, res ? ldr : 0, false, &p));
  return run(h, p, x, ldx, w, y, ldy, res, ldr, w_scales);
}

// y = epi(rmsnorm(x, alpha) . w^T).  Where the plan takes the GEMV (one or two sessions), the norm is folded into its
// activation staging (one kernel and one dependency less per linear); otherwise rmsnorm_kernel writes xn and the GEMM reads it.
int norm_linear(b200_lm* h, const bf16* x, const bf16* alpha, bf16* xn, const bf16* w, bf16* y, long long ldy, int M, int N, int K,
                int epi, int gate_rows, const float* w_scales) {
  tc::LinearPlan p;
  B200_TRY(plan(h, M, N, K, epi, gate_rows, ldy, 0, true, &p));
  if (p.norm_folded) return run(h, p, x, K, w, y, ldy, nullptr, 0, w_scales, alpha);
  B200_LAUNCH(rmsnorm_kernel, M, 256, 0, h->body, x, alpha, xn, K, 1e-8f);
  return run(h, p, xn, K, w, y, ldy, nullptr, 0, w_scales);
}

// A QLinear as model.q8.safetensors stores it (utils/quantize.py:16-21): "<name>" int8 [rows][K] + "<name>_scb" fp32 [rows]
int get_prequantised(b200_lm* h, const std::string& name, int rows, int K, const int8_t** q, const float** scb) {
  const Tensor* t = h->store.find(name);
  const Tensor* s = h->store.find(name + "_scb");
  if (!h->cfg.quantize) B200_FAIL(B200_ERR_INVALID, "lm tensor '%s' is int8 but the model was not built with quantize=True", name.c_str());
  if (!s || s->dtype != B200_F32) B200_FAIL(B200_ERR_MISSING, "lm finalize: '%s_scb' (float32 row scales of the int8 weight) was not loaded; "
                                            "care should be taken not to change its dtype (utils/quantize.py:31-35)", name.c_str());
  if (t->shape != std::vector<int64_t>{rows, K} || s->shape != std::vector<int64_t>{rows})
    B200_FAIL(B200_ERR_SHAPE, "lm tensor '%s' / its _scb: expected [%d, %d] / [%d]", name.c_str(), rows, K, rows);
  *q = static_cast<const int8_t*>(t->data);
  *scb = static_cast<const float*>(s->data);
  return B200_OK;
}

// Linear weight from the store -> packed tiles (gemm_sk.cu), which replace the row-major tensors (which are released), so the
// 15.4 GB checkpoint is resident once.  Several names: tensors of equal row counts stacked along N into one linear.
int get_linear(b200_lm* h, const std::vector<std::string>& names, int N, int K, int epi, int gate_rows, const bf16** out,
               const float** scales_out) {
  const int n = (int)names.size(), w_rows = epi == LIN_GATE ? 2 * gate_rows : N, rows = w_rows / n;
  const Tensor* t = h->store.find(names[0]);
  const bool pre = t && t->dtype == B200_I8;      // pre-quantised checkpoint: tile CB as it is, keep SCB
  const size_t el = pre ? 1 : 2;
  *scales_out = nullptr;
  struct Guard { void* p = nullptr; ~Guard() { cudaFree(p); } } stacked;      // several tensors: stacked here first
  if (n > 1) B200_CUDA(cudaMalloc(&stacked.p, (size_t)w_rows * K * el));
  float* scales = nullptr;
  if (pre) B200_TRY(h->weights.alloc_t(&scales, (size_t)w_rows, false));
  const void* w = nullptr;
  for (int i = 0; i < n; ++i) {
    if (pre) {
      const int8_t* q = nullptr; const float* scb = nullptr;
      if (!h->store.find(names[i])) B200_FAIL(B200_ERR_MISSING, "lm finalize: tensor '%s' was not loaded", names[i].c_str());
      B200_TRY(get_prequantised(h, names[i], rows, K, &q, &scb));
      B200_CUDA(cudaMemcpy(scales + (size_t)i * rows, scb, (size_t)rows * 4, cudaMemcpyDeviceToDevice));
      w = q;
    } else {
      const bf16* b = nullptr;
      B200_TRY(get_bf16(h, names[i], {rows, K}, &b));
      w = b;
    }
    if (n > 1)
      B200_CUDA(cudaMemcpy(static_cast<char*>(stacked.p) + (size_t)i * rows * K * el, w, (size_t)rows * K * el, cudaMemcpyDeviceToDevice));
  }
  if (n > 1) w = stacked.p;
  void* packed = nullptr;
  if (pre) {
    B200_TRY(h->weights.alloc(&packed, tc::sk_packed_bytes_i8(N, K, epi, gate_rows), false));
    B200_TRY(tc::sk_pack_weights_i8(static_cast<const int8_t*>(w), packed, N, K, epi, gate_rows, nullptr));
    h->weight_bytes += (int64_t)w_rows * K + (int64_t)w_rows * 4;
  } else if (h->cfg.quantize) {        // QLinear.__init__ (utils/quantize.py:16-21): row-wise absmax int8 of weight.to(float16)
    B200_TRY(h->weights.alloc(&packed, tc::sk_packed_bytes_i8(N, K, epi, gate_rows), false));
    B200_TRY(h->weights.alloc_t(&scales, (size_t)w_rows, false));
    B200_TRY(tc::sk_quant_pack_weights(static_cast<const bf16*>(w), packed, scales, N, K, epi, gate_rows, nullptr));
    h->weight_bytes -= (int64_t)w_rows * K;        // one byte per weight instead of two (get_bf16 counted two) ...
    h->weight_bytes += (int64_t)w_rows * 4;        // ... plus the row scales
  } else {
    B200_TRY(h->weights.alloc(&packed, tc::sk_packed_bytes(N, K, epi, gate_rows), false));
    B200_TRY(tc::sk_pack_weights(static_cast<const bf16*>(w), packed, N, K, epi, gate_rows, nullptr));
  }
  B200_CUDA(cudaStreamSynchronize(nullptr));
  for (const std::string& name : names) {
    h->store.release(name);
    if (pre) h->store.release(name + "_scb");
  }
  *out = static_cast<const bf16*>(packed);
  *scales_out = scales;
  return B200_OK;
}

// logits [MB][card] of the model -> the [batch][card] rows the sampler reads: the conditioned rows themselves, or (CFG) the
// guided combination written to `guided`
const bf16* guide(b200_lm* h, const bf16* logits, bf16* guided, int card, bool combine) {
  if (!cfg_on(h) || !combine) return logits;
  const long long n = (long long)h->batch * card;
  B200_LAUNCH(cfg_combine_kernel, (unsigned)ceil_div64(n, 256), 256, 0, h->body, logits, guided, h->batch, card, h->cfg_coef);
  return guided;
}

// text: the text sampler (the rows' own temp_text / top_k_text where they have them), else an audio sub-step's (temp / top_k)
int sample(b200_lm* h, const bf16* logits, int card, const float* noise, long long* out, float temp, int top_k, bool text) {
  B200_LAUNCH(sample_kernel, h->batch, SAMPLE_THREADS, 0, h->body, logits, (long long)card, noise,
              (long long)noise_per_row(h), out, card, h->use_sampling, temp, top_k, h->ss.rows(), text ? 1 : 0);
  return check_launch("sample");
}

// The step's text token from the sampler's logits [batch][text_card]: a session-sampling handle adjusts them per row and appends
// the tokens to the rows' histories
int sample_text(b200_lm* h, const bf16* logits) {
  if (!h->ss.on()) return sample(h, logits, h->cfg.text_card, h->noise, h->text_token, h->temp_text, h->top_k_text, true);
  text_rows_launch(logits, h->ss.scores, h->noise, noise_per_row(h), h->text_token, h->batch, h->cfg.text_card, h->use_sampling,
                   h->temp_text, h->top_k_text, h->ss.params, h->ss.history(), h->exec_mask, h->body);
  return check_launch("sample_text");
}

TokenRing ring(b200_lm* h) {
  TokenRing r;
  r.cache = h->cache; r.offsets = h->offsets; r.exec_mask = h->exec_mask; r.delays = h->delays_dev;
  r.Kc = h->Kc; r.CT = h->CT; r.dep_q = h->cfg.dep_q; r.n_q = h->cfg.n_q; r.card = h->cfg.card;
  r.text_card = h->cfg.text_card; r.max_delay = h->max_delay;
  r.cfg = cfg_on(h) ? 1 : 0; r.cfg_is_no_text = h->cfg_is_no_text; r.cfg_masked_until = h->cfg_until; r.err = h->err;
  return r;
}

// Taps of the temporal stack: the summed embeddings, then per layer the attention output [MB][dim], x after the attention
// residual [MB][dim], the gated hidden [MB][ffn_hidden] and x after the MLP residual [MB][dim].
// Cross-attention handles add, after those four, the cross-attention output [MB][dim] and x after the cross residual [MB][dim].
enum TapKind { TAP_ATTN_OUT, TAP_X_ATTN, TAP_GATED, TAP_X_OUT, TAP_CROSS_OUT, TAP_X_CROSS };
int64_t tap_elems(const b200_lm* h) {
  const int64_t MB = h->MB, d = h->cfg.dim;
  return MB * d + (int64_t)h->layers.size() * MB * ((h->cross.on ? 5 : 3) * d + h->cfg.ffn_hidden);
}
// first element of a tap (layer -1: the embeddings) and its element count
int64_t tap_slot(const b200_lm* h, int layer, int kind, int64_t* n) {
  const int64_t MB = h->MB, d = h->cfg.dim, F = h->cfg.ffn_hidden;
  *n = kind == TAP_GATED ? MB * F : MB * d;
  if (layer < 0) return 0;
  const int64_t at[6] = {0, MB * d, 2 * MB * d, 2 * MB * d + MB * F, 3 * MB * d + MB * F, 4 * MB * d + MB * F};
  return MB * d + (int64_t)layer * MB * ((h->cross.on ? 5 : 3) * d + F) + at[kind];
}
// device-to-device copy on the step's stream (a memcpy node of the captured graph); nothing when taps are off
int tap(b200_lm* h, const bf16* src, int layer, int kind) {
  if (!h->taps_on) return B200_OK;
  int64_t n = 0;
  const int64_t at = tap_slot(h, layer, kind, &n);
  B200_CUDA(cudaMemcpyAsync(h->taps + at, src, (size_t)n * 2, cudaMemcpyDeviceToDevice, h->body));
  return B200_OK;
}

// ---- depformer: loading and running ------------------------------------------------------------------------------------------
// An embedding table of the depformer as the step reads it, [V][dd] bf16.  Low-rank (lm_utils.py:80-124): "<name>.weight" [V][r]
// and "<name>.low_rank.weight" [dd][r] are expanded once into that table (lowrank_expand_kernel) and released.  The expansion
// is exact per token, so the step reads one row per (row, sub-step) from the same layout as a full-rank table; token -1 reads no
// row (embed_id_ok), as before.
int get_dep_table(b200_lm* h, const std::string& name, int V, int dd, int r, const bf16** out) {
  if (r == 0) return get_bf16(h, name + ".weight", {V, dd}, out);
  const bf16 *e = nullptr, *low = nullptr;
  const Tensor* lt = h->store.find(name + ".low_rank.weight");
  if (lt && lt->dtype == B200_I8)
    B200_FAIL(B200_ERR_INVALID, "lm tensor '%s.low_rank.weight' is pre-quantised (int8): low-rank factors are expanded from bf16 "
              "only; load the bf16 checkpoint with quantize=True", name.c_str());
  B200_TRY(get_bf16(h, name + ".weight", {V, r}, &e));
  B200_TRY(get_bf16(h, name + ".low_rank.weight", {dd, r}, &low));
  bf16* full = nullptr;
  B200_TRY(h->weights.alloc_t(&full, (size_t)V * dd, false));
  lowrank_expand_kernel<<<V, 256, (size_t)r * sizeof(float)>>>(e, low, full, r, dd, h->cfg.quantize);
  B200_TRY(check_launch("lowrank_expand"));
  B200_CUDA(cudaStreamSynchronize(nullptr));
  h->store.release(name + ".weight");
  h->store.release(name + ".low_rank.weight");
  h->weight_bytes += ((int64_t)V * dd - (int64_t)V * r - (int64_t)dd * r) * 2;     // the table instead of its factors
  *out = full;
  return B200_OK;
}

int Depformer::load(b200_lm* h) {
  if (dep_q == 0) return B200_OK;
  std::vector<std::string> in_names;
  for (int j = 0; j < n_sets; ++j) in_names.push_back("depformer_in." + std::to_string(j) + ".weight");
  B200_TRY(get_linear(h, in_names, n_sets * dd, h->cfg.dim, LIN_STORE, 0, &in_all, &in_s));
  tables.resize(dep_q); heads.resize(dep_q); heads_s.resize(dep_q); w.resize((size_t)dep_q * L); n1.resize(L); n2.resize(L);
  B200_TRY(get_dep_table(h, "depformer_text_emb", text_card + 1, dd, low_rank, &tables[0]));
  for (int k = 1; k < dep_q; ++k)
    B200_TRY(get_dep_table(h, "depformer_emb." + std::to_string(k - 1), card + 1, dd, low_rank, &tables[k]));
  for (int k = 0; k < dep_q; ++k)
    B200_TRY(get_linear(h, {"linears." + std::to_string(k) + ".weight"}, card, dd, LIN_STORE, 0, &heads[k], &heads_s[k]));
  std::vector<Step> sets((size_t)n_sets);      // one layer's weight sets, each packed once
  for (int l = 0; l < L; ++l) {
    const std::string p = "depformer.layers." + std::to_string(l);
    for (int j = 0; j < n_sets; ++j) {
      const std::string ks = std::to_string(j);
      Step& S = sets[j];
      B200_TRY(get_linear(h, {p + ".self_attn.in_projs." + ks + ".weight"}, 3 * dd, dd, LIN_STORE, 0, &S.in_w, &S.in_s));
      B200_TRY(get_linear(h, {p + ".self_attn.out_projs." + ks + ".weight"}, dd, dd, LIN_RESADD, 0, &S.out_w, &S.out_s));
      B200_TRY(get_linear(h, {p + ".gating." + ks + ".linear_in.weight"}, 2 * F, dd, LIN_GATE, F, &S.lin_in, &S.lin_in_s));
      B200_TRY(get_linear(h, {p + ".gating." + ks + ".linear_out.weight"}, dd, F, LIN_RESADD, 0, &S.lin_out, &S.lin_out_s));
    }
    for (int k = 0; k < dep_q; ++k) w[(size_t)k * L + l] = sets[sched[k]];
    B200_TRY(get_bf16(h, p + ".norm1.alpha", {1, 1, dd}, &n1[l]));
    B200_TRY(get_bf16(h, p + ".norm2.alpha", {1, 1, dd}, &n2[l]));
  }
  return B200_OK;
}

// streaming_begin, after linear_init: the persistent kernel's buffers and the kernel itself, where the plan takes it
int Depformer::alloc_fused(b200_lm* h) {
  if (plan.path != tc::DEP_FUSED) return B200_OK;
  Arena& A = h->state;
  B200_TRY(A.alloc_t(&part0, (size_t)plan.part_floats, false));
  B200_TRY(A.alloc_t(&part1, (size_t)plan.part_floats, false));
  B200_TRY(A.alloc_t(&bar, 1));
  if (const char* e = getenv("B200_DEP_TRACE")) {
    if (atoi(e)) B200_TRY(A.alloc_t(&trace, (size_t)tc::DEP_TRACE_SLOTS));
  }
  std::vector<tc::DepLayerW> lw;
  for (const Step& S : w)
    lw.push_back({reinterpret_cast<const uint8_t*>(S.in_w), reinterpret_cast<const uint8_t*>(S.out_w),
                  reinterpret_cast<const uint8_t*>(S.lin_in), reinterpret_cast<const uint8_t*>(S.lin_out)});
  tc::DepParams p{};
  p.B = B; p.dd = dd; p.H = H; p.F = F; p.card = card; p.text_card = text_card; p.dep_q = dep_q; p.L = L; p.err = h->err;
  p.w = lw.data(); p.heads = reinterpret_cast<const uint8_t* const*>(heads.data()); p.tables = tables.data();
  p.n1 = n1.data(); p.n2 = n2.data(); p.kc = kc.data(); p.vc = vc.data();
  std::vector<int> cols(dep_q);
  for (int k = 0; k < dep_q; ++k) cols[k] = din_col(k);
  p.din = din; p.din_ld = din_ld(); p.din_col = cols.data(); p.text_token = h->text_token;
  p.x = dx; p.xn = dxn; p.ao = dao; p.hbuf = dh; p.part0 = part0; p.part1 = part1;
  p.logits = logits; p.audio_tokens = h->audio_tokens;
  p.noise = h->noise; p.noise_ld = noise_at(dep_q); p.noise_off = (int)noise_at(0); p.ka = ka;
  p.use_sampling = h->use_sampling; p.top_k = h->top_k; p.temp = h->temp;
  p.rows = h->ss.rows();
  p.bar = bar; p.trace = trace;
  return tc::dep_fused_create(plan, p, &fused);
}

// The step from the depformer's input projection to the last sub-step's sampler (lm.py:809-850): fresh K / V every frame, all
// rows advance together.  replace: depformer_replace_tokens (lm.py:751-755), the caller supplies this frame's audio tokens and the
// depformer does not run; without a depformer (dep_q = 0, lm.py:219-222, "No-Depformer --- e.g., an ASR model") nothing runs.
int Depformer::run(b200_lm* h, bool replace) {
  cudaStream_t st = h->body;
  if (replace || plan.path == tc::DEP_NONE) {
    if (dep_q > 0) B200_LAUNCH(replace_audio_kernel, ceil_div(B * dep_q, 128), 128, 0, st, h->replace_tokens, h->audio_tokens, B, dep_q);
    return B200_OK;
  }
  const int d = h->cfg.dim;
  B200_TRY(linear(h, h->tout, d, in_all, din, din_ld(), nullptr, 0, MB, n_sets * dd, d, LIN_STORE, 0, in_s));
  if (plan.path == tc::DEP_FUSED) return tc::dep_fused_launch(fused, st);
  for (int k = 0; k < dep_q; ++k) {
    const long long* prev = k == 0 ? h->text_token : h->audio_tokens + (long long)(k - 1) * B;
    B200_LAUNCH(dep_input_kernel, ceil_div(MB * dd, 256), 256, 0, st, din, din_ld(), din_col(k), tables[k], prev, dx, MB, dd, B,
                k == 0 ? text_card : card, h->err);
    for (int l = 0; l < L; ++l) {
      const Step& S = w[(size_t)k * L + l];
      B200_TRY(norm_linear(h, dx, n1[l], dxn, S.in_w, dqkv, 3 * dd, MB, 3 * dd, dd, LIN_STORE, 0, S.in_s));
      B200_LAUNCH(dep_attn_step_kernel, ceil_div(MB * H * 32, 128), 128, 0, st, dqkv, kc[l], vc[l], dao, MB, H, dep_q, k);
      B200_TRY(linear(h, dao, dd, S.out_w, dx, dd, dx, dd, MB, dd, dd, LIN_RESADD, 0, S.out_s));
      B200_TRY(norm_linear(h, dx, n2[l], dxn, S.lin_in, dh, F, MB, F, dd, LIN_GATE, F, S.lin_in_s));
      B200_TRY(linear(h, dh, F, S.lin_out, dx, dd, dx, dd, MB, dd, F, LIN_RESADD, 0, S.lin_out_s));
    }
    bf16* lg = logits + (long long)k * MB * card;
    B200_TRY(linear(h, dx, dd, heads[k], lg, card, nullptr, 0, MB, card, dd, LIN_STORE, 0, heads_s[k]));
    const bf16* gl = guide(h, lg, cfg_on(h) ? logits_cfg + (long long)k * B * card : nullptr, card, true);   // lm.py:828-833
    B200_TRY(sample(h, gl, card, h->noise + noise_at(k), h->audio_tokens + (long long)k * B, h->temp, h->top_k, false));
  }
  return B200_OK;
}

// ---- cross-attention: loading, fill and step ----------------------------------------------------------------------------------
// Layer l's weights (transformer.py:495-505, 727-732): in_projs.0 rows [0, d) packed as the query linear, rows [d, 3d) as one
// [2d, d] K|V linear of the condition, out_projs.0 as a RESADD linear; norm_cross weight and bias.
int CrossAttention::load(b200_lm* h, int l) {
  if (!on) return B200_OK;
  const std::string p = "transformer.layers." + std::to_string(l);
  Layer& L = layers[l];
  const std::string x = p + ".cross_attention.in_projs.0.weight";
  const bf16* w = nullptr;
  B200_TRY(get_bf16(h, x, {3 * d, d}, &w));
  auto pack = [&](const bf16* rows, int N, const bf16** out) -> int {     // a slice of the loaded tensor -> packed tiles
    void* packed = nullptr;
    B200_TRY(h->weights.alloc(&packed, tc::sk_packed_bytes(N, d, LIN_STORE, 0), false));
    B200_TRY(tc::sk_pack_weights(rows, packed, N, d, LIN_STORE, 0, nullptr));
    *out = static_cast<const bf16*>(packed);
    return B200_OK;
  };
  B200_TRY(pack(w, d, &L.q_w));
  B200_TRY(pack(w + (size_t)d * d, 2 * d, &L.kv_w));
  B200_CUDA(cudaStreamSynchronize(nullptr));
  h->store.release(x);
  const float* no_scales = nullptr;
  B200_TRY(get_linear(h, {p + ".cross_attention.out_projs.0.weight"}, d, d, LIN_RESADD, 0, &L.out_w, &no_scales));
  B200_TRY(get_bf16(h, p + ".norm_cross.weight", {d}, &L.nw));
  return get_bf16(h, p + ".norm_cross.bias", {d}, &L.nb);
}

// b200_lm_set_condition_cross, outside the step (transformer.py:495-505 per layer): kv = src @ Wkv^T in chunks of rows, then
// "b t (p h d) -> p b h t d" into the rows' memory.  The chunk is staged in a fixed buffer so that the GEMM's activation plan is
// the same every call.
int CrossAttention::fill(b200_lm* h, const void* src, const int32_t* rows_host, int n_rows) const {
  if (!on) B200_FAIL(B200_ERR_INVALID, "lm_set_condition_cross: the model has no cross-attention layers");
  if (!src || n_rows < 1 || n_rows > MB) B200_FAIL(B200_ERR_INVALID, "lm_set_condition_cross: %d condition rows", n_rows);
  if (!rows_host && n_rows != MB)       // lm.py:650-651: "cfg requires 2x more conditions"
    B200_FAIL(B200_ERR_SHAPE, "lm_set_condition_cross: %d rows given, the model runs on %d", n_rows, MB);
  std::vector<int> rows(n_rows);
  for (int k = 0; k < n_rows; ++k) {
    rows[k] = rows_host ? rows_host[k] : k;
    if (rows[k] < 0 || rows[k] >= MB) B200_FAIL(B200_ERR_INVALID, "lm_set_condition_cross: model row %d outside [0, %d)", rows[k], MB);
  }
  B200_CUDA(cudaMemcpyAsync(rows_dev, rows.data(), rows.size() * 4, cudaMemcpyHostToDevice, h->stream));
  B200_TRY(tc::linear_prepare());
  h->body = h->stream;
  const long long total = (long long)n_rows * T;
  for (long long i0 = 0; i0 < total; i0 += CROSS_CHUNK) {
    const int n = (int)std::min<long long>(CROSS_CHUNK, total - i0);
    B200_CUDA(cudaMemcpyAsync(chunk, static_cast<const bf16*>(src) + i0 * d, (size_t)n * d * 2, cudaMemcpyDeviceToDevice, h->stream));
    for (const Layer& L : layers) {
      B200_TRY(linear(h, chunk, d, L.kv_w, chunk_kv, 2 * d, nullptr, 0, n, 2 * d, d, LIN_STORE, 0));
      B200_LAUNCH(cross_kv_scatter_kernel, (unsigned)ceil_div64((long long)n * 2 * H * (ATT_D / 8), 256), 256, 0, h->stream, chunk_kv,
                  i0, n, rows_dev, L.k, L.v, H, T);
    }
  }
  return check_launch("lm_set_condition_cross");
}

// Layer l's block between its self-attention and its MLP: x = x + cross_attention(norm_cross(x), memory) (transformer.py:779-798)
int CrossAttention::step(b200_lm* h, int l) const {
  if (!on) return B200_OK;
  const Layer& L = layers[l];
  B200_LAUNCH(layernorm_kernel, MB, 256, 0, h->body, h->x, L.nw, L.nb, h->xn, d, 1e-5f);
  B200_TRY(linear(h, h->xn, d, L.q_w, h->qkv, d, nullptr, 0, MB, d, d, LIN_STORE, 0));
  cross_attn_launch(h->qkv, d, L.k, L.v, h->ao, h->attn_part, h->attn_counters, MB, H, T, nsplit, h->body);
  B200_TRY(tap(h, h->ao, l, TAP_CROSS_OUT));
  B200_TRY(linear(h, h->ao, d, L.out_w, h->x, d, h->x, d, MB, d, d, LIN_RESADD, 0));
  return tap(h, h->x, l, TAP_X_CROSS);
}

// The whole frame as a fixed launch sequence over static buffers (captured into one CUDA graph).
int step_body(b200_lm* h) {
  const auto& c = h->cfg;
  const int B = h->batch, MB = h->MB, d = c.dim, H = c.num_heads, F = c.ffn_hidden;
  cudaStream_t st = h->body;

  B200_LAUNCH(lm_prepare_kernel, ceil_div(B * h->Kc, 128), 128, 0, st, ring(h), h->in_codes, h->n_in_static,
              h->input_tokens, B);
  {
    EmbedTables t = h->emb;
    t.condition_sum = h->cond_on ? h->cond_sum : nullptr;
    t.err = h->err;
    B200_LAUNCH(lm_embed_sum_kernel, ceil_div(MB * d / 2, 256), 256, 0, st, t, h->input_tokens, h->x, MB, d);
  }
  B200_TRY(tap(h, h->x, -1, 0));
  if (h->noise_static) {
    const long long n = (long long)B * noise_per_row(h);
    B200_LAUNCH(lm_noise_kernel, (unsigned)ceil_div64(ceil_div64(n, 4), 256), 256, 0, st, h->noise, n, h->noise_seed, h->noise_ctr);
  }
  h->kv.prologue(h->exec_mask_m, h->err, st);
  for (size_t l = 0; l < h->layers.size(); ++l) {
    const TLayer& L = h->layers[l];
    B200_TRY(norm_linear(h, h->x, L.n1, h->xn, L.in_w, h->qkv, 3 * d, MB, 3 * d, d, LIN_STORE, 0, L.in_s));
    // RoPE + ring append + split-KV attention + split merge in one launch
    attn_step_launch(h->qkv, h->kv.rings((int)l), h->ao, h->attn_part, h->attn_counters, h->pos, h->exec_mask_m, MB, H, h->kv.cap,
                     h->nsplit, c.max_period, h->kv.kind, st);
    B200_TRY(tap(h, h->ao, (int)l, TAP_ATTN_OUT));
    B200_TRY(linear(h, h->ao, d, L.out_w, h->x, d, h->x, d, MB, d, d, LIN_RESADD, 0, L.out_s));
    B200_TRY(tap(h, h->x, (int)l, TAP_X_ATTN));
    B200_TRY(h->cross.step(h, (int)l));
    B200_TRY(norm_linear(h, h->x, L.n2, h->xn, L.lin_in, h->hbuf, F, MB, F, d, LIN_GATE, F, L.lin_in_s));
    B200_TRY(tap(h, h->hbuf, (int)l, TAP_GATED));
    B200_TRY(linear(h, h->hbuf, F, L.lin_out, h->x, d, h->x, d, MB, d, F, LIN_RESADD, 0, L.lin_out_s));
    B200_TRY(tap(h, h->x, (int)l, TAP_X_OUT));
  }
  B200_LAUNCH(rmsnorm_kernel, MB, 256, 0, st, h->x, h->out_norm, h->tout, d, 1e-8f);
  B200_TRY(linear(h, h->tout, d, h->text_linear, h->text_logits, c.text_card, nullptr, 0, MB, c.text_card, d, LIN_STORE, 0, h->text_linear_s));
  // lm.py:728-732: with cfg_is_no_text the text logits are the conditioned rows, otherwise the guided combination
  const bf16* tl = guide(h, h->text_logits, h->text_logits_cfg, c.text_card, !h->cfg_is_no_text);
  B200_TRY(sample_text(h, tl));
  if (!h->extra_w.empty())
    B200_LAUNCH(extra_heads_kernel, ceil_div((int)h->extra_w.size() * MB * 32, 128), 128, 0, st, h->tout, h->extra_w_dev, h->extra_out, MB, d,
                c.extra_heads_dim, (int)h->extra_w.size());

  B200_TRY(h->dep.run(h, h->replace_static != 0));
  B200_LAUNCH(advance_pos_kernel, ceil_div(MB, 128), 128, 0, st, h->pos, h->exec_mask_m, MB);
  B200_LAUNCH(lm_finish_kernel, ceil_div(B, 128), 128, 0, st, ring(h), h->text_token, h->audio_tokens, h->out_tokens, B, h->noise_ctr);
  return check_launch("lm step");
}

// ---- session records (b200_lm_session_*) ----------------------------------------------------------------------------------
// After the 256-byte SessionHeader: the session's slices of exec_mask, cache, offsets, model.offset (1 or 2 rows), under CFG
// model.exec_mask (2 rows) and cfg_is_masked_until, and while it is on the condition_sum rows, each 16-byte aligned (the
// RowSlice table of streaming_begin).  From the next 256-byte boundary, the temporal K/V of slots [0, n), n = min(pos, ring
// capacity), slot s being position s mod capacity (TemporalKv::record).  A cross-attention handle's record continues with the
// session's condition memory (CrossAttention::record_section), a session-sampling handle's ends with the session's settings and
// text history (SessionSampling::record_section).
struct SessionPlan {
  int rows = 1;
  int64_t pos[2] = {0, 0};
  int64_t n = 0, kv_off = 0, cross_off = 0, ss_off = 0, bytes = 0;
  bool cond = false;
};

void session_size(const b200_lm* h, SessionPlan* p) {
  const long long end = p->cond ? h->slices_end_cond : h->slices_end;
  p->kv_off = (end + 255) / 256 * 256;
  p->bytes = h->ss.record_section(h->cross.record_section(p->kv_off + h->kv.record_bytes(p->rows, p->n), p->rows, &p->cross_off),
                                  &p->ss_off);
}

// The record row `row` would export now (synchronises): B200_ERR_STATE for a short-ring row whose ring has already wrapped.
int session_plan(b200_lm* h, int row, const char* what, SessionPlan* p) {
  B200_TRY(h->check_row(row, what));
  p->rows = h->MB / h->batch;
  B200_CUDA(cudaStreamSynchronize(h->stream));
  for (int k = 0; k < p->rows; ++k)
    B200_CUDA(cudaMemcpy(&p->pos[k], h->pos + row + (size_t)k * h->batch, 8, cudaMemcpyDeviceToHost));
  const int64_t top = std::max(p->pos[0], p->pos[1]);
  B200_TRY(h->kv.check_history(top, what));
  p->n = std::min<int64_t>(top, h->kv.cap);
  p->cond = h->cond_on != 0;
  session_size(h, p);
  return B200_OK;
}

// The session's temporal K/V and condition memory between the device and the record
int session_kv(b200_lm* h, int row, const SessionPlan& p, char* rec, bool gather) {
  B200_TRY(h->kv.record(row, p.rows, h->batch, (int)p.n, rec + p.kv_off, gather, h->stream));
  B200_TRY(h->cross.record(row, p.rows, h->batch, rec + p.cross_off, gather, h->stream));
  return h->ss.record(row, rec + p.ss_off, gather, h->stream);
}

}  // namespace

int b200_lm::copy_entry(const StateEntry& e, void* dst, const void* src) {
  const int arr = kv.paged_array(e.ptr);
  return arr < 0 ? StreamCore::copy_entry(e, dst, src) : kv.copy_entry(arr, dst, src, stream);
}

namespace b200 {
int lm_check_kv_pool(b200_lm* h) {
  if (!h || h->batch <= 0) return B200_OK;
  DeviceGuard g(h->device);
  return h->kv.check_pool_flag(h->err, "frame_step", h->stream);
}

int lm_frame_view(b200_lm* h, LmFrameView* v) {
  B200_TRY(check_streaming(h, "lm_frame_view"));
  const auto& c = h->cfg;
  *v = LmFrameView{h->batch, h->MB, c.n_q, c.dep_q, h->max_delay, (int)h->extra_w.size(), c.extra_heads_dim, h->extra_out};
  return B200_OK;
}

int lm_device(const b200_lm* h) { return h->device; }
}  // namespace b200

extern "C" {

int b200_lm_create(const b200_lm_config* cfg, b200_lm** out) {
  if (!cfg || !out) B200_FAIL(B200_ERR_INVALID, "lm_create: null argument");
  if (cfg->n_q < 1 || cfg->n_q > 32 || cfg->dep_q < 0 || cfg->dep_q > cfg->n_q || cfg->dep_q > DEP_MAX_Q)
    B200_FAIL(B200_ERR_INVALID, "lm_create: n_q=%d dep_q=%d unsupported (n_q <= 32, dep_q <= %d)", cfg->n_q, cfg->dep_q, DEP_MAX_Q);
  if (cfg->extra_heads_num_heads < 0 || cfg->extra_heads_num_heads > 8 || (cfg->extra_heads_num_heads > 0 && (cfg->extra_heads_dim < 1 || cfg->extra_heads_dim > 32)))
    B200_FAIL(B200_ERR_INVALID, "lm_create: extra heads %d x %d unsupported (<= 8 heads of <= 32 outputs)", cfg->extra_heads_num_heads, cfg->extra_heads_dim);
  if (cfg->dim % cfg->num_heads || cfg->dim / cfg->num_heads != ATT_D)
    B200_FAIL(B200_ERR_INVALID, "lm_create: temporal head dim must be %d", ATT_D);
  if (cfg->dep_q > 0 && (cfg->depformer_dim % cfg->depformer_num_heads || cfg->depformer_dim / cfg->depformer_num_heads != 64))
    B200_FAIL(B200_ERR_INVALID, "lm_create: depformer head dim must be 64");
  if (cfg->dim % 8 || cfg->ffn_hidden % 8 || (cfg->dep_q > 0 && (cfg->depformer_dim % 8 || cfg->depformer_ffn_hidden % 8)))
    B200_FAIL(B200_ERR_INVALID, "lm_create: feature sizes must be multiples of 8");
  if (cfg->text_card + 1 > 65535 || cfg->card + 1 > 65535)
    B200_FAIL(B200_ERR_INVALID, "lm_create: vocabularies above 65535 unsupported by the sampler");
  b200_lm* h = new b200_lm();
  h->cfg = *cfg;
  cudaGetDevice(&h->device);
  h->session_kind = SESSION_LM;
  h->fingerprint = config_fingerprint(&h->cfg, sizeof(h->cfg));
  h->Kc = cfg->n_q + 1;
  h->max_delay = 0;
  for (int k = 0; k < h->Kc; ++k) h->max_delay = cfg->delays[k] > h->max_delay ? cfg->delays[k] : h->max_delay;
  h->CT = h->max_delay + 2;     // lm.py:606-611
  if (const char* e = getenv("B200_PDL")) h->pdl = atoi(e) != 0;
  h->kv.context = cfg->context;
  h->kv.H = cfg->num_heads;
  h->dep.configure(*cfg);
  h->dep.set_sampling(h->use_sampling, h->temp, h->top_k, h->top_k_text);
  if (const char* e = getenv("B200_KV_DTYPE")) {
    const std::string v = e;
    h->kv.kind = (v == "fp8" || v == "fp8_e4m3") ? B200_KV_FP8_E4M3 : v == "int8" ? B200_KV_INT8 : B200_KV_BF16;
  }
  *out = h;
  return B200_OK;
}

int b200_lm_load_tensor(b200_lm* h, const char* name, const void* data_dev, int dtype, int ndim, const int64_t* shape) {
  if (!h) B200_FAIL(B200_ERR_INVALID, "lm_load_tensor: null handle");
  if (h->finalized) B200_FAIL(B200_ERR_STATE, "lm_load_tensor: already finalized");
  DeviceGuard g(h->device);
  return h->store.put(name, data_dev, dtype, ndim, shape);
}

int b200_lm_finalize(b200_lm* h) {
  if (!h) B200_FAIL(B200_ERR_INVALID, "lm_finalize: null handle");
  if (h->finalized) return B200_OK;
  const auto& c = h->cfg;
  const int d = c.dim, F = c.ffn_hidden;
  h->emb.n_q = c.n_q; h->emb.card = c.card; h->emb.text_card = c.text_card; h->emb.condition_sum = nullptr; h->emb.err = nullptr;
  DeviceGuard guard_dev(h->device);
  for (int k = 0; k < c.n_q; ++k)
    B200_TRY(get_bf16(h, "emb." + std::to_string(k) + ".weight", {c.card + 1, d}, &h->emb.audio[k]));
  B200_TRY(get_bf16(h, "text_emb.weight", {c.text_card + 1, d}, &h->emb.text));
  B200_TRY(get_linear(h, {"text_linear.weight"}, c.text_card, d, LIN_STORE, 0, &h->text_linear, &h->text_linear_s));
  B200_TRY(get_bf16(h, "out_norm.alpha", {1, 1, d}, &h->out_norm));
  h->layers.resize(c.num_layers);
  for (int l = 0; l < c.num_layers; ++l) {
    const std::string p = "transformer.layers." + std::to_string(l);
    TLayer& L = h->layers[l];
    B200_TRY(get_linear(h, {p + ".self_attn.in_projs.0.weight"}, 3 * d, d, LIN_STORE, 0, &L.in_w, &L.in_s));
    B200_TRY(get_linear(h, {p + ".self_attn.out_projs.0.weight"}, d, d, LIN_RESADD, 0, &L.out_w, &L.out_s));
    B200_TRY(get_bf16(h, p + ".norm1.alpha", {1, 1, d}, &L.n1));
    B200_TRY(get_bf16(h, p + ".norm2.alpha", {1, 1, d}, &L.n2));
    B200_TRY(get_linear(h, {p + ".gating.linear_in.weight"}, 2 * F, d, LIN_GATE, F, &L.lin_in, &L.lin_in_s));
    B200_TRY(get_linear(h, {p + ".gating.linear_out.weight"}, d, F, LIN_RESADD, 0, &L.lin_out, &L.lin_out_s));
    B200_TRY(h->cross.load(h, l));
  }
  for (int i = 0; i < c.extra_heads_num_heads; ++i) {      // lm.py:224-226
    const bf16* w = nullptr;
    B200_TRY(get_bf16(h, "extra_heads." + std::to_string(i) + ".weight", {c.extra_heads_dim, d}, &w));
    h->extra_w.push_back(w);
  }
  if (!h->extra_w.empty()) {
    B200_TRY(h->weights.alloc_t(&h->extra_w_dev, h->extra_w.size(), false));
    B200_CUDA(cudaMemcpy(h->extra_w_dev, h->extra_w.data(), h->extra_w.size() * sizeof(void*), cudaMemcpyHostToDevice));
  }
  B200_TRY(h->dep.load(h));
  B200_TRY(h->weights.alloc_t(&h->delays_dev, h->Kc, false));
  B200_CUDA(cudaMemcpy(h->delays_dev, c.delays, h->Kc * sizeof(int), cudaMemcpyHostToDevice));
  B200_CUDA(cudaDeviceSynchronize());
  h->finalized = true;
  return B200_OK;
}

int b200_lm_destroy(b200_lm* h) {
  if (!h) return B200_OK;
  DeviceGuard g(h->device);
  b200_lm_streaming_end(h);
  h->store.release_all();
  h->weights.free_all();
  delete h;
  return B200_OK;
}

int b200_lm_set_sampling(b200_lm* h, int use_sampling, float temp, float temp_text, int top_k, int top_k_text) {
  if (!h) B200_FAIL(B200_ERR_INVALID, "lm_set_sampling: null handle");
  if (top_k < 1 || top_k_text < 1 || top_k > SAMPLE_MAX_K || top_k_text > SAMPLE_MAX_K)
    B200_FAIL(B200_ERR_INVALID, "lm_set_sampling: top_k must be in [1, %d]", SAMPLE_MAX_K);
  if (h->batch > 0 && (top_k != h->top_k || top_k_text != h->top_k_text))
    B200_FAIL(B200_ERR_STATE, "lm_set_sampling: top_k cannot change while streaming");
  if (use_sampling == h->use_sampling && temp == h->temp && temp_text == h->temp_text && top_k == h->top_k && top_k_text == h->top_k_text)
    return B200_OK;
  h->use_sampling = use_sampling; h->temp = temp; h->temp_text = temp_text; h->top_k = top_k; h->top_k_text = top_k_text;
  h->dep.set_sampling(use_sampling, temp, top_k, top_k_text);
  h->graphs[0].drop();         // the sampling parameters are kernel arguments of the captured step
  return B200_OK;
}

int b200_lm_noise_per_row(b200_lm* h) { return h ? noise_per_row(h) : 0; }

int b200_lm_set_session_sampling(b200_lm* h, int history) {
  if (!h) B200_FAIL(B200_ERR_INVALID, "lm_set_session_sampling: null handle");
  return h->ss.set(history, h->batch > 0);
}

int b200_lm_set_row_sampling(b200_lm* h, const int32_t* rows, int n, const b200_row_sampling* p) {
  B200_STREAMING_ENTRY(h, "lm_set_row_sampling");
  return h->ss.set_rows(rows, n, p, h->top_k, h->top_k_text, h->stream);
}

int b200_lm_set_graph(b200_lm* h, int enable) {
  if (!h) B200_FAIL(B200_ERR_INVALID, "lm_set_graph: null handle");
  h->set_graph(enable);
  return B200_OK;
}

int b200_lm_set_depformer(b200_lm* h, int mode) {
  if (!h) B200_FAIL(B200_ERR_INVALID, "lm_set_depformer: null handle");
  if (h->batch > 0) B200_FAIL(B200_ERR_STATE, "lm_set_depformer: the depformer's path is planned at streaming_begin; set it before");
  if (mode < B200_DEPFORMER_AUTO || mode > B200_DEPFORMER_FUSED) B200_FAIL(B200_ERR_INVALID, "lm_set_depformer: unknown mode %d", mode);
  h->dep.mode = mode;
  return B200_OK;
}

int b200_lm_set_cfg(b200_lm* h, float cfg_coef, int cfg_is_no_text, const int64_t* masked_until_host, int n) {
  if (!h) B200_FAIL(B200_ERR_INVALID, "lm_set_cfg: null handle");
  if (h->batch > 0) B200_FAIL(B200_ERR_STATE, "lm_set_cfg: classifier-free guidance doubles the model's rows; set it before streaming_begin");
  if (masked_until_host && n < 1) B200_FAIL(B200_ERR_INVALID, "lm_set_cfg: empty cfg_is_masked_until");
  h->cfg_coef = cfg_coef;
  h->cfg_is_no_text = cfg_is_no_text ? 1 : 0;
  h->cfg_until_host.clear();
  if (masked_until_host) h->cfg_until_host.assign(masked_until_host, masked_until_host + n);
  return B200_OK;
}

int b200_lm_seed_noise(b200_lm* h, uint64_t seed) {
  if (!h) B200_FAIL(B200_ERR_INVALID, "lm_seed_noise: null handle");
  h->noise_seed = seed;
  DeviceGuard g(h->device);
  if (h->noise_ctr) B200_CUDA(cudaMemsetAsync(h->noise_ctr, 0, 8, h->stream));
  h->graphs[0].drop();         // the seed is a kernel argument of the captured step
  return B200_OK;
}

int b200_lm_set_stream(b200_lm* h, void* stream) {
  B200_STREAMING_ENTRY(h, "lm_set_stream");
  h->stream = static_cast<cudaStream_t>(stream);
  return B200_OK;
}

int b200_lm_streaming_begin(b200_lm* h, int batch, void* stream) {
  B200_TRY(check_begin(h, batch, "lm_streaming_begin"));
  DeviceGuard guard_dev(h->device);
  const auto& c = h->cfg;
  const bool cfg = cfg_on(h);
  const int B = batch, MB = cfg ? 2 * batch : batch, d = c.dim, H = c.num_heads;
  if (MB > 256) B200_FAIL(B200_ERR_INVALID, "lm_streaming_begin: %d model rows (the linears take at most 256)", MB);
  if (cfg && !h->cfg_until_host.empty() && (int)h->cfg_until_host.size() != B)      // lm.py:717 view(-1, 1, 1) broadcast
    B200_FAIL(B200_ERR_SHAPE, "lm_streaming_begin: cfg_is_masked_until has %zu entries for %d sessions", h->cfg_until_host.size(), B);
  h->stream = static_cast<cudaStream_t>(stream);
  Arena& A = h->state;
  struct Cleanup { b200_lm* h; bool armed = true; ~Cleanup() { if (armed) b200_lm_streaming_end(h); } } cleanup{h};
  size_t free_b = 0, total_b = 0;
  cudaMemGetInfo(&free_b, &total_b);
  B200_TRY(h->kv.plan(MB, c.num_layers));
  B200_TRY(h->cross.plan(MB));
  const size_t kv_bytes = h->kv.bytes() + h->cross.bytes(MB);
  if (kv_bytes + (1ull << 30) > free_b)
    B200_FAIL(B200_ERR_INVALID, "lm_streaming_begin: %d sessions need %.1f GB of KV ring, %.1f GB free", B, kv_bytes / 1e9,
              free_b / 1e9);
  B200_TRY(A.alloc_t(&h->exec_mask, B, false));
  B200_CUDA(cudaMemset(h->exec_mask, 1, B));
  if (cfg) {
    B200_TRY(A.alloc_t(&h->exec_mask_m, MB, false));
    B200_CUDA(cudaMemset(h->exec_mask_m, 1, MB));
  } else {
    h->exec_mask_m = h->exec_mask;
  }
  B200_TRY(A.alloc_t(&h->err, 1));
  B200_TRY(A.alloc_t(&h->noise_ctr, 1));
  h->cfg_until = nullptr;
  if (cfg && !h->cfg_until_host.empty()) {
    B200_TRY(A.alloc_t(&h->cfg_until, B, false));
    B200_CUDA(cudaMemcpy(h->cfg_until, h->cfg_until_host.data(), (size_t)B * 8, cudaMemcpyHostToDevice));
  }
  B200_TRY(A.alloc_t(&h->cache, (size_t)B * h->Kc * h->CT, false));
  {
    std::vector<long long> init((size_t)B * h->Kc * h->CT, -2);   // ungenerated_token_id, lm.py:606-611
    B200_CUDA(cudaMemcpy(h->cache, init.data(), init.size() * 8, cudaMemcpyHostToDevice));
  }
  B200_TRY(A.alloc_t(&h->offsets, B));
  B200_TRY(A.alloc_t(&h->pos, MB));
  h->kv.pos = h->pos;
  h->offset_cpu = 0;
  for (int l = 0; l < c.num_layers; ++l) {
    B200_TRY(h->kv.alloc_layer(A, l));
    B200_TRY(h->cross.alloc_layer(A, l));
  }
  B200_TRY(h->cross.alloc_fill(A));
  B200_TRY(h->kv.alloc_pages(A));
  B200_TRY(h->dep.begin(A, B, cfg, c.quantize != 0));
  const int n_in_max = c.n_q;   // callers may pass more columns than needed (lm.py:688-689)
  const int dq1 = c.dep_q > 0 ? c.dep_q : 1;
  B200_TRY(A.alloc_t(&h->in_codes, (size_t)B * n_in_max));
  B200_TRY(A.alloc_t(&h->input_tokens, (size_t)MB * h->Kc));
  B200_TRY(A.alloc_t(&h->text_token, B));
  B200_TRY(A.alloc_t(&h->audio_tokens, (size_t)B * dq1));
  B200_TRY(A.alloc_t(&h->replace_tokens, (size_t)B * dq1));
  B200_TRY(A.alloc_t(&h->out_tokens, (size_t)B * (c.dep_q + 1)));
  B200_TRY(h->ss.alloc(A, B, c.text_card));
  B200_TRY(A.alloc_t(&h->noise, (size_t)B * noise_per_row(h), false));
  {
    std::vector<float> ones((size_t)B * noise_per_row(h), 1.f);
    B200_CUDA(cudaMemcpy(h->noise, ones.data(), ones.size() * 4, cudaMemcpyHostToDevice));
  }
  B200_TRY(A.alloc_t(&h->x, (size_t)MB * d));
  B200_TRY(A.alloc_t(&h->xn, (size_t)MB * d));
  B200_TRY(A.alloc_t(&h->qkv, (size_t)MB * 3 * d));
  B200_TRY(A.alloc_t(&h->ao, (size_t)MB * d));
  B200_TRY(A.alloc_t(&h->hbuf, (size_t)MB * c.ffn_hidden));
  B200_TRY(A.alloc_t(&h->tout, (size_t)MB * d));
  B200_TRY(A.alloc_t(&h->cond_sum, (size_t)MB * d));
  h->cond_on = 0;
  B200_TRY(A.alloc_t(&h->text_logits, (size_t)MB * c.text_card));
  if (cfg) {
    B200_TRY(A.alloc_t(&h->text_logits_cfg, (size_t)B * c.text_card));
    B200_TRY(h->dep.alloc_guided(A));
  }
  if (!h->extra_w.empty()) B200_TRY(A.alloc_t(&h->extra_out, h->extra_w.size() * (size_t)MB * c.extra_heads_dim));
  B200_TRY(h->dep.alloc_activations(A));
  B200_TRY(A.alloc(reinterpret_cast<void**>(&h->sk_ws), tc::sk_workspace_bytes(std::max(MB, h->cross.max_m())), false));
  B200_TRY(A.alloc_t(&h->sk_counters, tc::SK_MAX_TILES));
  const int ns = attn_pick_splits(MB, H, h->kv.cap);
  h->nsplit = ns;
  B200_TRY(A.alloc_t(&h->attn_part, (size_t)MB * H * std::max(ns, h->cross.nsplit) * (ATT_D + 2)));   // the cross step's too
  B200_TRY(A.alloc_t(&h->attn_counters, (size_t)MB * H));
  B200_TRY(h->open_streams());
  B200_TRY(A.alloc_host(&h->pin_in, (size_t)B * n_in_max));
  B200_TRY(A.alloc_host(&h->pin_out, (size_t)B * (c.dep_q + 1)));
  B200_TRY(A.alloc_host(&h->pin_noise, (size_t)B * noise_per_row(h)));
  if (c.quantize) {     // activations are re-quantised row-wise before every linear (QLinear.forward, utils/quantize.py:28-36)
    const int kmax = std::max(std::max(d, c.ffn_hidden), std::max(c.depformer_dim, c.depformer_ffn_hidden));
    B200_TRY(A.alloc_t(&h->xq, (size_t)MB * kmax, false));
    B200_TRY(A.alloc_t(&h->xq_scale, (size_t)MB, false));
  }
  B200_TRY(tc::linear_init());
  B200_TRY(h->dep.alloc_fused(h));
  // streaming-state snapshot (lm.py:527-542 _LMGenState + the temporal transformer's ring caches, transformer.py:196-288)
  A.mark_state(h->exec_mask, B, "exec_mask", B200_U8, {B});
  if (cfg) A.mark_state(h->exec_mask_m, MB, "model.exec_mask", B200_U8, {MB});
  A.mark_state(h->cache, (size_t)B * h->Kc * h->CT * 8, "cache", B200_I64, {B, h->Kc, h->CT});
  A.mark_state(h->offsets, (size_t)B * 8, "offsets", B200_I64, {B});
  A.mark_state(h->pos, (size_t)MB * 8, "model.offset", B200_I64, {MB});
  A.mark_state(h->noise_ctr, 8, "noise_counter", B200_I64, {1});
  B200_TRY(h->kv.mark_state(A));
  h->cross.mark_state(A);
  h->ss.mark_state(A);
  {
    const int rows_add[2] = {0, B};
    std::vector<RowSlice> s;
    auto add = [&](void* p, long long row_bytes, int model_rows) {
      for (int k = 0; k < model_rows; ++k) s.push_back({static_cast<char*>(p), row_bytes, 0, rows_add[k]});
    };
    add(h->exec_mask, 1, 1);
    add(h->cache, (long long)h->Kc * h->CT * 8, 1);
    add(h->offsets, 8, 1);
    add(h->pos, 8, MB / B);
    if (cfg) add(h->exec_mask_m, 1, 2);
    if (h->cfg_until) add(h->cfg_until, 8, 1);
    h->n_slices = (int)s.size();
    add(h->cond_sum, (long long)d * 2, MB / B);
    h->n_slices_cond = (int)s.size();
    h->slices_end_cond = layout_row_slices(s, sizeof(SessionHeader));
    h->slices_end = s[h->n_slices].rec_off;
    h->slices_max = 0;
    for (auto& e : s) h->slices_max = std::max(h->slices_max, e.row_bytes);
    B200_TRY(A.alloc_t(&h->slices_dev, s.size(), false));
    B200_CUDA(cudaMemcpy(h->slices_dev, s.data(), s.size() * sizeof(RowSlice), cudaMemcpyHostToDevice));
  }
  B200_CUDA(cudaDeviceSynchronize());
  cleanup.armed = false;
  h->batch = B;
  h->MB = MB;
  return B200_OK;
}

/* get_streaming_state / set_streaming_state: device blob = marked buffers + the host step counter (last 256 B) */
int64_t b200_lm_state_bytes(b200_lm* h) { return (h && h->batch > 0) ? (int64_t)h->state.state_bytes() + 256 : 0; }

int b200_lm_get_state(b200_lm* h, void* dst_dev, int64_t capacity) {
  B200_STREAMING_ENTRY(h, "lm_get_state");
  B200_TRY(h->save_state(dst_dev, capacity, 256, "lm_get_state"));    // a paged handle's blob is a contiguous one's
  const size_t n = h->state.state_bytes();
  B200_CUDA(cudaMemcpyAsync(static_cast<char*>(dst_dev) + n, &h->offset_cpu, 8, cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200_OK;
}

int b200_lm_set_state(b200_lm* h, const void* src_dev, int64_t nbytes) {
  B200_STREAMING_ENTRY(h, "lm_set_state");
  B200_TRY(h->check_blob(src_dev, nbytes, 256, "lm_set_state"));
  const size_t n = h->state.state_bytes();
  size_t off_pos = 0;        // the rows take the snapshot's positions first (nothing changes if they cannot), then its K / V
  for (auto& e : h->state.snap) {
    if (e.name == "model.offset") break;
    off_pos += (e.bytes + 255) / 256 * 256;
  }
  B200_TRY(h->kv.hold_dev(static_cast<const char*>(src_dev) + off_pos, "lm_set_state", h->stream));
  B200_TRY(h->load_state(src_dev));
  B200_CUDA(cudaMemcpyAsync(&h->offset_cpu, static_cast<const char*>(src_dev) + n, 8, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200_OK;
}

/* the same state, entry by entry (the Python shim groups them into the reference's per-module State objects) */
int b200_lm_state_count(b200_lm* h) { return (h && h->batch > 0) ? (int)h->state.snap.size() : 0; }
int b200_lm_state_entry(b200_lm* h, int index, const char** name, int* dtype, int* ndim, int64_t* shape8, int64_t* nbytes) {
  B200_TRY(check_streaming(h, "lm_state_entry"));
  return h->state_entry_info(index, name, dtype, ndim, shape8, nbytes);
}
int b200_lm_state_read(b200_lm* h, const char* name, void* dst_dev, int64_t nbytes) {
  B200_STREAMING_ENTRY(h, "lm_state_read");
  return h->state_entry(name, dst_dev, nullptr, nbytes, "lm_state_read");
}
int b200_lm_state_write(b200_lm* h, const char* name, const void* src_dev, int64_t nbytes) {
  B200_STREAMING_ENTRY(h, "lm_state_write");
  if (src_dev && name && !strcmp(name, "model.offset")) {     // the rows take their new positions before they are written
    const StateEntry* e = nullptr;
    B200_TRY(h->find_entry(name, nbytes, &e));
    B200_TRY(h->kv.hold_dev(src_dev, "lm_state_write", h->stream));
  }
  return h->state_entry(name, nullptr, src_dev, nbytes, "lm_state_write");
}
int64_t b200_lm_get_offset_cpu(b200_lm* h) { return h ? h->offset_cpu : 0; }
int b200_lm_set_offset_cpu(b200_lm* h, int64_t v) {
  B200_TRY(check_streaming(h, "lm_set_offset_cpu"));
  h->offset_cpu = v;
  return B200_OK;
}

int b200_lm_streaming_end(b200_lm* h) {
  if (!h) return B200_OK;
  DeviceGuard g(h->device);
  h->end_streaming();
  h->maps.clear();
  h->dep.end();
  h->cfg_until = nullptr; h->noise_ctr = nullptr; h->cond_sum = nullptr; h->cond_on = 0;
  h->kv.end();
  h->cross.end();
  h->ss.end();
  h->taps = nullptr; h->taps_on = 0;
  h->pin_in = h->pin_out = nullptr;
  h->pin_noise = nullptr;
  h->MB = 0;
  return B200_OK;
}

int b200_lm_reset(b200_lm* h, const uint8_t* reset_mask_dev) {
  B200_STREAMING_ENTRY(h, "lm_reset");
  const int B = h->batch;
  h->kv.release(reset_mask_dev, B, h->stream);
  // per-row device offsets (lm.py:539, transformer.py:229-234, 331-333) ...
  B200_LAUNCH(lm_reset_kernel, ceil_div(B, 128), 128, 0, h->stream, h->offsets, h->pos, h->exec_mask, h->exec_mask_m,
              reset_mask_dev, B, cfg_on(h) ? 1 : 0);
  h->ss.clear(reset_mask_dev, h->stream);       // the rows' text histories; their settings stay
  // ... and the global host counter (lm.py:540): after any reset, step() reports "not ready" for max_delay calls
  h->offset_cpu = 0;
  return check_launch("lm_reset");
}

int b200_lm_set_exec_mask(b200_lm* h, const uint8_t* exec_mask_dev) {
  B200_STREAMING_ENTRY(h, "lm_set_exec_mask");
  if (!exec_mask_dev) B200_FAIL(B200_ERR_INVALID, "lm_set_exec_mask: null mask");
  B200_CUDA(cudaMemcpyAsync(h->exec_mask, exec_mask_dev, h->batch, cudaMemcpyDeviceToDevice, h->stream));
  if (cfg_on(h)) {      // exec_mask.repeat(2) (lm.py:658-661)
    B200_CUDA(cudaMemcpyAsync(h->exec_mask_m, exec_mask_dev, h->batch, cudaMemcpyDeviceToDevice, h->stream));
    B200_CUDA(cudaMemcpyAsync(h->exec_mask_m + h->batch, exec_mask_dev, h->batch, cudaMemcpyDeviceToDevice, h->stream));
  }
  return B200_OK;
}

int b200_lm_set_condition_sum(b200_lm* h, const void* sum_bf16_dev, int rows) {
  B200_STREAMING_ENTRY(h, "lm_set_condition_sum");
  const int on = sum_bf16_dev ? 1 : 0;
  if (on && rows != h->MB)      // lm.py:648-651: "cfg requires 2x more conditions"
    B200_FAIL(B200_ERR_SHAPE, "lm_set_condition_sum: %d rows given, the model runs on %d", rows, h->MB);
  if (on) B200_CUDA(cudaMemcpyAsync(h->cond_sum, sum_bf16_dev, (size_t)h->MB * h->cfg.dim * 2, cudaMemcpyDeviceToDevice, h->stream));
  if (on != h->cond_on) h->graphs[0].drop();
  h->cond_on = on;
  return B200_OK;
}

int b200_lm_set_cross_attention(b200_lm* h, int enable) {
  if (!h) B200_FAIL(B200_ERR_INVALID, "lm_set_cross_attention: null handle");
  if (h->finalized) B200_FAIL(B200_ERR_STATE, "lm_set_cross_attention: the layers' weights are packed at finalize; set it before");
  return h->cross.set(enable, h->cfg);
}

int b200_lm_set_depformer_schedule(b200_lm* h, const int* schedule, int n) {
  if (!h) B200_FAIL(B200_ERR_INVALID, "lm_set_depformer_schedule: null handle");
  if (h->finalized || !h->store.items.empty())
    B200_FAIL(B200_ERR_STATE, "lm_set_depformer_schedule: the weight sets are named by the schedule; set it before the first tensor");
  const int dep_q = h->cfg.dep_q;
  if (n != 0 && (n != dep_q || !schedule))
    B200_FAIL(B200_ERR_INVALID, "lm_set_depformer_schedule: %d entries, the depformer has %d steps", n, dep_q);
  for (int k = 0; k < n; ++k)
    if (schedule[k] < 0 || schedule[k] >= dep_q)
      B200_FAIL(B200_ERR_INVALID, "lm_set_depformer_schedule: entry %d = %d outside [0, %d)", k, schedule[k], dep_q);
  h->dep.set_schedule(schedule, n);
  return B200_OK;
}

int b200_lm_set_depformer_low_rank(b200_lm* h, int rank) {
  if (!h) B200_FAIL(B200_ERR_INVALID, "lm_set_depformer_low_rank: null handle");
  if (h->finalized || !h->store.items.empty())
    B200_FAIL(B200_ERR_STATE, "lm_set_depformer_low_rank: the tables' shapes follow the rank; set it before the first tensor");
  // without a depformer (dep_q = 0) there are no tables to factor and the rank is ignored, as lm.py:186-196 does
  if (rank < 0 || rank > DEP_LOW_RANK_MAX)
    B200_FAIL(B200_ERR_INVALID, "lm_set_depformer_low_rank: rank %d (in [1, %d]; 0 = full rank)", rank, DEP_LOW_RANK_MAX);
  h->dep.low_rank = rank;
  return B200_OK;
}

int b200_lm_set_cross_len(b200_lm* h, int keys) {
  if (!h) B200_FAIL(B200_ERR_INVALID, "lm_set_cross_len: null handle");
  return h->cross.set_len(keys, h->batch > 0);
}

int b200_lm_set_condition_cross(b200_lm* h, const void* src_bf16_dev, const int32_t* rows_host, int n_rows) {
  B200_STREAMING_ENTRY(h, "lm_set_condition_cross");
  return h->cross.fill(h, src_bf16_dev, rows_host, n_rows);
}

int b200_lm_set_taps(b200_lm* h, int enable) {
  B200_STREAMING_ENTRY(h, "lm_set_taps");
  const int on = enable ? 1 : 0;
  if (on && !h->taps) B200_TRY(h->state.alloc_t(&h->taps, (size_t)tap_elems(h)));     // freed with the state at streaming_end
  if (on != h->taps_on) h->graphs[0].drop();
  h->taps_on = on;
  return B200_OK;
}

int b200_lm_set_kv_dtype(b200_lm* h, int kv_dtype) {
  if (!h) B200_FAIL(B200_ERR_INVALID, "lm_set_kv_dtype: null handle");
  if (h->batch > 0) B200_FAIL(B200_ERR_STATE, "lm_set_kv_dtype: the rings are allocated at streaming_begin; set the dtype before it");
  return h->kv.set_dtype(kv_dtype);
}

int b200_lm_set_kv_capacity(b200_lm* h, int slots) {
  if (!h) B200_FAIL(B200_ERR_INVALID, "lm_set_kv_capacity: null handle");
  if (h->batch > 0) B200_FAIL(B200_ERR_STATE, "lm_set_kv_capacity: the rings are allocated at streaming_begin; set the capacity before it");
  return h->kv.set_capacity(slots);
}

int b200_lm_set_kv_pool(b200_lm* h, int64_t frames, int page_slots) {
  if (!h) B200_FAIL(B200_ERR_INVALID, "lm_set_kv_pool: null handle");
  if (h->batch > 0) B200_FAIL(B200_ERR_STATE, "lm_set_kv_pool: the pool is allocated at streaming_begin; set it before it");
  return h->kv.set_pool(frames, page_slots);
}

int b200_lm_kv_pool_usage(b200_lm* h, int* pages_used, int* pages_total) {
  B200_STREAMING_ENTRY(h, "lm_kv_pool_usage");
  return h->kv.usage(pages_used, pages_total, h->stream);
}

int b200_lm_session_bytes(b200_lm* h, int row, int64_t* nbytes) {
  B200_STREAMING_ENTRY(h, "lm_session_bytes");
  SessionPlan p;
  B200_TRY(session_plan(h, row, "lm_session_bytes", &p));
  if (nbytes) *nbytes = p.bytes;
  return B200_OK;
}

int b200_lm_session_export(b200_lm* h, int row, void* dst_dev, int64_t capacity) {
  B200_STREAMING_ENTRY(h, "lm_session_export");
  SessionPlan p;
  B200_TRY(session_plan(h, row, "lm_session_export", &p));
  if (!dst_dev) B200_FAIL(B200_ERR_INVALID, "lm_session_export: null destination");
  if (capacity < p.bytes) B200_FAIL(B200_ERR_SHAPE, "lm_session_export: the record takes %lld bytes, capacity %lld", (long long)p.bytes, (long long)capacity);
  SessionHeader s = h->session_header(p.bytes);
  s.kv_dtype = (uint32_t)h->kv.kind; s.rows = p.rows;
  s.flags = (p.cond ? SESSION_COND : 0) | (h->cfg_until ? SESSION_CFG_UNTIL : 0);
  h->cross.stamp(&s);
  h->ss.stamp(&s);
  s.pos[0] = p.pos[0]; s.pos[1] = p.pos[1]; s.n = p.n;
  char* rec = static_cast<char*>(dst_dev);
  B200_CUDA(cudaMemcpyAsync(rec, &s, sizeof(s), cudaMemcpyHostToDevice, h->stream));
  B200_TRY(row_slice_copy(h->slices_dev, p.cond ? h->n_slices_cond : h->n_slices, h->slices_max, rec, row, true, h->stream));
  B200_TRY(session_kv(h, row, p, rec, true));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200_OK;
}

int b200_lm_session_import(b200_lm* h, int row, const void* src_dev, int64_t nbytes) {
  B200_STREAMING_ENTRY(h, "lm_session_import");
  const auto& c = h->cfg;
  B200_TRY(h->check_row(row, "lm_session_import"));
  SessionHeader s;
  B200_TRY(h->read_session_header(src_dev, nbytes, "lm_session_import", &s));
  B200_TRY(h->kv.check_record(s.kv_dtype, "lm_session_import"));
  SessionPlan p;
  p.rows = h->MB / h->batch;
  if (s.rows != p.rows || ((s.flags & SESSION_CFG_UNTIL) != 0) != (h->cfg_until != nullptr))
    B200_FAIL(B200_ERR_INVALID, "lm_session_import: classifier-free guidance (or cfg_is_masked_until) on one side only");
  p.cond = (s.flags & SESSION_COND) != 0;
  if (p.cond != (h->cond_on != 0)) B200_FAIL(B200_ERR_INVALID, "lm_session_import: condition_sum on one side only");
  B200_TRY(h->cross.check_record(s, "lm_session_import"));
  B200_TRY(h->ss.check_record(s, "lm_session_import"));
  p.pos[0] = s.pos[0]; p.pos[1] = p.rows > 1 ? s.pos[1] : 0;
  const int64_t top = std::max(p.pos[0], p.pos[1]);
  if (p.pos[0] < 0 || p.pos[1] < 0 || s.n != std::min<int64_t>(top, c.context))
    B200_FAIL(B200_ERR_INVALID, "lm_session_import: corrupt record (positions %lld / %lld, %lld slots)", (long long)p.pos[0],
              (long long)p.pos[1], (long long)s.n);
  p.n = s.n;
  session_size(h, &p);
  if (s.bytes != p.bytes || nbytes != p.bytes)
    B200_FAIL(B200_ERR_SHAPE, "lm_session_import: the record takes %lld bytes, header says %lld, caller passed %lld", (long long)p.bytes,
              (long long)s.bytes, (long long)nbytes);
  B200_TRY(h->kv.check_history(top, "lm_session_import"));
  B200_TRY(h->kv.hold(row, h->batch, std::vector<long long>(p.pos, p.pos + p.rows), "lm_session_import", h->stream));
  char* rec = const_cast<char*>(static_cast<const char*>(src_dev));
  B200_TRY(row_slice_copy(h->slices_dev, p.cond ? h->n_slices_cond : h->n_slices, h->slices_max, rec, row, false, h->stream));
  B200_TRY(session_kv(h, row, p, rec, false));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200_OK;
}

int b200_lm_assume_fill(b200_lm* h, int fill) {
  B200_STREAMING_ENTRY(h, "lm_assume_fill");
  if (fill < 0) B200_FAIL(B200_ERR_INVALID, "lm_assume_fill: negative fill");
  std::vector<long long> v(h->MB, fill);
  B200_TRY(h->kv.hold(0, 1, v, "lm_assume_fill", h->stream));
  B200_CUDA(cudaMemcpyAsync(h->offsets, v.data(), (size_t)h->batch * 8, cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaMemcpyAsync(h->pos, v.data(), v.size() * 8, cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  h->offset_cpu = fill;
  return B200_OK;
}

/* Synchronises the handle's stream and returns (and clears) the device error flags: B200_FLAG_TOKEN_RANGE = a token id outside
 * its embedding table reached the model (the reference would hit a device assert in F.embedding). */
int b200_lm_error_flags(b200_lm* h, int* flags_out) {
  B200_STREAMING_ENTRY(h, "lm_error_flags");
  return h->error_flags(flags_out);
}

static int run_step(b200_lm* h, int n_in, int replace, int internal_noise) {
  if (n_in != h->n_in_static || replace != h->replace_static || internal_noise != h->noise_static) {     // the captured graph is specific to all three
    h->n_in_static = n_in;
    h->replace_static = replace;
    h->noise_static = internal_noise;
    h->graphs[0].drop();
  }
  B200_TRY(tc::linear_prepare());
  return h->run(h->graphs[0], "the LM step", [h] { return step_body(h); });
}

static bool sampling_on(const b200_lm* h) { return h->use_sampling && (h->temp > 0.f || h->temp_text > 0.f); }

int b200_lm_step(b200_lm* h, const int64_t* in_codes_dev, int n_in, const float* noise_dev, int64_t* out_tokens_dev,
                 int support_out_of_sync, int* ready_host) {
  return b200_lm_step_ex(h, in_codes_dev, n_in, noise_dev, nullptr, out_tokens_dev, support_out_of_sync, ready_host);
}

int b200_lm_step_ex(b200_lm* h, const int64_t* in_codes_dev, int n_in, const float* noise_dev, const int64_t* replace_audio_dev,
                    int64_t* out_tokens_dev, int support_out_of_sync, int* ready_host) {
  B200_STREAMING_ENTRY(h, "lm_step");
  const auto& c = h->cfg;
  const int B = h->batch, needed = c.n_q - c.dep_q;
  if (!in_codes_dev || !out_tokens_dev) B200_FAIL(B200_ERR_SHAPE, "lm_step: null buffers");
  if (n_in < needed || n_in > c.n_q)   // lm.py:683-686 assertion
    B200_FAIL(B200_ERR_SHAPE, "lm_step: expected at least %d user codebooks, got %d", needed, n_in);
  if (replace_audio_dev && c.dep_q == 0) B200_FAIL(B200_ERR_INVALID, "lm_step: depformer_replace_tokens on a model without depformer");
  B200_CUDA(cudaMemcpyAsync(h->in_codes, in_codes_dev, (size_t)B * n_in * 8, cudaMemcpyDeviceToDevice, h->stream));
  if (noise_dev)
    B200_CUDA(cudaMemcpyAsync(h->noise, noise_dev, (size_t)B * noise_per_row(h) * 4, cudaMemcpyDeviceToDevice, h->stream));
  if (replace_audio_dev)
    B200_CUDA(cudaMemcpyAsync(h->replace_tokens, replace_audio_dev, (size_t)B * c.dep_q * 8, cudaMemcpyDeviceToDevice, h->stream));
  B200_TRY(run_step(h, n_in, replace_audio_dev ? 1 : 0, (!noise_dev && sampling_on(h)) ? 1 : 0));
  B200_CUDA(cudaMemcpyAsync(out_tokens_dev, h->out_tokens, (size_t)B * (c.dep_q + 1) * 8, cudaMemcpyDeviceToDevice,
                            h->stream));
  h->offset_cpu += 1;
  if (ready_host) *ready_host = (support_out_of_sync || h->offset_cpu > h->max_delay) ? 1 : 0;   // lm.py:774-776
  return B200_OK;
}

int b200_lm_step_host(b200_lm* h, const int64_t* in_codes_host, int n_in, const float* noise_host,
                      int64_t* out_tokens_host, int support_out_of_sync, int* ready_host) {
  B200_STREAMING_ENTRY(h, "lm_step_host");
  const auto& c = h->cfg;
  const int B = h->batch, needed = c.n_q - c.dep_q;
  if (!in_codes_host || !out_tokens_host) B200_FAIL(B200_ERR_SHAPE, "lm_step_host: null buffers");
  if (n_in < needed || n_in > c.n_q) B200_FAIL(B200_ERR_SHAPE, "lm_step_host: expected at least %d user codebooks, got %d", needed, n_in);
  memcpy(h->pin_in, in_codes_host, (size_t)B * n_in * 8);
  B200_CUDA(cudaMemcpyAsync(h->in_codes, h->pin_in, (size_t)B * n_in * 8, cudaMemcpyHostToDevice, h->stream));
  if (noise_host) {
    memcpy(h->pin_noise, noise_host, (size_t)B * noise_per_row(h) * 4);
    B200_CUDA(cudaMemcpyAsync(h->noise, h->pin_noise, (size_t)B * noise_per_row(h) * 4, cudaMemcpyHostToDevice, h->stream));
  }
  B200_TRY(run_step(h, n_in, 0, (!noise_host && sampling_on(h)) ? 1 : 0));
  B200_CUDA(cudaMemcpyAsync(h->pin_out, h->out_tokens, (size_t)B * (c.dep_q + 1) * 8, cudaMemcpyDeviceToHost, h->stream));
  int flags = 0;
  B200_CUDA(cudaMemcpyAsync(&flags, h->err, 4, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  memcpy(out_tokens_host, h->pin_out, (size_t)B * (c.dep_q + 1) * 8);
  h->offset_cpu += 1;
  if (ready_host) *ready_host = (support_out_of_sync || h->offset_cpu > h->max_delay) ? 1 : 0;
  if (flags) {
    cudaMemsetAsync(h->err, 0, 4, h->stream);
    B200_TRY(h->kv.flag_error(flags, "lm_step_host"));
    B200_FAIL(B200_ERR_INVALID, "lm_step_host: a token id outside its embedding table reached the model (flags %d)", flags);
  }
  return B200_OK;
}

int b200_lm_read_buffer(b200_lm* h, const char* name, void* dst_dev, int64_t capacity_bytes, int64_t* nbytes) {
  B200_STREAMING_ENTRY(h, "lm_read_buffer");
  const auto& c = h->cfg;
  const std::string n = name ? name : "";
  const int B = h->batch, MB = h->MB;
  const bool cfg = cfg_on(h);
  const void* src = nullptr;
  int64_t sz = 0;
  // with CFG "text_logits" is what the sampler reads (the guided rows, lm.py:728-732); the model's own 2B rows are
  // "model_text_logits"
  if (h->dep.buffer(n, cfg, &src, &sz)) {}
  else if (n == "text_logits") { src = (cfg && !h->cfg_is_no_text) ? h->text_logits_cfg : h->text_logits; sz = (int64_t)B * c.text_card * 2; }
  else if (n == "model_text_logits") { src = h->text_logits; sz = (int64_t)MB * c.text_card * 2; }
  else if (n == "transformer_out") { src = h->tout; sz = (int64_t)MB * c.dim * 2; }
  else if (n == "input_tokens") { src = h->input_tokens; sz = (int64_t)MB * h->Kc * 8; }
  else if (n == "text_token") { src = h->text_token; sz = (int64_t)B * 8; }
  else if (n == "audio_tokens") { src = h->audio_tokens; sz = (int64_t)c.dep_q * B * 8; }
  else if (n == "noise") { src = h->noise; sz = (int64_t)B * noise_per_row(h) * 4; }
  else if (n == "extra_heads") { src = h->extra_out; sz = (int64_t)h->extra_w.size() * MB * c.extra_heads_dim * 2; }
  else if (n.rfind("temporal.", 0) == 0) {
    // the taps of the last step taken with b200_lm_set_taps on: "temporal.embed", "temporal.layers.<l>.<kind>"
    if (!h->taps) B200_FAIL(B200_ERR_STATE, "lm_read_buffer: '%s' is a tap; turn the taps on (b200_lm_set_taps) before the step", n.c_str());
    int layer = -1, kind = 0;
    if (n != "temporal.embed") {
      const std::string rest = n.rfind("temporal.layers.", 0) == 0 ? n.substr(16) : "";
      const size_t dot = rest.find('.');
      const std::string idx = rest.substr(0, dot), k = dot == std::string::npos ? "" : rest.substr(dot + 1);
      const bool digits = !idx.empty() && idx.size() <= 4 && idx.find_first_not_of("0123456789") == std::string::npos;
      layer = digits ? atoi(idx.c_str()) : -1;
      kind = k == "attn_out" ? TAP_ATTN_OUT : k == "x_attn" ? TAP_X_ATTN : k == "gated" ? TAP_GATED : k == "x_out" ? TAP_X_OUT : -1;
      if (h->cross.on && kind < 0) kind = k == "cross_out" ? TAP_CROSS_OUT : k == "x_cross" ? TAP_X_CROSS : -1;
      if (layer < 0 || layer >= (int)h->layers.size() || kind < 0)
        B200_FAIL(B200_ERR_INVALID, "lm_read_buffer: unknown buffer '%s'", n.c_str());
    }
    int64_t elems = 0;
    src = h->taps + tap_slot(h, layer, kind, &elems);
    sz = elems * 2;
  }
  else B200_FAIL(B200_ERR_INVALID, "lm_read_buffer: unknown buffer '%s'", n.c_str());
  return copy_out(src, sz, sz, dst_dev, capacity_bytes, nbytes, h->stream, "lm_read_buffer");
}

int64_t b200_lm_algorithmic_bytes(b200_lm* h, int kv_fill) {
  if (!h || h->batch <= 0) return 0;
  const auto& c = h->cfg;
  const int64_t B = h->MB;
  if (kv_fill > c.context) kv_fill = c.context;
  // weights streamed once per step (embedding tables are gathers, counted per row below)
  int64_t w = 0;
  w += (int64_t)c.num_layers * ((int64_t)3 * c.dim * c.dim + (int64_t)c.dim * c.dim + (int64_t)3 * c.ffn_hidden * c.dim) * 2;
  w += (int64_t)c.text_card * c.dim * 2;
  w += (int64_t)h->dep.n_sets * c.depformer_dim * c.dim * 2;      // depformer_in: one linear per weight set
  w += (int64_t)c.dep_q * c.depformer_num_layers *
       ((int64_t)4 * c.depformer_dim * c.depformer_dim + (int64_t)3 * c.depformer_ffn_hidden * c.depformer_dim) * 2;
  w += (int64_t)c.dep_q * c.card * c.depformer_dim * 2;
  if (c.quantize) w /= 2;        // one byte per weight (the fp32 row scales are < 0.1 % of that)
  // per session: KV ring read (valid slots only) + append, embedding rows, logits written + read by the sampler
  const int64_t kv_row = c.num_heads * h->kv.slot_bytes();      // bytes of one K (or V) slot of a layer, all heads
  int64_t per = (int64_t)c.num_layers * 2 * kv_fill * kv_row + (int64_t)c.num_layers * 2 * kv_row;
  per += (int64_t)(c.n_q + 1) * c.dim * 2 + (int64_t)c.dep_q * c.depformer_dim * 2;
  per += (int64_t)2 * (c.text_card + (int64_t)c.dep_q * c.card) * 2;
  return w + per * B + h->cross.algorithmic_bytes(B);
}

}  // extern "C"
