// Shared helpers for the moshi_b200 CUDA library (sm_90a only).
#pragma once

#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <functional>
#include <map>
#include <string>
#include <vector>

#include "../../include/moshi_b200.h"

namespace b200 {

// ---------------------------------------------------------------------------------------------
// error plumbing
// ---------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
extern std::atomic<int64_t> g_launches;

#define B200_CUDA(expr)                                                                      \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess) {                                                                 \
      b200::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return B200_ERR_CUDA;                                                                  \
    }                                                                                        \
  } while (0)

#define B200_TRY(expr)             \
  do {                             \
    int _rc = (expr);              \
    if (_rc != B200_OK) return _rc; \
  } while (0)

#define B200_FAIL(code, ...)      \
  do {                            \
    b200::set_error(__VA_ARGS__); \
    return code;                  \
  } while (0)

// Every kernel launch goes through this so that `gpu_launches` is a count, not a guess.
#define B200_LAUNCH(kernel, grid, block, smem, stream, ...)                    \
  do {                                                                         \
    kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);                \
    b200::g_launches.fetch_add(1, std::memory_order_relaxed);                  \
  } while (0)

inline int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("launch of %s failed: %s", what, cudaGetErrorString(e));
    return B200_ERR_CUDA;
  }
  return B200_OK;
}

// ---------------------------------------------------------------------------------------------
// named tensor store (the state-dict side of the ABI)
// ---------------------------------------------------------------------------------------------
struct Tensor {
  void* data = nullptr;   // device, owned by the store
  int dtype = B200_F32;
  std::vector<int64_t> shape;
  int64_t numel() const {
    int64_t n = 1;
    for (auto s : shape) n *= s;
    return n;
  }
};

inline size_t dtype_size(int dtype) {
  switch (dtype) {
    case B200_F32: return 4;
    case B200_BF16: return 2;
    case B200_F16: return 2;
    case B200_I64: return 8;
    case B200_U8: return 1;
    case B200_I8: return 1;
    case B200_I32: return 4;
  }
  return 0;
}

struct TensorStore {
  std::map<std::string, Tensor> items;
  int put(const char* name, const void* dev, int dtype, int ndim, const int64_t* shape);
  const Tensor* find(const std::string& name) const;
  void release(const std::string& name);
  void release_all();
};

// Device and pinned host allocation bookkeeping for a handle: everything freed in one place, at the latest when the arena goes.
struct StateEntry {
  std::string name;        // handle-local name; the Python shims map these onto the reference's per-module State fields
  void* ptr; size_t bytes; int dtype; std::vector<int64_t> shape;
};
struct Arena {
  std::vector<void*> ptrs, host;
  // buffers that make up the streaming state (get/set_streaming_state, streaming.py:158-181), in registration order
  std::vector<StateEntry> snap;
  void mark_state(void* p, size_t bytes, const std::string& name = "", int dtype = B200_U8, std::vector<int64_t> shape = {}) {
    if (!p || !bytes) return;
    if (shape.empty()) shape = {(int64_t)bytes};
    snap.push_back({name, p, bytes, dtype, shape});
  }
  const StateEntry* find_state(const std::string& name) const {
    for (auto& e : snap) if (e.name == name) return &e;
    return nullptr;
  }
  size_t state_bytes() const;                 // each segment padded to 256 B
  int alloc(void** out, size_t bytes, bool zero = true);
  template <typename T>
  int alloc_t(T** out, size_t count, bool zero = true) {
    return alloc(reinterpret_cast<void**>(out), count * sizeof(T), zero);
  }
  template <typename T>
  int alloc_host(T** out, size_t count) {     // pinned host memory
    *out = nullptr;
    B200_CUDA(cudaMallocHost(reinterpret_cast<void**>(out), count * sizeof(T)));
    host.push_back(*out);
    return B200_OK;
  }
  void free_all();
  Arena() = default;
  Arena(const Arena&) = delete;
  Arena& operator=(const Arena&) = delete;
  ~Arena() { free_all(); }
};

// Makes the handle's device current for the duration of an entry point (the reference's modules carry their device; a caller
// whose current device is another GPU must still be able to drive this handle).
struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    if (dev >= 0 && cudaGetDevice(&prev) == cudaSuccess && prev != dev) cudaSetDevice(dev); else prev = -1;
  }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

// The tail of every *_read_buffer entry point: reports the buffer's size, then (dst non-null) checks the capacity and copies
// `bytes` from src on `st`.  size and capacity are in the entry point's unit.
int copy_out(const void* src, int64_t size, int64_t bytes, void* dst, int64_t capacity, int64_t* size_out, cudaStream_t st,
             const char* what);

// What the frame services (frame.cu) check their handles against and read from them; B200_ERR_STATE unless streaming.  The
// pointer stays valid until the handle's streaming ends.
struct LmFrameView {
  int batch, model_rows, n_q, dep_q, max_delay, extra_heads, extra_dim;
  const __nv_bfloat16* extra_out;          // [extra_heads][model_rows][extra_dim] softmaxed heads of the last step
};
struct MimiFrameView {
  int batch, num_codebooks, frame_size;
};
int lm_frame_view(b200_lm* h, LmFrameView* out);         // lm.cu
int mimi_frame_view(b200_mimi* h, MimiFrameView* out);   // mimi.cu
int lm_device(const b200_lm* h);                         // lm.cu: the device the frame services allocate and run on
// lm.cu: a row the KV pool could not serve (B200_FLAG_KV_POOL) fails the frame with B200_ERR_STATE, as b200_lm_step_host does.
// Synchronises; clears that flag only, the others stay for b200_lm_error_flags.  Nothing without a pool.
int lm_check_kv_pool(b200_lm* h);

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// ---------------------------------------------------------------------------------------------
// session records (b200_{lm,mimi}_session_*): one session of a handle as a self-describing device buffer
// ---------------------------------------------------------------------------------------------
constexpr uint32_t SESSION_MAGIC = 0x5345534Du;      // "MSES"
constexpr uint32_t SESSION_VERSION = 1;
enum { SESSION_LM = 1, SESSION_MIMI = 2 };
// The first 256 bytes of a record; the host reads them before an import writes anything.  The body's layout is the handle's
// (lm.cu, mimi.cu).
struct SessionHeader {
  uint32_t magic, version, kind, kv_dtype;   // kv_dtype: B200_KV_* of an LM record, 0 for Mimi
  uint64_t fingerprint;                      // config_fingerprint of the model configuration
  int32_t rows;                              // model rows per session (LM: 2 under classifier-free guidance, else 1)
  int32_t flags;                             // LM: SESSION_COND / SESSION_CFG_UNTIL / SESSION_CROSS / SESSION_SAMPLING
  int64_t pos[2];                            // LM: model position of each row
  int64_t n;                                 // LM: temporal KV slots carried, min(pos, ring capacity)
  int64_t bytes;                             // size of the whole record
  uint8_t reserved[256 - 64];                // LM: int32 keys of the condition memory (SESSION_CROSS), then int32
                                             // history length (SESSION_SAMPLING)
};
static_assert(sizeof(SessionHeader) == 256, "session header is 256 bytes");
enum { SESSION_COND = 1, SESSION_CFG_UNTIL = 2, SESSION_CROSS = 4, SESSION_SAMPLING = 8 };

// FNV-1a over a configuration struct: records only go into handles built from the same configuration
inline uint64_t config_fingerprint(const void* p, size_t n) {
  uint64_t h = 0xcbf29ce484222325ull;
  for (size_t i = 0; i < n; ++i) h = (h ^ static_cast<const uint8_t*>(p)[i]) * 0x100000001b3ull;
  return h;
}

// One per-session slice of a handle's state: row r's bytes are ptr + (r + row_add) * row_bytes, stored at rec_off in a record.
struct RowSlice {
  char* ptr;
  long long row_bytes, rec_off;
  int row_add;
};
// Copies the slices of row `row` between the handle and `rec` (gather: handle -> record), one launch for the whole table.
// Offsets into the record are 16-byte aligned; max_row_bytes bounds the grid.
int row_slice_copy(const RowSlice* table_dev, int n, long long max_row_bytes, char* rec, int row, bool gather, cudaStream_t st);
// Lays out `slices` (row_bytes / ptr / row_add filled) from record offset `off` on, 16-byte aligned; returns the end offset.
inline long long layout_row_slices(std::vector<RowSlice>& slices, long long off) {
  for (auto& s : slices) {
    s.rec_off = off;
    off += (s.row_bytes + 15) / 16 * 16;
  }
  return off;
}

// ---------------------------------------------------------------------------------------------
// the streaming core of the LM and Mimi handles
// ---------------------------------------------------------------------------------------------
// A CUDA graph captured from a fixed launch sequence over static buffers.
struct Graph {
  cudaGraphExec_t exec = nullptr;
  int64_t kernels = 0;                 // kernel launches recorded in it: b200_launch_count advances by these per replay
  void drop() {
    if (exec) cudaGraphExecDestroy(exec);
    exec = nullptr;
  }
};

// What b200_lm and b200_mimi share: the device, the streams a batch of sessions runs on, its state arena and error flags, the
// captured graphs, the state blob and entries, and session-record framing.
struct StreamCore {
  int device = -1;                     // CUDA device the handle lives on (made current by every entry point)
  bool finalized = false;
  int batch = 0;                       // sessions streaming; 0: not streaming
  cudaStream_t stream = nullptr;       // caller's stream (inputs and outputs are ordered on it)
  cudaStream_t gstream = nullptr;      // private stream: graphs cannot be captured on the legacy default stream
  cudaStream_t body = nullptr;         // stream the kernels are being enqueued on (caller's, or gstream while capturing)
  cudaEvent_t ev_in = nullptr, ev_out = nullptr;
  int graph_enabled = 1;
  Graph graphs[2];                     // the handle's captured bodies (LM: the step; Mimi: encode, decode)
  Arena state;                         // everything a streaming batch allocates, freed by end_streaming
  int* err = nullptr;                  // device error flags (B200_FLAG_*)
  uint32_t session_kind = 0;           // SESSION_LM / SESSION_MIMI
  uint64_t fingerprint = 0;            // config_fingerprint of the handle's configuration

  virtual ~StreamCore() = default;
  // streaming_begin: the private stream and the fence events; end_streaming: waits for both streams, then drops the graphs,
  // destroys the streams and events and frees the state (also on a failed streaming_begin)
  int open_streams();
  void end_streaming();
  void drop_graphs() {
    for (auto& g : graphs) g.drop();
  }
  void set_graph(int enable) {
    graph_enabled = enable;
    if (!enable) drop_graphs();
  }
  // Runs `fn` (a fixed launch sequence over static buffers, enqueued on `body`) as graph g on the private stream, fenced against
  // the caller's stream on both sides; the first call captures it, and a failed capture leaves no graph.  With graphs off `fn`
  // runs eagerly on the caller's stream.
  int run(Graph& g, const char* what, const std::function<int()>& fn);
  // Synchronises the caller's stream, returns the device error flags and clears them.
  int error_flags(int* flags_out);

  // One state entry between the handle and a device buffer (exactly one of dst / src non-null), on the caller's stream.
  virtual int copy_entry(const StateEntry& e, void* dst, const void* src);
  int find_entry(const char* name, int64_t nbytes, const StateEntry** out) const;   // the entry, if it holds nbytes bytes
  int state_entry_info(int index, const char** name, int* dtype, int* ndim, int64_t* shape8, int64_t* nbytes) const;
  int state_entry(const char* name, void* dst, const void* src, int64_t nbytes, const char* what);
  // The state blob: every entry in marking order, each 256-byte aligned, then `trailer` bytes the handle owns.  save_state checks
  // the capacity, check_blob the size of a blob to load.
  int save_state(void* dst, int64_t capacity, size_t trailer, const char* what);
  int check_blob(const void* src, int64_t nbytes, size_t trailer, const char* what) const;
  int load_state(const void* src);
  // Session records: the header of this handle's kind and configuration for a record of `bytes` (one row, the rest zero), and the
  // header read back from a device record (synchronises) after checking the size, magic, version, kind and fingerprint.
  int check_row(int row, const char* what) const;
  SessionHeader session_header(int64_t bytes) const;
  int read_session_header(const void* src, int64_t nbytes, const char* what, SessionHeader* s);
};

// The prologue of every entry point that needs a streaming handle: B200_ERR_INVALID for a null handle, B200_ERR_STATE unless it
// is finalized and streaming; then the handle's device stays current until the entry point returns.
int check_streaming(const StreamCore* h, const char* what);
#define B200_STREAMING_ENTRY(h, what)          \
  B200_TRY(b200::check_streaming((h), (what))); \
  b200::DeviceGuard b200_entry_device_((h)->device)
// The checks of streaming_begin: a finalized handle that is not streaming yet, at least one session.
int check_begin(const StreamCore* h, int batch, const char* what);

// ---------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float elu1(float x) { return x > 0.f ? x : expm1f(x); }
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752440f)); }
__device__ __forceinline__ float bf2f(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ __nv_bfloat16 f2bf(float v) { return __float2bfloat16_rn(v); }
// round-trip through bf16: the reference materialises most intermediates as bf16 tensors
__device__ __forceinline__ float rbf(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

}  // namespace b200
