#include <algorithm>

#include "tc_host.cuh"

namespace b200 {

static thread_local char g_err[1024] = "";
std::atomic<int64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int TensorStore::put(const char* name, const void* dev, int dtype, int ndim, const int64_t* shape) {
  if (!name || !dev || ndim < 0 || ndim > 8) B200_FAIL(B200_ERR_INVALID, "load_tensor: bad arguments");
  size_t es = dtype_size(dtype);
  if (es == 0) B200_FAIL(B200_ERR_INVALID, "load_tensor(%s): unknown dtype %d", name, dtype);
  Tensor t;
  t.dtype = dtype;
  t.shape.assign(shape, shape + ndim);
  size_t bytes = (size_t)t.numel() * es;
  B200_CUDA(cudaMalloc(&t.data, bytes ? bytes : 1));
  B200_CUDA(cudaMemcpy(t.data, dev, bytes, cudaMemcpyDeviceToDevice));
  auto it = items.find(name);
  if (it != items.end()) {
    cudaFree(it->second.data);
    items.erase(it);
  }
  items[name] = t;
  return B200_OK;
}

const Tensor* TensorStore::find(const std::string& name) const {
  auto it = items.find(name);
  return it == items.end() ? nullptr : &it->second;
}

void TensorStore::release(const std::string& name) {
  auto it = items.find(name);
  if (it != items.end()) {
    cudaFree(it->second.data);
    items.erase(it);
  }
}

void TensorStore::release_all() {
  for (auto& kv : items) cudaFree(kv.second.data);
  items.clear();
}

int Arena::alloc(void** out, size_t bytes, bool zero) {
  *out = nullptr;
  B200_CUDA(cudaMalloc(out, bytes ? bytes : 1));
  ptrs.push_back(*out);
  if (zero) B200_CUDA(cudaMemset(*out, 0, bytes));
  return B200_OK;
}

void Arena::free_all() {
  for (void* p : ptrs) cudaFree(p);
  for (void* p : host) cudaFreeHost(p);
  ptrs.clear();
  host.clear();
  snap.clear();
}

static size_t pad256(size_t n) { return (n + 255) / 256 * 256; }

size_t Arena::state_bytes() const {
  size_t n = 0;
  for (auto& s : snap) n += pad256(s.bytes);
  return n;
}

int copy_out(const void* src, int64_t size, int64_t bytes, void* dst, int64_t capacity, int64_t* size_out, cudaStream_t st,
             const char* what) {
  if (size_out) *size_out = size;
  if (!dst || !size) return B200_OK;
  if (capacity < size) B200_FAIL(B200_ERR_SHAPE, "%s: destination too small", what);
  if (bytes) B200_CUDA(cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyDeviceToDevice, st));
  return B200_OK;
}

// ---- the streaming core -------------------------------------------------------------------------------------------------------
int check_streaming(const StreamCore* h, const char* what) {
  if (!h) B200_FAIL(B200_ERR_INVALID, "%s: null handle", what);
  if (!h->finalized) B200_FAIL(B200_ERR_STATE, "%s: handle not finalized", what);
  if (h->batch <= 0) B200_FAIL(B200_ERR_STATE, "%s: not streaming (call streaming_begin first)", what);
  return B200_OK;
}

int check_begin(const StreamCore* h, int batch, const char* what) {
  if (!h || !h->finalized) B200_FAIL(B200_ERR_STATE, "%s: handle not finalized", what);
  if (h->batch > 0) B200_FAIL(B200_ERR_STATE, "%s: already streaming", what);     // streaming.py:112
  if (batch < 1) B200_FAIL(B200_ERR_INVALID, "%s: batch %d", what, batch);
  return B200_OK;
}

int StreamCore::open_streams() {
  B200_CUDA(cudaStreamCreateWithFlags(&gstream, cudaStreamNonBlocking));
  B200_CUDA(cudaEventCreateWithFlags(&ev_in, cudaEventDisableTiming));
  B200_CUDA(cudaEventCreateWithFlags(&ev_out, cudaEventDisableTiming));
  return B200_OK;
}

void StreamCore::end_streaming() {
  if (batch > 0) {
    cudaStreamSynchronize(stream);
    if (gstream) cudaStreamSynchronize(gstream);
  }
  drop_graphs();
  if (gstream) cudaStreamDestroy(gstream);
  if (ev_in) cudaEventDestroy(ev_in);
  if (ev_out) cudaEventDestroy(ev_out);
  gstream = nullptr;
  ev_in = ev_out = nullptr;
  state.free_all();
  err = nullptr;
  batch = 0;
}

int StreamCore::run(Graph& g, const char* what, const std::function<int()>& fn) {
  if (!graph_enabled) {
    body = stream;
    return fn();
  }
  B200_CUDA(cudaEventRecord(ev_in, stream));
  B200_CUDA(cudaStreamWaitEvent(gstream, ev_in, 0));
  if (!g.exec) {
    cudaGraph_t graph = nullptr;
    const int64_t before = g_launches.load();
    body = gstream;
    B200_CUDA(cudaStreamBeginCapture(gstream, cudaStreamCaptureModeRelaxed));
    const int rc = fn();
    cudaError_t e = cudaStreamEndCapture(gstream, &graph);
    g.kernels = g_launches.load() - before;
    g_launches.fetch_sub(g.kernels);      // recorded, not executed
    body = stream;
    if (rc != B200_OK) {
      if (graph) cudaGraphDestroy(graph);
      return rc;
    }
    if (e != cudaSuccess) B200_FAIL(B200_ERR_CUDA, "graph capture of %s failed: %s", what, cudaGetErrorString(e));
    e = cudaGraphInstantiate(&g.exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) {
      g.exec = nullptr;
      B200_FAIL(B200_ERR_CUDA, "graph instantiate failed: %s", cudaGetErrorString(e));
    }
  }
  B200_CUDA(cudaGraphLaunch(g.exec, gstream));
  g_launches.fetch_add(g.kernels);
  B200_CUDA(cudaEventRecord(ev_out, gstream));
  B200_CUDA(cudaStreamWaitEvent(stream, ev_out, 0));
  return B200_OK;
}

int StreamCore::error_flags(int* flags_out) {
  int v = 0;
  B200_CUDA(cudaMemcpyAsync(&v, err, 4, cudaMemcpyDeviceToHost, stream));
  B200_CUDA(cudaStreamSynchronize(stream));
  if (v) B200_CUDA(cudaMemsetAsync(err, 0, 4, stream));
  if (flags_out) *flags_out = v;
  return B200_OK;
}

int StreamCore::copy_entry(const StateEntry& e, void* dst, const void* src) {
  if (dst) B200_CUDA(cudaMemcpyAsync(dst, e.ptr, e.bytes, cudaMemcpyDeviceToDevice, stream));
  else B200_CUDA(cudaMemcpyAsync(e.ptr, src, e.bytes, cudaMemcpyDeviceToDevice, stream));
  return B200_OK;
}

int StreamCore::find_entry(const char* name, int64_t nbytes, const StateEntry** out) const {
  const StateEntry* e = state.find_state(name ? name : "");
  if (!e) B200_FAIL(B200_ERR_INVALID, "state entry '%s' does not exist", name ? name : "(null)");
  if (nbytes != (int64_t)e->bytes) B200_FAIL(B200_ERR_SHAPE, "state entry '%s' holds %zu bytes, caller passed %lld", e->name.c_str(), e->bytes, (long long)nbytes);
  *out = e;
  return B200_OK;
}

int StreamCore::state_entry_info(int index, const char** name, int* dtype, int* ndim, int64_t* shape8, int64_t* nbytes) const {
  if (index < 0 || index >= (int)state.snap.size()) B200_FAIL(B200_ERR_INVALID, "state_entry: index %d out of range", index);
  const StateEntry& e = state.snap[index];
  if (name) *name = e.name.c_str();
  if (dtype) *dtype = e.dtype;
  if (ndim) *ndim = (int)e.shape.size();
  if (shape8) for (size_t i = 0; i < e.shape.size() && i < 8; ++i) shape8[i] = e.shape[i];
  if (nbytes) *nbytes = (int64_t)e.bytes;
  return B200_OK;
}

int StreamCore::state_entry(const char* name, void* dst, const void* src, int64_t nbytes, const char* what) {
  if (!dst && !src) B200_FAIL(B200_ERR_INVALID, "%s: null buffer", what);
  const StateEntry* e = nullptr;
  B200_TRY(find_entry(name, nbytes, &e));
  return copy_entry(*e, dst, src);
}

int StreamCore::save_state(void* dst, int64_t capacity, size_t trailer, const char* what) {
  if (!dst || capacity < (int64_t)(state.state_bytes() + trailer)) B200_FAIL(B200_ERR_SHAPE, "%s: destination too small", what);
  size_t off = 0;
  for (auto& e : state.snap) {
    B200_TRY(copy_entry(e, static_cast<char*>(dst) + off, nullptr));
    off += pad256(e.bytes);
  }
  return B200_OK;
}

int StreamCore::check_blob(const void* src, int64_t nbytes, size_t trailer, const char* what) const {
  const int64_t n = (int64_t)(state.state_bytes() + trailer);
  if (!src || nbytes != n)
    B200_FAIL(B200_ERR_SHAPE, "%s: snapshot of %lld bytes does not fit this session layout (%lld)", what, (long long)nbytes, (long long)n);
  return B200_OK;
}

int StreamCore::load_state(const void* src) {
  size_t off = 0;
  for (auto& e : state.snap) {
    B200_TRY(copy_entry(e, nullptr, static_cast<const char*>(src) + off));
    off += pad256(e.bytes);
  }
  return B200_OK;
}

int StreamCore::check_row(int row, const char* what) const {
  if (row < 0 || row >= batch) B200_FAIL(B200_ERR_INVALID, "%s: row %d outside [0, %d)", what, row, batch);
  return B200_OK;
}

SessionHeader StreamCore::session_header(int64_t bytes) const {
  SessionHeader s;
  memset(&s, 0, sizeof(s));
  s.magic = SESSION_MAGIC; s.version = SESSION_VERSION; s.kind = session_kind;
  s.fingerprint = fingerprint; s.rows = 1; s.bytes = bytes;
  return s;
}

int StreamCore::read_session_header(const void* src, int64_t nbytes, const char* what, SessionHeader* s) {
  if (!src) B200_FAIL(B200_ERR_INVALID, "%s: null record", what);
  if (nbytes < (int64_t)sizeof(SessionHeader)) B200_FAIL(B200_ERR_SHAPE, "%s: %lld bytes hold no record header", what, (long long)nbytes);
  B200_CUDA(cudaStreamSynchronize(stream));
  B200_CUDA(cudaMemcpy(s, src, sizeof(*s), cudaMemcpyDeviceToHost));
  if (s->magic != SESSION_MAGIC || s->version != SESSION_VERSION)
    B200_FAIL(B200_ERR_INVALID, "%s: not a session record (magic %08x, version %u)", what, s->magic, s->version);
  if (s->kind != session_kind)
    B200_FAIL(B200_ERR_INVALID, "%s: the record is not %s session (kind %u)", what, session_kind == SESSION_LM ? "an LM" : "a Mimi", s->kind);
  if (s->fingerprint != fingerprint) B200_FAIL(B200_ERR_INVALID, "%s: the record was taken with another configuration", what);
  return B200_OK;
}

// blockIdx.y = slice; 16-byte vectors where both sides and the length allow, bytes otherwise
static __global__ void row_slice_copy_kernel(const RowSlice* __restrict__ table, char* rec, int row, int gather) {
  const RowSlice d = table[blockIdx.y];
  char* p = d.ptr + (long long)(row + d.row_add) * d.row_bytes;
  char* r = rec + d.rec_off;
  char* dst = gather ? r : p;
  const char* src = gather ? p : r;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (((uintptr_t)dst | (uintptr_t)src | (uintptr_t)d.row_bytes) & 15) {
    for (long long i = i0; i < d.row_bytes; i += stride) dst[i] = src[i];
  } else {
    for (long long i = i0; i < d.row_bytes / 16; i += stride)
      reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(src)[i];
  }
}

int row_slice_copy(const RowSlice* table_dev, int n, long long max_row_bytes, char* rec, int row, bool gather, cudaStream_t st) {
  if (n <= 0) return B200_OK;
  if (n > 65535) B200_FAIL(B200_ERR_INVALID, "row_slice_copy: %d slices", n);
  const unsigned gx = (unsigned)std::min<long long>(std::max<long long>(ceil_div64(max_row_bytes, 16 * 256), 1), 256);
  B200_LAUNCH(row_slice_copy_kernel, dim3(gx, n), 256, 0, st, table_dev, rec, row, gather ? 1 : 0);
  return check_launch("row_slice_copy");
}

int encode_tiled(CUtensorMap* m, CUtensorMapDataType type, cuuint32_t rank, const void* base, const cuuint64_t* dims,
                 const cuuint64_t* strides, const cuuint32_t* box, const cuuint32_t* estr, const char* what) {
  typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static EncodeTiledFn encode = nullptr;
  if (!encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    B200_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    if (!fn || qres != cudaDriverEntryPointSuccess) B200_FAIL(B200_ERR_CUDA, "cuTensorMapEncodeTiled not available");
    encode = reinterpret_cast<EncodeTiledFn>(fn);
  }
  const CUresult r = encode(m, type, rank, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) B200_FAIL(B200_ERR_CUDA, "%s: cuTensorMapEncodeTiled failed (%d)", what, (int)r);
  return B200_OK;
}

int act_map(CUtensorMap* m, const void* base, long long ld, int rows, int cols, int box_rows, int elem_bytes) {
  const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)ld * elem_bytes};
  const cuuint32_t box[2] = {(cuuint32_t)(128 / elem_bytes), (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  return encode_tiled(m, elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, base, dims, strides, box,
                      estr, "activation map");
}

int num_sms() {
  static int sms = 0;
  int dev = 0;
  if (!sms && cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}

}  // namespace b200

extern "C" {
const char* b200_last_error(void) { return b200::g_err; }
int b200_abi_version(void) { return B200_ABI_VERSION; }
int64_t b200_launch_count(void) { return b200::g_launches.load(); }
}
