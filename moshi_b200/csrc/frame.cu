// One dialogue frame for every session slot of a GPU, host buffers in and out, one host synchronisation.
//
// This is the per-frame body of the reference's callers, moved below the C ABI so that the masks, the
// Mimi -> LM -> Mimi hand-offs and the "is this row's output ready" decision stay on the device:
//   * moshi/moshi/server.py:120-147 (recv_loop: chunk -> mimi.encode -> lm_gen.step -> mimi.decode -> .cpu()),
//     where `main_pcm.cpu()` and `tokens[0, 0, 0].item()` are two blocking D2H reads per frame (:82-86);
//   * rust/moshi-server/batched_asr.py:138-215 (ASRService.step: per-slot update flags -> reset / exec masks ->
//     encode -> step -> host copies), the batched form the Rust server binds through py_basr_module.rs.
// Everything is enqueued on the stream both handles stream on; the only wait is the one before the host reads.
//
// b200_frame_* is the dialogue frame (encode -> step -> decode).  b200_asr_* is ASRService itself (batched_asr.py:100-213) for
// the speech-to-text models (dep_q = 0, extra heads): per-slot client state and end-of-stream countdown on the device, encode ->
// step_with_extra_heads, no decoder.
#include <algorithm>
#include <string>

#include "common.cuh"

namespace b200 {
namespace {

// ClientState of every slot (batched_asr.py:85-98), one array per field.
struct AsrSlots {
  uint8_t* active;
  uint8_t* complete;
  int64_t* offset;
  int64_t* real_end;
};

// Slot updates -> client state, flags and the reset / exec masks (batched_asr.py:142-177).  flags[b] is the MaskFlags value the
// reference assigns to flags_out[b], flags[B + b] = 1 where it assigns one at all: a slot it leaves alone keeps the caller's value.
__global__ void asr_updates_kernel(const int32_t* __restrict__ updates, AsrSlots s, uint8_t* __restrict__ flags,
                                   uint8_t* __restrict__ reset, uint8_t* __restrict__ exec, int B, int asr_delay) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int u = updates[b];
  uint8_t f = 0, written = 1, r = 0;
  if (u == B200_SLOT_IDLE) {
    s.active[b] = 0;
  } else if (u == B200_SLOT_ACTIVE) {
    s.active[b] = 1;
    f = B200_ASR_ACTIVE;
  } else if (u == B200_SLOT_RESET) {           // ClientState.reset(), then active
    s.complete[b] = 0; s.offset[b] = 0; s.real_end[b] = 0; s.active[b] = 1;
    f = B200_ASR_ACTIVE;
    r = 1;
  } else if (u > 0) {                          // end-of-stream marker: `u` more steps, the ASR delay and 2 frames of padding
    s.complete[b] = 1;
    s.real_end[b] = s.offset[b] + u + asr_delay + 2;
    f = B200_ASR_MARKER_RECEIVED;
  } else {
    written = 0;
  }
  flags[b] = f;
  flags[B + b] = written;
  reset[b] = r;
  exec[b] = s.active[b];
}

// After the step (batched_asr.py:196-213): extra[b][i] = heads[i][b][0] as f32 (extra_heads_stacked[:, :, 0, 0].T), then every
// active slot advances; a slot whose marker has run out becomes inactive with IS_EOS.
__global__ void asr_finish_kernel(const __nv_bfloat16* __restrict__ heads, int n_heads, int model_rows, int head_dim,
                                  float* __restrict__ extra, AsrSlots s, uint8_t* __restrict__ flags, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  for (int i = 0; i < n_heads; ++i) extra[(size_t)b * n_heads + i] = bf2f(heads[((size_t)i * model_rows + b) * head_dim]);
  if (!s.active[b]) return;
  const int64_t off = s.offset[b] + 1;
  s.offset[b] = off;
  if (s.complete[b] && off >= s.real_end[b]) {
    s.active[b] = 0;
    flags[b] = B200_ASR_IS_EOS;
    flags[B + b] = 1;
  }
}

// Slot updates -> reset / exec masks (batched_asr.py:146-177 builds them on the host and copies three tensors).
__global__ void frame_masks_kernel(const int32_t* __restrict__ updates, uint8_t* __restrict__ active, uint8_t* __restrict__ reset,
                                   uint8_t* __restrict__ exec, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int u = updates[b];
  uint8_t a = active[b];
  uint8_t r = 0;
  if (u == B200_SLOT_IDLE) a = 0;
  else if (u == B200_SLOT_ACTIVE) a = 1;
  else if (u == B200_SLOT_RESET) { a = 1; r = 1; }
  // u > 0: an end-of-stream marker (batched_asr.py:161-170) leaves the slot's activity as it is
  active[b] = a;
  reset[b] = r;
  exec[b] = a;
}

// LMGen.step output -> the decoder's codes and its exec mask.  A row whose output is not ready yet (-2, lm.py:779-782:
// fewer than max_delay + 1 steps since its reset, or not executing) must not advance the decoder's streaming state:
// the reference server simply does not call mimi.decode until step() stops returning None (server.py:139-142).
__global__ void frame_decode_inputs_kernel(const int64_t* __restrict__ tokens, const uint8_t* __restrict__ exec, int64_t* __restrict__ codes,
                                           uint8_t* __restrict__ dec_exec, uint8_t* __restrict__ ready, int B, int dep_q) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int64_t* t = tokens + (size_t)b * (dep_q + 1);
  bool ok = exec[b] != 0;
  for (int k = 0; k <= dep_q; ++k) ok = ok && t[k] >= 0;
  for (int k = 0; k < dep_q; ++k) codes[(size_t)b * dep_q + k] = ok ? t[1 + k] : 0;
  dec_exec[b] = ok ? 1 : 0;
  ready[b] = ok ? 1 : 0;
}

// PCM of rows without a decoded frame is silence, not whatever the masked decoder left in the buffer.
__global__ void frame_silence_kernel(float* __restrict__ pcm, const uint8_t* __restrict__ ready, int frame) {
  if (ready[blockIdx.x]) return;
  for (int i = threadIdx.x; i < frame; i += blockDim.x) pcm[(size_t)blockIdx.x * frame + i] = 0.f;
}

}  // namespace
}  // namespace b200

using namespace b200;

struct b200_frame {
  b200_mimi* mimi = nullptr;
  b200_lm* lm = nullptr;
  int device = -1;                   // the LM handle's: every entry point makes it current
  int B = 0, dep_q = 0, n_in = 0, frame = 0, noise_row = 0;
  cudaStream_t stream = nullptr;
  Arena mem;                         // the buffers below
  // device
  float* pcm_in = nullptr; float* pcm_out = nullptr; float* noise = nullptr;
  int64_t* codes_in = nullptr; int64_t* tokens = nullptr; int64_t* codes_out = nullptr;
  int32_t* updates = nullptr;
  uint8_t* active = nullptr; uint8_t* reset = nullptr; uint8_t* exec = nullptr; uint8_t* dec_exec = nullptr; uint8_t* ready = nullptr;
  // pinned host staging
  float* h_pcm_in = nullptr; float* h_pcm_out = nullptr; float* h_noise = nullptr;
  int64_t* h_tokens = nullptr; int32_t* h_updates = nullptr; uint8_t* h_ready = nullptr;
  cudaEvent_t done = nullptr;
  std::vector<uint8_t> h_active;     // host mirror of `active` (only to skip a frame in which no slot executes)
};

struct b200_asr {
  b200_mimi* mimi = nullptr;
  b200_lm* lm = nullptr;
  int device = -1;                   // the LM handle's: every entry point makes it current
  Arena mem;                         // the buffers below
  int B = 0, n_codes = 0, n_user = 0, frame = 0, asr_delay = 0, n_heads = 0;   // n_codes: the codec's, n_user: the LM's n_q - dep_q
  cudaStream_t stream = nullptr;
  // device
  float* pcm_in = nullptr; float* extra = nullptr;
  int64_t* codes_in = nullptr; int64_t* codes_lm = nullptr; int64_t* tokens = nullptr;
  int32_t* updates = nullptr;
  uint8_t* flags = nullptr; uint8_t* reset = nullptr; uint8_t* exec = nullptr; uint8_t* all_rows = nullptr;
  AsrSlots slots{};
  // pinned host staging
  float* h_pcm_in = nullptr; float* h_extra = nullptr; int64_t* h_tokens = nullptr; int32_t* h_updates = nullptr; uint8_t* h_flags = nullptr;
  cudaEvent_t done = nullptr;
  std::vector<uint8_t> h_active;     // host mirror of ClientState.active (only to skip a frame in which no slot executes)
};

namespace {

// Exec masks -> mimi.encode -> lm_gen.step_with_extra_heads (batched_asr.py:182-197), enqueued on the handles' stream.
int asr_run(b200_asr* a, const uint8_t* exec) {
  B200_TRY(b200_lm_set_exec_mask(a->lm, exec));
  B200_TRY(b200_mimi_set_exec_mask(a->mimi, exec));
  B200_TRY(b200_mimi_encode(a->mimi, a->pcm_in, 1, a->codes_in));
  const int64_t* codes = a->codes_in;
  if (a->n_codes > a->n_user) {      // the step reads the first n_q - dep_q codebooks (lm.py:688-689)
    B200_CUDA(cudaMemcpy2DAsync(a->codes_lm, (size_t)a->n_user * 8, a->codes_in, (size_t)a->n_codes * 8, (size_t)a->n_user * 8,
                                (size_t)a->B, cudaMemcpyDeviceToDevice, a->stream));
    codes = a->codes_lm;
  }
  int ready = 0;                     // always 1: b200_asr_create refuses models with delays
  return b200_lm_step(a->lm, codes, a->n_user, nullptr, a->tokens, /*support_out_of_sync=*/0, &ready);
}

int asr_init(b200_asr* a) {
  const size_t B = (size_t)a->B;
  Arena& m = a->mem;
  B200_TRY(m.alloc_t(&a->pcm_in, B * a->frame, false));
  B200_TRY(m.alloc_t(&a->extra, B * std::max(a->n_heads, 1), false));
  B200_TRY(m.alloc_t(&a->codes_in, B * a->n_codes, false));
  B200_TRY(m.alloc_t(&a->codes_lm, B * a->n_user, false));
  B200_TRY(m.alloc_t(&a->tokens, B, false));
  B200_TRY(m.alloc_t(&a->updates, B, false));
  B200_TRY(m.alloc_t(&a->flags, 2 * B, false));
  B200_TRY(m.alloc_t(&a->reset, B, false));
  B200_TRY(m.alloc_t(&a->exec, B, false));
  B200_TRY(m.alloc_t(&a->all_rows, B, false));
  B200_TRY(m.alloc_t(&a->slots.active, B, false));
  B200_TRY(m.alloc_t(&a->slots.complete, B, false));
  B200_TRY(m.alloc_t(&a->slots.offset, B, false));
  B200_TRY(m.alloc_t(&a->slots.real_end, B, false));
  B200_TRY(m.alloc_host(&a->h_pcm_in, B * a->frame));
  B200_TRY(m.alloc_host(&a->h_extra, B * std::max(a->n_heads, 1)));
  B200_TRY(m.alloc_host(&a->h_tokens, B));
  B200_TRY(m.alloc_host(&a->h_updates, B));
  B200_TRY(m.alloc_host(&a->h_flags, 2 * B));
  B200_CUDA(cudaEventCreateWithFlags(&a->done, cudaEventDisableTiming));
  cudaStream_t st = a->stream;
  B200_CUDA(cudaMemsetAsync(a->all_rows, 1, B, st));
  B200_CUDA(cudaMemsetAsync(a->exec, 0, B, st));
  B200_CUDA(cudaMemsetAsync(a->reset, 0, B, st));
  B200_CUDA(cudaMemsetAsync(a->flags, 0, 2 * B, st));
  B200_CUDA(cudaMemsetAsync(a->extra, 0, B * std::max(a->n_heads, 1) * 4, st));
  B200_CUDA(cudaMemsetAsync(a->tokens, 0, B * 8, st));
  // ClientState() for every slot: inactive, no marker
  B200_CUDA(cudaMemsetAsync(a->slots.active, 0, B, st));
  B200_CUDA(cudaMemsetAsync(a->slots.complete, 0, B, st));
  B200_CUDA(cudaMemsetAsync(a->slots.offset, 0, B * 8, st));
  B200_CUDA(cudaMemsetAsync(a->slots.real_end, 0, B * 8, st));
  // warm-up (batched_asr.py:119-130): three frames of silence with every row executing
  B200_CUDA(cudaMemsetAsync(a->pcm_in, 0, B * a->frame * 4, st));
  for (int i = 0; i < 3; ++i) B200_TRY(asr_run(a, a->all_rows));
  a->h_active.assign(B, 0);
  B200_CUDA(cudaStreamSynchronize(st));
  return lm_check_kv_pool(a->lm);
}

int frame_init(b200_frame* f) {
  const size_t B = (size_t)f->B;
  Arena& m = f->mem;
  B200_TRY(m.alloc_t(&f->pcm_in, B * f->frame, false));
  B200_TRY(m.alloc_t(&f->pcm_out, B * f->frame, false));
  B200_TRY(m.alloc_t(&f->noise, B * std::max(f->noise_row, 1), false));
  B200_TRY(m.alloc_t(&f->codes_in, B * f->n_in, false));
  B200_TRY(m.alloc_t(&f->tokens, B * (f->dep_q + 1), false));
  B200_TRY(m.alloc_t(&f->codes_out, B * f->dep_q, false));
  B200_TRY(m.alloc_t(&f->updates, B, false));
  B200_TRY(m.alloc_t(&f->active, B, false));
  B200_TRY(m.alloc_t(&f->reset, B, false));
  B200_TRY(m.alloc_t(&f->exec, B, false));
  B200_TRY(m.alloc_t(&f->dec_exec, B, false));
  B200_TRY(m.alloc_t(&f->ready, B, false));
  B200_CUDA(cudaMemsetAsync(f->active, 1, B, f->stream));          // streaming() starts with every row executing (streaming.py:31-33)
  B200_CUDA(cudaMemsetAsync(f->exec, 1, B, f->stream));
  B200_CUDA(cudaMemsetAsync(f->reset, 0, B, f->stream));
  B200_TRY(m.alloc_host(&f->h_pcm_in, B * f->frame));
  B200_TRY(m.alloc_host(&f->h_pcm_out, B * f->frame));
  B200_TRY(m.alloc_host(&f->h_noise, B * std::max(f->noise_row, 1)));
  B200_TRY(m.alloc_host(&f->h_tokens, B * (f->dep_q + 1)));
  B200_TRY(m.alloc_host(&f->h_updates, B));
  B200_TRY(m.alloc_host(&f->h_ready, B));
  B200_CUDA(cudaEventCreateWithFlags(&f->done, cudaEventDisableTiming));
  return B200_OK;
}

}  // namespace

extern "C" {

int b200_frame_create(b200_mimi* mimi, b200_lm* lm, int batch, int n_codebooks, int dep_q, int frame_size, void* stream,
                      b200_frame** out) {
  if (!mimi || !lm || !out || batch <= 0 || n_codebooks <= 0 || dep_q <= 0 || frame_size <= 0)
    B200_FAIL(B200_ERR_INVALID, "frame_create: bad arguments");
  if (n_codebooks != dep_q)
    B200_FAIL(B200_ERR_SHAPE, "frame_create: the decoder takes the dep_q generated codebooks (%d), the codec has %d", dep_q, n_codebooks);
  auto* f = new b200_frame();
  f->mimi = mimi; f->lm = lm; f->device = lm_device(lm);
  f->B = batch; f->dep_q = dep_q; f->n_in = n_codebooks; f->frame = frame_size;
  f->stream = static_cast<cudaStream_t>(stream);
  f->noise_row = b200_lm_noise_per_row(lm);
  f->h_active.assign((size_t)batch, 1);
  DeviceGuard g(f->device);
  const int rc = frame_init(f);
  if (rc != B200_OK) {
    const std::string msg = b200_last_error();
    b200_frame_destroy(f);
    B200_FAIL(rc, "%s", msg.c_str());
  }
  *out = f;
  return B200_OK;
}

int b200_frame_destroy(b200_frame* f) {
  if (!f) return B200_OK;
  DeviceGuard g(f->device);
  if (f->done) cudaEventDestroy(f->done);
  delete f;
  return B200_OK;
}

int b200_frame_read_buffer(b200_frame* f, const char* name, void* dst_dev, int64_t capacity_bytes, int64_t* nbytes) {
  if (!f || !name) B200_FAIL(B200_ERR_INVALID, "frame_read_buffer: null argument");
  DeviceGuard g(f->device);
  const std::string n = name;
  const size_t B = (size_t)f->B;
  const void* src = nullptr; int64_t sz = 0;
  if (n == "codes_in") { src = f->codes_in; sz = (int64_t)(B * f->n_in * 8); }
  else if (n == "codes_out") { src = f->codes_out; sz = (int64_t)(B * f->dep_q * 8); }
  else if (n == "tokens") { src = f->tokens; sz = (int64_t)(B * (f->dep_q + 1) * 8); }
  else if (n == "exec") { src = f->exec; sz = (int64_t)B; }
  else if (n == "decoder_exec") { src = f->dec_exec; sz = (int64_t)B; }
  else B200_FAIL(B200_ERR_INVALID, "frame_read_buffer: unknown buffer '%s'", name);
  return copy_out(src, sz, sz, dst_dev, capacity_bytes, nbytes, f->stream, "frame_read_buffer");
}

int b200_frame_step(b200_frame* f, const float* pcm_in_host, const int32_t* updates_host, const float* noise_host,
                    const float* noise_dev, float* pcm_out_host, int64_t* tokens_out_host, uint8_t* ready_out_host) {
  if (!f || !pcm_in_host || !pcm_out_host || !tokens_out_host) B200_FAIL(B200_ERR_INVALID, "frame_step: null buffers");
  DeviceGuard g(f->device);
  const size_t B = (size_t)f->B;
  cudaStream_t st = f->stream;
  memcpy(f->h_pcm_in, pcm_in_host, B * f->frame * 4);
  B200_CUDA(cudaMemcpyAsync(f->pcm_in, f->h_pcm_in, B * f->frame * 4, cudaMemcpyHostToDevice, st));
  if (noise_host && f->noise_row > 0) {
    memcpy(f->h_noise, noise_host, B * f->noise_row * 4);
    B200_CUDA(cudaMemcpyAsync(f->noise, f->h_noise, B * f->noise_row * 4, cudaMemcpyHostToDevice, st));
  }
  if (updates_host) {
    bool any_reset = false, all_idle = true;
    for (size_t b = 0; b < B; ++b) {
      const int32_t u = updates_host[b];
      if (u < B200_SLOT_RESET) B200_FAIL(B200_ERR_INVALID, "frame_step: unknown slot update %d for slot %zu", (int)u, b);
      any_reset |= u == B200_SLOT_RESET;
      if (u == B200_SLOT_IDLE) f->h_active[b] = 0;
      else if (u < 0) f->h_active[b] = 1;
      all_idle &= f->h_active[b] == 0;
      f->h_updates[b] = u;
    }
    B200_CUDA(cudaMemcpyAsync(f->updates, f->h_updates, B * 4, cudaMemcpyHostToDevice, st));
    B200_LAUNCH(frame_masks_kernel, (unsigned)((B + 127) / 128), 128, 0, st, f->updates, f->active, f->reset, f->exec, (int)B);
    B200_TRY(check_launch("frame_masks"));
    if (any_reset) {                  // batched_asr.py:179-181
      B200_TRY(b200_lm_reset(f->lm, f->reset));
      B200_TRY(b200_mimi_reset(f->mimi, f->reset));
    }
    if (all_idle) {                   // skip_exec (batched_asr.py:183-184): nothing runs, nothing is ready
      B200_CUDA(cudaStreamSynchronize(st));
      if (ready_out_host) memset(ready_out_host, 0, B);
      memset(pcm_out_host, 0, B * f->frame * 4);
      for (size_t i = 0; i < B * (f->dep_q + 1); ++i) tokens_out_host[i] = -2;      // ungenerated_token_id (lm.py:779-782)
      return B200_OK;
    }
  }
  B200_TRY(b200_lm_set_exec_mask(f->lm, f->exec));
  B200_TRY(b200_mimi_set_exec_mask(f->mimi, f->exec));
  B200_TRY(b200_mimi_encode(f->mimi, f->pcm_in, 1, f->codes_in));
  int ready_all = 0;
  B200_TRY(b200_lm_step(f->lm, f->codes_in, f->n_in, noise_host ? f->noise : noise_dev, f->tokens, /*support_out_of_sync=*/1, &ready_all));
  B200_LAUNCH(frame_decode_inputs_kernel, (unsigned)((B + 127) / 128), 128, 0, st, f->tokens, f->exec, f->codes_out, f->dec_exec, f->ready,
              (int)B, f->dep_q);
  B200_TRY(check_launch("frame_decode_inputs"));
  B200_TRY(b200_mimi_set_exec_mask(f->mimi, f->dec_exec));
  B200_TRY(b200_mimi_decode(f->mimi, f->codes_out, f->dep_q, 1, f->pcm_out));
  B200_LAUNCH(frame_silence_kernel, (unsigned)B, 256, 0, st, f->pcm_out, f->ready, f->frame);
  B200_TRY(check_launch("frame_silence"));
  B200_CUDA(cudaMemcpyAsync(f->h_tokens, f->tokens, B * (f->dep_q + 1) * 8, cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaMemcpyAsync(f->h_pcm_out, f->pcm_out, B * f->frame * 4, cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaMemcpyAsync(f->h_ready, f->ready, B, cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaEventRecord(f->done, st));
  B200_CUDA(cudaEventSynchronize(f->done));           // the frame's only host wait
  memcpy(tokens_out_host, f->h_tokens, B * (f->dep_q + 1) * 8);
  memcpy(pcm_out_host, f->h_pcm_out, B * f->frame * 4);
  if (ready_out_host) memcpy(ready_out_host, f->h_ready, B);
  return lm_check_kv_pool(f->lm);
}

int b200_asr_create(b200_mimi* mimi, b200_lm* lm, int batch, int asr_delay_in_tokens, void* stream, b200_asr** out) {
  if (!mimi || !lm || !out || batch <= 0) B200_FAIL(B200_ERR_INVALID, "asr_create: bad arguments");
  MimiFrameView mv{};
  LmFrameView lv{};
  B200_TRY(mimi_frame_view(mimi, &mv));
  B200_TRY(lm_frame_view(lm, &lv));
  if (lv.dep_q != 0)
    B200_FAIL(B200_ERR_INVALID, "asr_create: the speech-to-text service runs models without depformer (dep_q = 0), got dep_q = %d", lv.dep_q);
  if (mv.num_codebooks < lv.n_q - lv.dep_q)
    B200_FAIL(B200_ERR_INVALID, "asr_create: the LM reads %d codebooks, the codec produces %d", lv.n_q - lv.dep_q, mv.num_codebooks);
  if (mv.batch != batch || lv.batch != batch)
    B200_FAIL(B200_ERR_INVALID, "asr_create: batch %d, but the codec streams %d rows and the LM %d", batch, mv.batch, lv.batch);
  if (lv.max_delay != 0)     // step() would return None for the first frames: the reference's warm-up asserts it does not
    B200_FAIL(B200_ERR_INVALID, "asr_create: the speech-to-text service runs models without delays, got max delay %d", lv.max_delay);
  auto* a = new b200_asr();
  a->mimi = mimi; a->lm = lm; a->device = lm_device(lm); a->B = batch; a->n_codes = mv.num_codebooks; a->n_user = lv.n_q - lv.dep_q; a->frame = mv.frame_size;
  a->asr_delay = asr_delay_in_tokens; a->n_heads = lv.extra_heads;
  a->stream = static_cast<cudaStream_t>(stream);
  DeviceGuard g(a->device);
  const int rc = asr_init(a);
  if (rc != B200_OK) {
    const std::string msg = b200_last_error();
    b200_asr_destroy(a);
    B200_FAIL(rc, "%s", msg.c_str());
  }
  *out = a;
  return B200_OK;
}

int b200_asr_destroy(b200_asr* a) {
  if (!a) return B200_OK;
  DeviceGuard g(a->device);
  cudaStreamSynchronize(a->stream);
  if (a->done) cudaEventDestroy(a->done);
  delete a;
  return B200_OK;
}

int b200_asr_read_buffer(b200_asr* a, const char* name, void* dst_dev, int64_t capacity_bytes, int64_t* nbytes) {
  if (!a || !name) B200_FAIL(B200_ERR_INVALID, "asr_read_buffer: null argument");
  DeviceGuard g(a->device);
  const std::string n = name;
  const size_t B = (size_t)a->B;
  const void* src = nullptr; int64_t sz = 0;
  if (n == "codes_in") { src = a->codes_in; sz = (int64_t)(B * a->n_codes * 8); }
  else if (n == "tokens") { src = a->tokens; sz = (int64_t)(B * 8); }
  else if (n == "extra_heads") { src = a->extra; sz = (int64_t)(B * a->n_heads * 4); }
  else if (n == "exec") { src = a->exec; sz = (int64_t)B; }
  else if (n == "reset") { src = a->reset; sz = (int64_t)B; }
  else if (n == "offset") { src = a->slots.offset; sz = (int64_t)(B * 8); }
  else if (n == "real_end") { src = a->slots.real_end; sz = (int64_t)(B * 8); }
  else B200_FAIL(B200_ERR_INVALID, "asr_read_buffer: unknown buffer '%s'", name);
  return copy_out(src, sz, sz, dst_dev, capacity_bytes, nbytes, a->stream, "asr_read_buffer");
}

int b200_asr_step(b200_asr* a, const float* pcm_in_host, const int32_t* updates_host, uint8_t* flags_inout_host,
                  int64_t* tokens_out_host, float* extra_heads_out_host, int* ran) {
  if (ran) *ran = 0;
  if (!a || !pcm_in_host || !updates_host || !flags_inout_host || !tokens_out_host || (a->n_heads && !extra_heads_out_host))
    B200_FAIL(B200_ERR_INVALID, "asr_step: null buffers");
  DeviceGuard g(a->device);
  MimiFrameView mv{};
  LmFrameView lv{};
  B200_TRY(mimi_frame_view(a->mimi, &mv));
  B200_TRY(lm_frame_view(a->lm, &lv));
  if (mv.batch != a->B || mv.num_codebooks != a->n_codes || lv.batch != a->B)
    B200_FAIL(B200_ERR_STATE, "asr_step: the handles' streaming batch or the codec's codebooks changed since asr_create");
  const size_t B = (size_t)a->B;
  cudaStream_t st = a->stream;
  bool any_reset = false, any_active = false;
  for (size_t b = 0; b < B; ++b) {             // the host mirror of `active`; EOS is merged in below
    const int32_t u = updates_host[b];
    if (u == B200_SLOT_IDLE) a->h_active[b] = 0;
    else if (u == B200_SLOT_ACTIVE || u == B200_SLOT_RESET) a->h_active[b] = 1;
    any_reset |= u == B200_SLOT_RESET;
    any_active |= a->h_active[b] != 0;
  }
  memcpy(a->h_updates, updates_host, B * 4);
  B200_CUDA(cudaMemcpyAsync(a->updates, a->h_updates, B * 4, cudaMemcpyHostToDevice, st));
  B200_LAUNCH(asr_updates_kernel, (unsigned)((B + 127) / 128), 128, 0, st, a->updates, a->slots, a->flags, a->reset, a->exec, (int)B,
              a->asr_delay);
  B200_TRY(check_launch("asr_updates"));
  if (any_reset) {                             // batched_asr.py:175-177
    B200_TRY(b200_lm_reset(a->lm, a->reset));
    B200_TRY(b200_mimi_reset(a->mimi, a->reset));
  }
  if (any_active) {                            // else skip_exec (batched_asr.py:179-180): no step, tokens and extra heads untouched
    memcpy(a->h_pcm_in, pcm_in_host, B * a->frame * 4);
    B200_CUDA(cudaMemcpyAsync(a->pcm_in, a->h_pcm_in, B * a->frame * 4, cudaMemcpyHostToDevice, st));
    B200_TRY(asr_run(a, a->exec));
    B200_LAUNCH(asr_finish_kernel, (unsigned)((B + 127) / 128), 128, 0, st, lv.extra_out, a->n_heads, lv.model_rows, lv.extra_dim,
                a->extra, a->slots, a->flags, (int)B);
    B200_TRY(check_launch("asr_finish"));
    B200_CUDA(cudaMemcpyAsync(a->h_tokens, a->tokens, B * 8, cudaMemcpyDeviceToHost, st));
    if (a->n_heads) B200_CUDA(cudaMemcpyAsync(a->h_extra, a->extra, B * a->n_heads * 4, cudaMemcpyDeviceToHost, st));
  }
  B200_CUDA(cudaMemcpyAsync(a->h_flags, a->flags, 2 * B, cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaEventRecord(a->done, st));
  B200_CUDA(cudaEventSynchronize(a->done));    // the frame's only host wait
  for (size_t b = 0; b < B; ++b) {
    if (!a->h_flags[B + b]) continue;
    flags_inout_host[b] = a->h_flags[b];
    if (a->h_flags[b] == B200_ASR_IS_EOS) a->h_active[b] = 0;
  }
  if (!any_active) return B200_OK;
  memcpy(tokens_out_host, a->h_tokens, B * 8);
  if (a->n_heads) memcpy(extra_heads_out_host, a->h_extra, B * a->n_heads * 4);
  if (ran) *ran = 1;
  return lm_check_kv_pool(a->lm);
}

}  // extern "C"
