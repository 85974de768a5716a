/*
 * moshi_b200 — C ABI of the H100-native (sm_90a) streaming inference path for
 * Mimi (SEANet + transformer bottleneck + split RVQ) and the Moshi LM decode step.
 *
 * The reference (kyutai-labs/moshi) has no native boundary on this path: its Python classes call
 * ATen/cuBLAS/cuDNN directly.  The closest precedent is the PyO3 module `rustymimi`
 * (rust/mimi-pyo3/src/lib.rs:103-236: Tokenizer.encode_step / decode_step / reset).  Each entry
 * point below cites the reference method it stands behind; `moshi_b200/models/*.py` are the
 * Python shims that keep the reference signatures and call these functions through ctypes.
 *
 * Conventions
 *   - plain C, opaque handles, `int` return code (0 = B200_OK); on failure b200_last_error()
 *     returns a thread-local message.  No C++/torch types cross this boundary.
 *   - pointers named *_dev are device pointers on the handle's GPU; *_host are host pointers.
 *     Device entry points enqueue work on the stream given to *_streaming_begin and do not
 *     synchronise; *_host entry points copy in/out through pinned staging buffers and return
 *     after the result is in the caller's buffer (this is the end-to-end path bench.py times).
 *   - a handle is thread-compatible, not thread-safe (same as the reference modules,
 *     moshi/moshi/server.py:160 serialises with one asyncio.Lock).
 *   - masks are one byte per batch row (torch.bool layout), non-zero = true.
 *   - all streaming state (conv left-context, overlap-add partials, KV rings, token ring,
 *     per-row offsets) is owned by the handle between streaming_begin and streaming_end.
 */
#ifndef MOSHI_B200_H
#define MOSHI_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_ABI_VERSION 2

enum {
  B200_OK = 0,
  B200_ERR_INVALID = 1,   /* bad argument / unknown tensor name / unsupported option      */
  B200_ERR_SHAPE = 2,     /* shape or dtype mismatch (reference: AssertionError)          */
  B200_ERR_STATE = 3,     /* call outside streaming, double streaming (reference: RuntimeError / AssertionError) */
  B200_ERR_CUDA = 4,      /* CUDA runtime/driver failure; message carries the CUDA error   */
  B200_ERR_MISSING = 5    /* finalize: a required tensor was never loaded                  */
};

enum { B200_F32 = 0, B200_BF16 = 1, B200_F16 = 2, B200_I64 = 3, B200_U8 = 4, B200_I8 = 5, B200_I32 = 6 };

const char* b200_last_error(void);
int b200_abi_version(void);
/* Number of kernels this library has launched in the calling process (bench.py `gpu_launches`). */
int64_t b200_launch_count(void);

/* ------------------------------------------------------------------------------------------ */
/* Mimi  (reference: moshi/moshi/models/compression.py:97-433, loaders.py:38-88, 323-363)       */
/* ------------------------------------------------------------------------------------------ */

typedef struct b200_mimi b200_mimi;

typedef struct {
  int sample_rate;            /* 24000 */
  float frame_rate;           /* 12.5 */
  int channels;               /* 1 */
  int dimension;              /* 512 */
  int n_filters;              /* 64 */
  int n_residual_layers;      /* 1 */
  int n_ratios;               /* 4 */
  int ratios[8];              /* decoder order: 8,6,5,4 */
  int kernel_size;            /* 7 */
  int residual_kernel_size;   /* 3 */
  int last_kernel_size;       /* 3 */
  int dilation_base;          /* 2 */
  int compress;               /* 2 */
  int tr_d_model;             /* 512 */
  int tr_num_heads;           /* 8 */
  int tr_num_layers;          /* 8 */
  int tr_dim_feedforward;     /* 2048 */
  int tr_context;             /* 250 */
  float tr_max_period;        /* 10000 */
  int q_dimension;            /* 256 */
  int q_bins;                 /* 2048 */
  int q_n_q;                  /* 32 codebooks stored */
  int q_n_semantic;           /* 1 */
  int num_codebooks;          /* 8 active (MimiModel.set_num_codebooks) */
} b200_mimi_config;

/* loaders.get_mimi (loaders.py:323-363): build, then feed the state dict tensor by tensor using the
 * reference's key names (SURVEY.md appendix A; legacy names are normalised by the Python shim),
 * then finalize (derives centroids = embedding_sum / clamp(cluster_usage, 1e-5), core_vq.py:181-183,
 * and repacks weights into the kernels' HBM layouts).  Source tensors may be freed after each call. */
int b200_mimi_create(const b200_mimi_config* cfg, b200_mimi** out);
int b200_mimi_load_tensor(b200_mimi* h, const char* name, const void* data_dev, int dtype,
                          int ndim, const int64_t* shape);
int b200_mimi_finalize(b200_mimi* h);
int b200_mimi_destroy(b200_mimi* h);

/* MimiModel.set_num_codebooks (compression.py:263-265 -> vq.py:315-317). */
int b200_mimi_set_num_codebooks(b200_mimi* h, int n);

/* StreamingModule.streaming(batch) enter / exit (streaming.py:131-137). `stream` is a cudaStream_t. */
int b200_mimi_streaming_begin(b200_mimi* h, int batch, void* stream);
int b200_mimi_streaming_end(b200_mimi* h);
/* reset_streaming(reset_mask) (streaming.py:139-156); NULL = all rows. */
int b200_mimi_reset(b200_mimi* h, const uint8_t* reset_mask_dev);
/* set_exec_mask(mask) (streaming.py:183-211). */
int b200_mimi_set_exec_mask(b200_mimi* h, const uint8_t* exec_mask_dev);

/* MimiModel.encode in streaming mode (compression.py:376-388): pcm f32 [B,1,1920*n] -> codes i64 [B,K,n]. */
int b200_mimi_encode(b200_mimi* h, const float* pcm_dev, int n_frames, int64_t* codes_dev);
/* MimiModel._encode_to_unquantized_latent (compression.py:338-374): -> latent f32 [B,512,n]. */
int b200_mimi_encode_to_latent(b200_mimi* h, const float* pcm_dev, int n_frames, float* latent_dev);
/* SplitResidualVectorQuantizer.encode on a caller-provided latent (vq.py:269-279): [B,512,n] -> [B,K,n]. */
int b200_mimi_quantize(b200_mimi* h, const float* latent_dev, int n_frames, int64_t* codes_dev);
/* MimiModel.decode in streaming mode (compression.py:406-429): codes i64 [B,K,n] -> pcm f32 [B,1,1920*n]. */
int b200_mimi_decode(b200_mimi* h, const int64_t* codes_dev, int n_codebooks, int n_frames, float* pcm_dev);
/* MimiModel.decode_latent (compression.py:431-433): codes -> quantized latent f32 [B,512,n]. */
int b200_mimi_decode_latent(b200_mimi* h, const int64_t* codes_dev, int n_codebooks, int n_frames,
                            float* latent_dev);
/* Same as encode / decode with HOST buffers (H2D + D2H inside, returns when the result is ready): what the reference's
 * server does around the two calls, `chunk.to(device)` ... `main_pcm.cpu()` (server.py:80-81, 131-135). */
int b200_mimi_encode_host(b200_mimi* h, const float* pcm_host, int n_frames, int64_t* codes_host);
int b200_mimi_decode_host(b200_mimi* h, const int64_t* codes_host, int n_codebooks, int n_frames,
                          float* pcm_host);
/* StreamingModule.get_streaming_state / set_streaming_state (streaming.py:158-181) as one opaque device blob of
 * b200_mimi_state_bytes() bytes: masks, carried conv samples, overlap-add partials, transformer KV rings, offsets.
 * A snapshot can only be restored into a session with the same batch size and configuration. */
int64_t b200_mimi_state_bytes(b200_mimi* h);
int b200_mimi_get_state(b200_mimi* h, void* dst_dev, int64_t capacity);
int b200_mimi_set_state(b200_mimi* h, const void* src_dev, int64_t nbytes);
/* The same state entry by entry (b200_lm_state_* has the conventions).  Names: "exec_mask" u8 [B]; per SEANet layer
 * "<encoder|decoder>.model.<i>....ext_hi" / ".ext_lo" f32 [B, P + T, Cin]: the layer's extended input, token-major, whose first P
 * rows are StreamingConv1d's `previous` (conv.py:161-169; value = hi + lo; P = 1 for a transposed conv: its previous input step,
 * which determines the reference's `partial`, conv.py:349-361) and whose other T rows are scratch; "downsample.previous" f32
 * [B, C, 2], "downsample.first" u8 [B], "upsample.partial" f32 [B, C, 2]; "<encoder|decoder>_transformer.offset" i64 [B] and
 * ".layers.<i>.k" / ".v" f32 [B, 8, 250, 64]. */
int b200_mimi_state_count(b200_mimi* h);
int b200_mimi_state_entry(b200_mimi* h, int index, const char** name, int* dtype, int* ndim, int64_t* shape8, int64_t* nbytes);
int b200_mimi_state_read(b200_mimi* h, const char* name, void* dst_dev, int64_t nbytes);
int b200_mimi_state_write(b200_mimi* h, const char* name, const void* src_dev, int64_t nbytes);
/* One session (one row) of a Mimi handle, encoder and decoder state, as a device record of b200_mimi_session_bytes bytes
 * (fixed per configuration): the row's slice of every entry above.  Export does not change the source; import replaces row
 * `row` only, after the same checks as b200_lm_session_import (B200_ERR_INVALID: not a record, an LM record, another codec
 * configuration, row outside [0, B); B200_ERR_SHAPE: nbytes differs).  Both synchronise the handle's stream. */
int b200_mimi_session_bytes(b200_mimi* h, int64_t* nbytes);
int b200_mimi_session_export(b200_mimi* h, int row, void* dst_dev, int64_t capacity);
int b200_mimi_session_import(b200_mimi* h, int row, const void* src_dev, int64_t nbytes);
/* Synchronises, returns and clears the device error flags: B200_FLAG_CODE_RANGE = MimiModel.decode was given a code outside
 * [0, bins) (it decodes as the zero vector; the reference indexes out of bounds: "dramatic CUDA crash", vq.py:144-145). */
int b200_mimi_error_flags(b200_mimi* h, int* flags_out);
/* 0 = one launch per kernel, 1 = replay each one-frame encode / decode as a CUDA graph (default 1): the reference's
 * CUDAGraphed wrappers and its NO_CUDA_GRAPH switch (utils/compile.py:169-175, 190-280; compression.py:151-155). */
int b200_mimi_set_graph(b200_mimi* h, int enable);
/* Debug taps: copies a named fp32 intermediate of the last call into dst_dev (capacity in elements;
 * pass dst_dev = NULL to query *numel only).  Names: "enc.<i>", "dec.<i>" = output of SEANet module i
 * ([B,C,T]; the last encoder module is token-major [B,T,C]), "enc.tr", "dec.up", "dec.tr" ([B,T,C]),
 * "enc.latent", "dec.latent" ([B,C]). */
int b200_mimi_read_buffer(b200_mimi* h, const char* name, float* dst_dev, int64_t capacity, int64_t* numel);
/* Bytes of weights + per-step state traffic of one encode+decode frame at the current batch
 * (the algorithmic-bytes figure of DESIGN.md, used for the roofline line in bench.py). */
int64_t b200_mimi_algorithmic_bytes(b200_mimi* h);

/* ------------------------------------------------------------------------------------------ */
/* Moshi LM  (reference: moshi/moshi/models/lm.py:49-850, loaders.py:366-446)                   */
/* ------------------------------------------------------------------------------------------ */

typedef struct b200_lm b200_lm;

typedef struct {
  int dim;                    /* 4096 */
  int text_card;              /* 32000 */
  int n_q;                    /* 16 */
  int dep_q;                  /* 8 */
  int card;                   /* 2048 */
  int num_heads;              /* 32 */
  int num_layers;             /* 32 */
  int ffn_hidden;             /* 11264 = gating.py:52-58 applied to hidden_scale*dim */
  int context;                /* 3000 (= KV ring capacity, transformer.py:466-470) */
  float max_period;           /* 10000 */
  int depformer_dim;          /* 1024 */
  int depformer_num_heads;    /* 16 */
  int depformer_num_layers;   /* 6 */
  int depformer_ffn_hidden;   /* 2816 */
  int delays[33];             /* n_q + 1 entries */
  int quantize;               /* LMModel(quantize=True) (lm.py:107,242-243; utils/quantize.py): every linear is an int8 QLinear,
                                 quantised here from the bf16 weights at load */
  int extra_heads_num_heads;  /* 0 for the dialogue models; the STT models carry nn.Linear(dim, extra_heads_dim) heads on the   */
  int extra_heads_dim;        /* temporal output (lm.py:224-226), read by LMGen.step_with_extra_heads (lm.py:793-807)          */
} b200_lm_config;
/* Family limits: n_q <= 32, 0 <= dep_q <= 16 (dep_q = 0: no depformer, lm.py:219-222), temporal head dim 128, depformer head
 * dim 64, vocabularies < 65535: covers configs/moshi_7b_202409.json, configs/moshi_dev_2b.json and the STT checkpoints.
 * Depformer weight-sharing schedules and low-rank depformer embeddings are set by the two setters below.  Not supported:
 * demux_second_text_stream, text_card_out, depformer_norm, norm_emb, and candle / GGUF-layout checkpoints of models with a
 * schedule or low-rank embeddings (the Python loader refuses them: the candle layout unrolls a schedule into per-step slices). */

/* loaders.get_moshi_lm (loaders.py:366-446). Tensors are bf16 with the reference's key names.  With cfg.quantize a linear may
 * instead arrive pre-quantised, the way `model.q8.safetensors` stores a QLinear (loaders.py:33; utils/quantize.py:16-21):
 * "<linear>.weight" B200_I8 [out, in] (CB) + "<linear>.weight_scb" B200_F32 [out] (SCB, the row absmax); such tensors are
 * tiled as they are, nothing is re-quantised. */
int b200_lm_create(const b200_lm_config* cfg, b200_lm** out);
int b200_lm_load_tensor(b200_lm* h, const char* name, const void* data_dev, int dtype,
                        int ndim, const int64_t* shape);
int b200_lm_finalize(b200_lm* h);
int b200_lm_destroy(b200_lm* h);

/* LMGen(...) sampling arguments (lm.py:556-571). */
int b200_lm_set_sampling(b200_lm* h, int use_sampling, float temp, float temp_text, int top_k,
                         int top_k_text);
/* Per-session sampling settings (the SessionConfigReq of Kyutai's Rust server).  b200_lm_set_session_sampling(h, history) turns
 * them on before streaming_begin: history in [1, 1024] is the length of each session's text-history ring, 0 turns them off.
 * While on, b200_lm_set_row_sampling gives rows rows[0..n) the settings p[0..n) (p NULL: those rows return to the handle-wide
 * values), ordered on the handle's stream before the next step (and before the next b200_frame_step that drives the handle).
 * A row that was never given settings follows b200_lm_set_sampling's values at every step, with pad_mult 0, no penalty.
 * Text token of row b, after the classifier-free-guidance combination: l = float(bf16 logit); each distinct id among the newest
 * repetition_context tokens of the row's history gets l = l >= 0 ? l / repetition_penalty : l * repetition_penalty; a sampling
 * row (use_sampling and temp_text > 0) samples softmax(l / temp_text, with pad_mult added to the score of the padding token 3)
 * over its top_k_text; a greedy row takes the first argmax of the penalised l and ignores pad_mult.  The history holds the
 * row's sampled text tokens of the steps it executed, without 0, 3 and text_card; b200_lm_reset empties it and keeps the
 * settings.  The audio tokens use temp and top_k, with no penalty and no pad bias.  Ranges (else B200_ERR_INVALID and nothing
 * changes): temperatures >= 0 and finite; top_k in [1, handle top_k], top_k_text in [1, handle top_k_text] (the noise row is
 * laid out by the handle's top-k; a row's top-k is also held to the handle's at every step, so settings that arrive through a
 * session record or a state snapshot of a handle with larger values sample as if given the handle's); pad_mult finite;
 * repetition_context in [0, 1024], the window holding at most the `history` tokens the row keeps; repetition_penalty in
 * (0, 1000].  Int32 state entries (the histories) carry dtype B200_I32. */
typedef struct {
  float temp_text, temp;
  int32_t top_k_text, top_k;
  float pad_mult;
  int32_t repetition_context;
  float repetition_penalty;
} b200_row_sampling;
int b200_lm_set_session_sampling(b200_lm* h, int history);
int b200_lm_set_row_sampling(b200_lm* h, const int32_t* rows, int n, const b200_row_sampling* p);
/* LMGen(cfg_coef, cfg_is_masked_until, cfg_is_no_text) (lm.py:556-604): classifier-free guidance.  cfg_coef != 1 makes the
 * model run on 2 * batch rows (lm.py:646-647), the second half with the text stream zeroed (cfg_is_no_text) and / or every
 * stream zeroed until a per-session step (masked_until_host i64 [n = batch], NULL = not used) (lm.py:714-726); the logits
 * the samplers read are logits_null + (logits - logits_null) * cfg_coef (lm.py:728-732, 828-833).  Before streaming_begin. */
int b200_lm_set_cfg(b200_lm* h, float cfg_coef, int cfg_is_no_text, const int64_t* masked_until_host, int n);
/* _LMGenState.condition_sum (lm.py:616-626 -> forward_text lm.py:398-399): fuser.get_sum(condition_tensors) cast to bf16,
 * [rows = batch (2 * batch with CFG)][dim], added to the summed input embeddings of every step.  NULL switches it off.
 * While streaming; the tensor is copied.  (Evaluating the conditioners themselves is per-session work outside the step.) */
int b200_lm_set_condition_sum(b200_lm* h, const void* sum_bf16_dev, int rows);
/* Cross-attention conditioning (LMModel(cross_attention=True), transformer.py:727-732, 779-798): every temporal layer runs
 * x = x + cross_attention(norm_cross(x), condition) between its self-attention and its MLP, the query from x, keys and values
 * from a per-row condition memory.  Before finalize; the layers then need "transformer.layers.<i>.cross_attention.in_projs.0
 * .weight" [3*dim,dim], ".cross_attention.out_projs.0.weight" [dim,dim] and ".norm_cross.weight" / ".norm_cross.bias" [dim].
 * Not with quantize (B200_ERR_INVALID). */
int b200_lm_set_cross_attention(b200_lm* h, int enable);
/* LMModel(depformer_weights_per_step_schedule=...) (lm.py:125-127, 172-181; transformer.py:291-316, 399-401): depformer sub-step
 * k runs weight set schedule[k] of "depformer_in.<j>", and of every layer's "self_attn.in_projs.<j>", "self_attn.out_projs.<j>"
 * and "gating.<j>.*"; the checkpoint holds n_sets = max(schedule) + 1 of each, resident once.  n = dep_q entries in
 * [0, dep_q); n = 0: no schedule (one set per sub-step).  After b200_lm_create and before the
 * first b200_lm_load_tensor (B200_ERR_STATE after); B200_ERR_INVALID on a bad schedule. */
int b200_lm_set_depformer_schedule(b200_lm* h, const int* schedule, int n);
/* LMModel(depformer_low_rank_embeddings=rank) (lm.py:186-196; lm_utils.py:80-124): "depformer_text_emb.weight" [text_card+1,
 * rank], "depformer_emb.<i>.weight" [card+1, rank], each with ".low_rank.weight" [depformer_dim, rank].  Finalize expands every
 * table to the full-rank [V, depformer_dim] rows the step reads, row t = bf16(low_rank . e_t) with fp32 accumulation (under
 * quantize the QLinear product: row-wise int8 of e_t and of low_rank, int32 sums), and releases the factors.  rank in
 * [1, 4096]; 0 = full-rank tables; ignored on a model without a depformer (dep_q = 0).  The factors must be bf16: the
 * pre-quantised form of a q8 checkpoint (int8 ".low_rank.weight" + "_scb") is refused at finalize (B200_ERR_INVALID).  Same
 * timing and errors as b200_lm_set_depformer_schedule. */
int b200_lm_set_depformer_low_rank(b200_lm* h, int rank);
/* Keys T of every row's condition memory (k_cross / v_cross bf16 [MB,H,T,128] per layer, allocated at streaming_begin).
 * Before streaming_begin; a cross-attention handle cannot stream without it. */
int b200_lm_set_cross_len(b200_lm* h, int keys);
/* _MHAState.k_cross / v_cross of model rows rows_host[0..n_rows) (b, and batch + b under CFG): K and V = condition @
 * in_projs.0.weight[dim:]^T of every layer (transformer.py:495-505) for condition bf16 [n_rows,T,dim] (fuser.get_cross of
 * lm.py:616-627, one row per model row).  rows_host NULL: all MB rows, n_rows = MB.  While streaming, on the handle's stream,
 * outside the step; the other rows' memory and every row's position are unchanged (a reset keeps the memory). */
int b200_lm_set_condition_cross(b200_lm* h, const void* src_bf16_dev, const int32_t* rows_host, int n_rows);
/* Seed of the Exp(1) noise the step draws itself when the caller passes noise = NULL with sampling on (sampling.py:44 draws
 * it from torch's generator; here a Philox4x32-10 stream keyed by (seed, step counter) inside the step's CUDA graph). */
int b200_lm_seed_noise(b200_lm* h, uint64_t seed);
/* Stream the next calls are ordered on (default: the one given to streaming_begin). */
int b200_lm_set_stream(b200_lm* h, void* stream);
/* LMGen.streaming(batch) enter / exit (lm.py:604-666): allocates token ring, KV rings, offsets. */
int b200_lm_streaming_begin(b200_lm* h, int batch, void* stream);
int b200_lm_streaming_end(b200_lm* h);
/* _LMGenState.reset (lm.py:537-542) incl. the host step counter quirk (offset_cpu = 0). */
int b200_lm_reset(b200_lm* h, const uint8_t* reset_mask_dev);
int b200_lm_set_exec_mask(b200_lm* h, const uint8_t* exec_mask_dev);
/* Floats of Exp(1) noise one step consumes per batch row: min(top_k_text, text_card) +
 * dep_q * min(top_k, card), in the draw order of the reference (sampling.py:44). */
int b200_lm_noise_per_row(b200_lm* h);

/* LMGen.step (lm.py:785-791 -> _step :668-783).
 *   in_codes_dev  i64 [B, n_in] (n_in >= n_q - dep_q; extra columns ignored, lm.py:688-689)
 *   noise_dev     f32 [B, b200_lm_noise_per_row] Exp(1) draws in the reference's order, or NULL: drawn inside the step
 *                 (b200_lm_seed_noise); ignored when use_sampling == 0
 *   out_tokens_dev i64 [B, dep_q + 1] (row 0 text, 1.. audio; -2 = not ready for that row)
 *   *ready_host   0 while the reference would return None (offset_cpu <= max_delay), else 1
 *   support_out_of_sync: LMGen(support_out_of_sync=...) (lm.py:774-776) */
int b200_lm_step(b200_lm* h, const int64_t* in_codes_dev, int n_in, const float* noise_dev,
                 int64_t* out_tokens_dev, int support_out_of_sync, int* ready_host);
/* LMGen.step(input_tokens, depformer_replace_tokens) (lm.py:668-669, 751-755: the TTS caller forces the audio tokens of a
 * frame): replace_audio_dev i64 [B, dep_q] or NULL; when given, the depformer does not run and the text token is still
 * sampled from the temporal transformer. */
int b200_lm_step_ex(b200_lm* h, const int64_t* in_codes_dev, int n_in, const float* noise_dev, const int64_t* replace_audio_dev,
                    int64_t* out_tokens_dev, int support_out_of_sync, int* ready_host);
int b200_lm_step_host(b200_lm* h, const int64_t* in_codes_host, int n_in, const float* noise_host,
                      int64_t* out_tokens_host, int support_out_of_sync, int* ready_host);
/* Hook / debug taps of the last step, copied into dst_dev (capacity in bytes; NULL = query size); MB = rows the model ran
 * on (B, or 2B with CFG):  "text_logits" bf16 [B,text_card] (what LMGen.on_text_logits_hook sees: guided under CFG),
 * "transformer_out" bf16 [MB,dim], "dep_logits" bf16 [dep_q,B,card], "input_tokens" i64 [MB,n_q+1], "text_token" i64 [B],
 * "audio_tokens" i64 [dep_q,B], "noise" f32 [B,b200_lm_noise_per_row] (the Exp(1) draws the samplers read: the step's own
 * draws, or the caller's copy), "extra_heads" bf16 [n_heads,MB,extra_heads_dim] (softmax(extra_head(transformer_out)),
 * lm.py:803-806), "model_text_logits" bf16 [MB,text_card], "model_dep_logits" bf16 [dep_q,MB,card], "dep_in" bf16
 * [MB,n_sets,depformer_dim] (depformer_in[j](transformer_out) for every weight set j; n_sets = dep_q without a schedule, and
 * sub-step k reads set schedule[k]), "depformer.layers.<l>.k" / ".v" bf16 [MB,depformer_heads,dep_q,64] (layer l's per-frame
 * cache: every sub-step's key / value after the frame), "depformer.tables.<k>" bf16 [V,depformer_dim] (sub-step k's embedding
 * table as the step reads it, V = text_card + 1 for k = 0 and card + 1 after: a low-rank table after its expansion).  With the taps on
 * (b200_lm_set_taps), the temporal transformer of the last step: "temporal.embed" bf16 [MB,dim] (the summed input embeddings
 * entering layer 0) and per layer l "temporal.layers.<l>.attn_out" bf16 [MB,dim] (the attention output, before out_proj),
 * ".x_attn" [MB,dim] (x after the attention residual), ".gated" [MB,ffn_hidden] (silu(gate) * value) and ".x_out" [MB,dim]
 * (x after the MLP residual); on a cross-attention handle also ".cross_out" [MB,dim] (the cross-attention output, before its
 * out_proj) and ".x_cross" [MB,dim] (x after the cross-attention residual); B200_ERR_STATE if the taps were never turned on
 * while streaming. */
int b200_lm_read_buffer(b200_lm* h, const char* name, void* dst_dev, int64_t capacity_bytes, int64_t* nbytes);
/* Test taps of the temporal transformer (read through b200_lm_read_buffer "temporal.*"): when on, every step also copies the
 * embeddings and each layer's four activations into per-layer buffers, on the step's stream.  Needs streaming; the buffers
 * are allocated at the first enable and freed at b200_lm_streaming_end.  Turning them on or off drops the captured step graph
 * (it is captured again at the next step); off, the step launches exactly what it launches without this call. */
int b200_lm_set_taps(b200_lm* h, int enable);
/* LMGen.get_streaming_state / set_streaming_state: token ring, per-row offsets, exec mask, the temporal KV rings
 * (1.573 GB per session at full context) and the host step counter, as one opaque device blob. */
int64_t b200_lm_state_bytes(b200_lm* h);
int b200_lm_get_state(b200_lm* h, void* dst_dev, int64_t capacity);
int b200_lm_set_state(b200_lm* h, const void* src_dev, int64_t nbytes);
/* The same state entry by entry, so that the Python shim can present the reference's per-module State objects
 * (streaming.py:158-181; _LMGenState lm.py:523-547, RingKVCache transformer.py:196-288).  Names: "exec_mask" u8 [B], "cache" i64
 * [B,n_q+1,max_delay+2], "offsets" i64 [B], "model.offset" i64 [MB], "model.exec_mask" u8 [MB] (CFG only), "noise_counter",
 * "layers.<i>.k" / ".v" bf16 [MB,H,context,128] (8-bit rings: ".k8" / ".v8" u8 + ".k_scale" / ".v_scale" f32 [MB,H,context]).
 * shape8 receives up to 8 extents.  read / write copy one entry device-to-device on the handle's stream. */
int b200_lm_state_count(b200_lm* h);
int b200_lm_state_entry(b200_lm* h, int index, const char** name, int* dtype, int* ndim, int64_t* shape8, int64_t* nbytes);
int b200_lm_state_read(b200_lm* h, const char* name, void* dst_dev, int64_t nbytes);
int b200_lm_state_write(b200_lm* h, const char* name, const void* src_dev, int64_t nbytes);
/* _LMGenState.offset_cpu (lm.py:529): the host step counter behind "step() returns None while offset_cpu <= max_delay". */
int64_t b200_lm_get_offset_cpu(b200_lm* h);
int b200_lm_set_offset_cpu(b200_lm* h, int64_t value);
/* Synchronises the handle's stream, returns and clears the device error flags.  The kernels never read out of bounds:
 * a token id outside its embedding table (anything but [0, card] and -1; the reference hits a device assert in F.embedding,
 * lm_utils.py:103-121) embeds as the zero row and raises B200_FLAG_TOKEN_RANGE; the *_host entry points check the flags at
 * their own synchronisation and return B200_ERR_INVALID. */
#define B200_FLAG_TOKEN_RANGE 1
#define B200_FLAG_CODE_RANGE 2
#define B200_FLAG_KV_CAPACITY 4
/* A row of a paged handle (b200_lm_set_kv_pool) did not get a page because the pool was full: that row's output is garbage
 * until it is reset; no other row is affected.  b200_lm_step_host and b200_frame_step return B200_ERR_STATE on it. */
#define B200_FLAG_KV_POOL 8
int b200_lm_error_flags(b200_lm* h, int* flags_out);
/* Algorithmic HBM bytes of one step at the current batch and ring fill (DESIGN.md): weights once
 * + per-row KV read/append + embeddings + logits. */
int64_t b200_lm_algorithmic_bytes(b200_lm* h, int kv_fill);
/* Test/bench helper: declare that every row already holds `fill` steps of history (positions and
 * ring offsets are advanced; ring contents are whatever is in memory) so that the steady-state
 * full-ring step can be timed without running 3000 warm-up steps.  On a paged handle (b200_lm_set_kv_pool) every row then
 * holds the pages of that fill (B200_ERR_STATE, nothing changed, if they do not fit). */
int b200_lm_assume_fill(b200_lm* h, int fill);
/* 0 = one launch per kernel, 1 = replay the whole step as one CUDA graph (default 1): the reference graphs forward_text and
 * depformer_step separately (lm.py:628-634, utils/compile.py:190-280). */
int b200_lm_set_graph(b200_lm* h, int enable);
/* How the depformer runs, chosen before b200_lm_streaming_begin (B200_ERR_STATE while streaming).  B200_DEPFORMER_AUTO (default):
 * one persistent cooperative kernel per frame from three sessions on, a launch chain of GEMVs at one or two, and a launch chain
 * of tensor-core GEMMs under classifier-free guidance or int8 linears.  B200_DEPFORMER_CHAIN: always the launch chain.
 * B200_DEPFORMER_FUSED: the persistent kernel wherever it can run, at any batch.  Every mode computes what the reference does. */
#define B200_DEPFORMER_AUTO 0
#define B200_DEPFORMER_CHAIN 1
#define B200_DEPFORMER_FUSED 2
int b200_lm_set_depformer(b200_lm* h, int mode);
/* Storage type of the temporal KV rings, chosen before b200_lm_streaming_begin.  B200_KV_BF16 (default) is the
 * reference's ring (RingKVCache, transformer.py:196-288: 1.573 GB per session at context 3000).  B200_KV_FP8_E4M3 is
 * an opt-in extension outside the reference's numerics (SURVEY.md 8f item 3): e4m3 bytes plus one fp32 scale per
 * (session, head, slot), 0.811 GB per session; its logit error is reported by tests/test_gpu_zv_kv_q8.py. */
#define B200_KV_BF16 0
#define B200_KV_FP8_E4M3 1
#define B200_KV_INT8 2
int b200_lm_set_kv_dtype(b200_lm* h, int kv_dtype);
/* Slots per temporal KV ring, chosen before b200_lm_streaming_begin (0 or >= context: the reference's ring of `context` slots,
 * RingKVCache transformer.py:196-288).  A shorter ring holds the same keys as the reference's for a session's first `slots`
 * frames (nothing is evicted before position `context`), at slots/context of the 1.573 GB per session: a pool of young sessions
 * (SURVEY.md 8f item 3, "rings sized to live fill").  A row that steps past the capacity raises B200_FLAG_KV_CAPACITY; the
 * caller moves such a session to a full-size handle (b200_lm_session_export / _import) before that. */
int b200_lm_set_kv_capacity(b200_lm* h, int slots);
/* Paged temporal KV rings, chosen before b200_lm_streaming_begin (frames = 0: off, the default).  The rings of all model
 * rows share one pool of `frames` slots, rounded up to whole pages of `page_slots` slots (a power of two in [4, 256]) and
 * capped at what every row's full ring needs.  A row takes pages as its fill grows (inside the step) and returns them on
 * b200_lm_reset, so young and old sessions share one handle.  Keys are only stored elsewhere: the numerics are those of the
 * contiguous ring, bit for bit.  The streaming state keeps the contiguous layout (entries layers.<i>.k / .v [MB,H,context,128];
 * slots past a row's fill read as zeros), so snapshots move between paged and contiguous handles; writing model.offset (or a
 * whole snapshot) maps exactly the pages of the new fill, and returns B200_ERR_STATE, changing nothing, if they do not fit.
 * A row the step cannot serve raises B200_FLAG_KV_POOL.  Bf16 rings of the full context only: with b200_lm_set_kv_dtype
 * other than B200_KV_BF16 or with b200_lm_set_kv_capacity it returns B200_ERR_INVALID (here or at streaming_begin). */
int b200_lm_set_kv_pool(b200_lm* h, int64_t frames, int page_slots);
/* Pages held by rows and pages in the pool (0 / 0 without a pool).  Synchronises the handle's stream. */
int b200_lm_kv_pool_usage(b200_lm* h, int* pages_used, int* pages_total);
/* One session (one row) of an LM handle as a self-describing device record (layout in DESIGN.md §2): moves a session between
 * rows, handles and GPUs, e.g. from a short ring (B200_FLAG_KV_CAPACITY) or a paged pool close to dry into another handle.
 * The record holds the session's token ring, offsets, model positions (and under CFG its model exec flags and
 * cfg_is_masked_until, with condition_sum on its rows) and the temporal K/V of slots [0, min(pos, ring capacity)), so its size
 * follows the session's fill.  All three synchronise the handle's stream.
 *   session_bytes: the size b200_lm_session_export would write for `row` now.
 *   session_export: does not change the source.  It is ordered after every step already enqueued on the handle's stream; the
 *     row keeps running, and the caller resets or releases it when the move is complete.  B200_ERR_STATE for a short-ring row
 *     (b200_lm_set_kv_capacity) that has stepped past its capacity: its ring no longer holds the history.  B200_ERR_SHAPE if
 *     capacity is below the record's size.
 *   session_import: replaces model rows `row` (and row + B under CFG) with the record and changes no other row, page-table
 *     entry or output.  On a paged handle the row first gives back its pages, then holds exactly
 *     ceil(min(pos, context) / page_slots) pages.  Every check runs before the first write; on failure nothing changes:
 *     B200_ERR_INVALID: not a record of this version, a Mimi record, another model configuration, another KV storage type,
 *       CFG (or cfg_is_masked_until) or condition_sum on one side only, a row outside [0, B);
 *     B200_ERR_SHAPE: nbytes differs from the record's size;
 *     B200_ERR_STATE: the handle cannot hold the history: too few free pages in the pool, or a ring shorter than the
 *       session's position (this includes a wrapped session, pos > context, sent to a short ring).
 * Handle-wide values do not travel: the host step counter (offset_cpu) and the noise seed and counter; a moved session
 * continues with the destination's noise stream.  Its readiness (tokens -2 until offsets > max_delay) travels with offsets. */
int b200_lm_session_bytes(b200_lm* h, int row, int64_t* nbytes);
int b200_lm_session_export(b200_lm* h, int row, void* dst_dev, int64_t capacity);
int b200_lm_session_import(b200_lm* h, int row, const void* src_dev, int64_t nbytes);

/* ------------------------------------------------------------------------------------------ */
/* One dialogue frame for every session slot: host PCM in, host PCM + tokens out, one host wait  */
/* ------------------------------------------------------------------------------------------ */
/* Replaces the per-frame body of the reference's callers: moshi/moshi/server.py:120-147 (chunk -> mimi.encode ->
 * lm_gen.step -> mimi.decode -> main_pcm.cpu(), tokens[0,0,0].item(): two blocking reads per frame, :82-86) and
 * rust/moshi-server/batched_asr.py:138-215 (ASRService.step: slot updates -> reset / exec masks -> encode -> step ->
 * host copies), which the Rust server binds through py_basr_module.rs:243-256.  Slot updates use the values of
 * batched_asr.py:23-30 (UpdateFlags). */
typedef struct b200_frame b200_frame;
#define B200_SLOT_IDLE 0      /* UpdateFlags.NODATA: the slot does not execute from this frame on            */
#define B200_SLOT_ACTIVE (-1) /* UpdateFlags.ACTIVE: the slot executes from this frame on                     */
#define B200_SLOT_RESET (-2)  /* UpdateFlags.RESET: reset the slot's streaming state, then execute             */
                              /* > 0 (end-of-stream marker): the slot keeps its current activity               */
/* Both handles must be streaming with `batch` rows on `stream`; n_codebooks = the codec's codebooks = dep_q. */
int b200_frame_create(b200_mimi* mimi, b200_lm* lm, int batch, int n_codebooks, int dep_q, int frame_size, void* stream,
                      b200_frame** out);
int b200_frame_destroy(b200_frame* f);
/*   pcm_in_host     f32 [B, frame_size]   one 80 ms frame per slot (idle slots: ignored)
 *   updates_host    i32 [B] or NULL (= no change; every slot active after create)
 *   noise_host / noise_dev  f32 [B, b200_lm_noise_per_row] Exp(1) draws, host or device; both NULL = the LM step draws
 *                   its own (b200_lm_seed_noise) when sampling is on
 *   pcm_out_host    f32 [B, frame_size]   decoded frame; silence for rows with ready == 0
 *   tokens_out_host i64 [B, dep_q + 1]    LMGen.step output (row 0 text); -2 for rows that are not ready
 *   ready_out_host  u8  [B] or NULL       1 = the row executed and is past its max_delay warm-up (lm.py:774-782)
 * The decoder only advances for ready rows (server.py:139-142 skips mimi.decode while step() returns None). */
int b200_frame_step(b200_frame* f, const float* pcm_in_host, const int32_t* updates_host, const float* noise_host,
                    const float* noise_dev, float* pcm_out_host, int64_t* tokens_out_host, uint8_t* ready_out_host);

/* Hand-offs of the last frame, copied device-to-device into dst_dev (NULL = query size): "codes_in" i64 [B,K] (what
 * mimi.encode produced and lm_gen.step consumed, server.py:133-138), "tokens" i64 [B,dep_q+1], "codes_out" i64 [B,dep_q] (what
 * mimi.decode consumed), "exec" / "decoder_exec" u8 [B]. */
int b200_frame_read_buffer(b200_frame* f, const char* name, void* dst_dev, int64_t capacity_bytes, int64_t* nbytes);

/* ------------------------------------------------------------------------------------------ */
/* Batched speech-to-text: ASRService.step for every session slot, one host wait per frame        */
/* ------------------------------------------------------------------------------------------ */
/* rust/moshi-server/batched_asr.py:100-213 (ASRService, bound by py_basr_module.rs:224-256) for the STT models: dep_q = 0, every
 * codebook from the user, extra heads = voice-activity probabilities.  Per-slot client state (active, is_complete, offset,
 * real_end; ClientState, :85-98) and the end-of-stream countdown live on the device; one frame is slot updates -> resets ->
 * exec masks -> mimi.encode -> lm_gen.step_with_extra_heads -> flags, one stream-ordered chain with a single host wait.
 * Flags are MaskFlags (:14-20). */
typedef struct b200_asr b200_asr;
#define B200_ASR_ACTIVE 1            /* MaskFlags of batched_asr.py:14-20 */
#define B200_ASR_MARKER_RECEIVED 2
#define B200_ASR_IS_EOS 4
/* Both handles must be streaming with `batch` rows on `stream`.  B200_ERR_INVALID for an LM with dep_q != 0 or with delays (the
 * reference's warm-up asserts that step() returns a frame), a codec with fewer than n_q - dep_q codebooks, or a batch other than
 * both handles'.  Runs the reference's warm-up (:119-130: three frames of silence, every row executing) and returns with every
 * slot inactive, as after ClientState(); a slot used without a RESET continues from that state. */
int b200_asr_create(b200_mimi* mimi, b200_lm* lm, int batch, int asr_delay_in_tokens, void* stream, b200_asr** out);
int b200_asr_destroy(b200_asr* a);
/*   pcm_in_host          f32 [B, frame_size]  one 80 ms frame per slot (read only if some slot executes)
 *   updates_host         i32 [B]  B200_SLOT_IDLE / _ACTIVE / _RESET, or n > 0: an end-of-stream marker; the slot's activity
 *                        is unchanged and it ends (IS_EOS, inactive) on the frame its count of executed frames since its
 *                        reset reaches (the count when the marker arrived) + n + asr_delay_in_tokens + 2.  Other values are
 *                        ignored, as the reference does.
 *   flags_inout_host     u8  [B]  written where the reference writes flags_out (NODATA 0, ACTIVE / RESET 1, marker 2, end of
 *                        stream 4); every other entry keeps the caller's value
 *   tokens_out_host      i64 [B]  text token of each row (-2 for rows that do not execute)
 *   extra_heads_out_host f32 [B, extra_heads_num_heads]  element 0 of each softmaxed extra head (NULL without extra heads)
 *   *ran                 1 if the model ran; 0 if no slot was active (skip_exec, :179-180): tokens and extra heads untouched
 * B200_ERR_STATE if a row's KV ring did not get a page (B200_FLAG_KV_POOL), as b200_frame_step. */
int b200_asr_step(b200_asr* a, const float* pcm_in_host, const int32_t* updates_host, uint8_t* flags_inout_host,
                  int64_t* tokens_out_host, float* extra_heads_out_host, int* ran);
/* Buffers of the last frame, copied device-to-device (NULL = query size): "codes_in" i64 [B,K] (mimi.encode's output), "tokens"
 * i64 [B], "extra_heads" f32 [B,n_heads], "exec" / "reset" u8 [B], client state "offset" / "real_end" i64 [B]. */
int b200_asr_read_buffer(b200_asr* a, const char* name, void* dst_dev, int64_t capacity_bytes, int64_t* nbytes);

/* ------------------------------------------------------------------------------------------ */
/* Kernel-level entry points (used by the parity tests; same kernels the handles launch)        */
/* ------------------------------------------------------------------------------------------ */

/* y[M,N] = x[M,K] * w[N,K]^T, bf16 in, fp32 accumulate, bf16 out, on row-major weights: packs them into tiles and runs
 * the LM's linear for this shape (GEMV kernel up to 2 rows, wgmma stream-K / whole-tile / cluster split-K kernels above);
 * synchronises the stream (test helper).  Reference op: every nn.Linear of the LM (transformer.py:304-305,554-555,588-589). */
int b200_op_linear_bf16(const void* x_dev, const void* w_dev, void* y_dev, int M, int N, int K, void* stream);
/* Stream-K wgmma GEMM over pre-tiled weights (the LM's linear kernel; csrc/gemm_sk.cu).
 *   b200_op_packed_bytes / b200_op_pack_tiles: repack w bf16 [N,K] (epi 2: [2*gate_rows,K], rows gate|value,
 *   gating.py:18-20) into 16 KB SWIZZLE_128B tiles.
 *   b200_op_linear_sk: y = epi(x . W^T); epi 0 store [M,N], 1 residual add (y = res + .), 2 silu(gate)*value
 *   -> [M,gate_rows].  grid / smem_budget / stream_only are tuning & diagnostics knobs (0 = defaults). */
int64_t b200_op_packed_bytes(int N, int K, int epi, int gate_rows);
int b200_op_pack_tiles(const void* w_dev, void* out_dev, int N, int K, int epi, int gate_rows, void* stream);
int b200_op_linear_sk(const void* x_dev, const void* w_tiles_dev, void* y_dev, const void* res_dev, int M, int N,
                      int K, int epi, int gate_rows, int grid, int smem_budget, int stream_only, void* stream);
/* The LM's linear kernel for 33..256 sessions (csrc/gemm_ns.cu): activations as the wgmma A operand, two pre-tiled weight tiles
 * as B (N = 256 per wgmma), K cut over a cluster of `cluster` CTAs and reduced over distributed shared memory
 * (0 = the LM's own choice; 100 + n = single-tile units, N = 128 per instruction, n K-splits); same packed weights and
 * epilogues as b200_op_linear_sk, any M <= 256.
 * (b200_op_linear_sk with smem_budget = -1 keeps the swap-AB kernels at every M: the comparison row of tools/kbench.py.) */
int b200_op_linear_ns(const void* x_dev, const void* w_tiles_dev, void* y_dev, const void* res_dev, int M, int N, int K,
                      int epi, int gate_rows, int cluster, void* stream);
/* Up to how many activation rows the linears take the GEMV path (plain 16-byte loads on the CUDA cores instead of the
 * tensor-core GEMM; csrc/gemm_sk.cu): 0..4, default 2.  Returns the previous value. */
int b200_op_set_gemv_max_rows(int max_rows);
/* The launches the LM makes for one linear (b200_op_linear_sk / b200_op_linear_i8 with the LM's own choice, rows contiguous), for a
 * device of `sms` multiprocessors and GEMV path up to `gemv_max_rows` rows; needs no GPU.  norm: an RMSNorm in front, folded
 * where the plan takes the GEMV.  out[0] = launches, out[1] = 1 if the norm is folded, then 19 values per launch: kernel
 * (1 GEMV, 2 non-swapped, 3 cluster split-K, 4 swap-AB stream-K), first row, rows, grid, cluster size, dynamic shared memory,
 * stages, stage bytes, activation box rows, padded rows, k-blocks per split, GEMV splits, GEMV k-blocks per split,
 * weight tiles per unit, receive row floats, cluster columns per rank, whole rounds, first stream-K tile, stream-K items
 * (0 where a kernel has no such parameter).  `capacity` int64 slots at out; 2 + 4 * 19 always suffice.  Returns the errors
 * the linear would return for the shape. */
int b200_op_linear_plan(int M, int N, int K, int epi, int gate_rows, int int8, int norm, int sms, int gemv_max_rows, int64_t* out,
                        int capacity);
/* The depformer path the LM plans at streaming_begin (needs no GPU): `batch` sessions, cfg = classifier-free guidance on, int8 =
 * quantize=True, mode as b200_lm_set_depformer, for a device of `sms` multiprocessors and GEMV path up to `gemv_max_rows` rows.
 * out[0] = path (0 none: dep_q = 0, 1 launch chain, 2 persistent kernel); for the kernel out[1..5] = partial-buffer floats,
 * stages, stage bytes, dynamic shared memory, grid, then 6 values per GEMM phase (in_proj, out_proj, linear_in, linear_out,
 * head): weight tiles, k-blocks, k-blocks per split, splits, accumulators, output columns; 0 elsewhere.  `capacity` int64 slots
 * at out, at least 36.  B200_ERR_INVALID for out-of-range input and for a configuration the kernel refuses. */
int b200_op_depformer_plan(int dep_q, int depformer_dim, int depformer_num_heads, int depformer_ffn_hidden, int card, int batch,
                           int cfg, int int8, int mode, int sms, int gemv_max_rows, int64_t* out, int capacity);
/* What one Mimi frame launches at `batch` sessions (b200_mimi_streaming_begin's plan; needs no GPU), for a device of `sms`
 * multiprocessors and `num_codebooks` active codebooks.  out[0..5] = tensor-core layers of the encoder SEANet and of the
 * decoder SEANet, K slices of the down-sampling conv, split-K workspace bytes, kernels of one encode frame (RVQ included) and
 * of one decode frame (a split layer counts its reduction); then 21 values per tensor-core layer (encoder SEANet, decoder
 * SEANet, then the transformers' in_proj, out_proj, linear1, linear2, each serving every layer of both): SEANet layer index
 * (0..3 for the linears), kind (0 conv, 1 transposed conv, 2 linear), Cin, N, taps, dilation, stride, features per tile,
 * feature tiles, k-blocks, tile steps tt, tile sessions bb, steps per session T, sessions, row tiles, K splits, k-blocks per
 * split, stages, stage bytes, grid, dynamic shared memory.  `capacity` int64 slots at out (6 + 21 * layers; 1024 suffice for
 * the default configuration).  B200_ERR_INVALID for out-of-range input and for a configuration b200_mimi_create refuses. */
int b200_op_mimi_plan(const b200_mimi_config* cfg, int batch, int sms, int num_codebooks, int64_t* out, int capacity);
/* int8 x int8 linear (QLinear, utils/quantize.py:13-40: bitsandbytes row-wise absmax quantisation of weights and
 * activations, int32 accumulation, dequantisation by both row scales / 127^2), on wgmma s8 x s8 -> s32.
 *   b200_op_quant_pack_tiles: w bf16 [N,K] -> int8 SWIZZLE_128B tiles (b200_op_packed_bytes_i8 bytes) + scales f32 [N]
 *   b200_op_quantize_rows:    x bf16 [M,K] -> xq int8 [M,K] + scales f32 [M]
 *   b200_op_linear_i8:        y bf16 = epi(dequant(xq . Wq^T)), epilogues as b200_op_linear_sk */
int64_t b200_op_packed_bytes_i8(int N, int K, int epi, int gate_rows);
int b200_op_quant_pack_tiles(const void* w_dev, void* tiles_dev, float* scales_dev, int N, int K, int epi, int gate_rows,
                             void* stream);
int b200_op_quantize_rows(const void* x_dev, void* xq_dev, float* sa_dev, int M, int K, void* stream);
int b200_op_linear_i8(const void* xq_dev, const float* sa_dev, const void* w_tiles_dev, const float* sw_dev, void* y_dev,
                      const void* res_dev, int M, int N, int K, int epi, int gate_rows, void* stream);
/* StreamingConv1d.forward on one layer (conv.py:245-274): x [B,Cin,T], w [Cout,Cin,K], state
 * previous [B,Cin,Keff-S] (updated in place where exec_mask), y [B,Cout,T/S]. elu_in applies ELU to x.
 * Runs the kernels of the Mimi handle's down-sampling conv: split-K fp32 GEMM, in-order reduction, state commit. */
int b200_op_conv1d(const float* x_dev, const float* w_dev, const float* bias_dev, float* prev_dev,
                   const uint8_t* exec_mask_dev, float* y_dev, int B, int Cin, int Cout, int T,
                   int K, int stride, int dilation, int elu_in, void* stream);
/* mimi_tc_kernel (TMA + wgmma tf32, 3xTF32 split products: fp32-equivalent accuracy) on the reference's layouts;
 * test scaffolding around the kernel the Mimi handle launches for every conv / convtr / linear (the handle itself keeps all
 * activations token-major and never transposes).
 *   b200_op_tc_linear_f32: y[M,N] = x[M,K] . w[N,K]^T  (K % 32 == 0, N % 16 == 0)
 *   b200_op_tc_conv1d:     same contract as b200_op_conv1d (transposed = 0); transposed = 1: StreamingConvTranspose1d.forward
 *                          (conv.py:340-362), x [B,Cin,T], w [Cin,Cout,2*stride], y [B,Cout,T*stride], where the carried state is the
 *                          LAST INPUT STEP previous [B,Cin,1] instead of the overlap-add partial (the same information,
 *                          conv.py:349-361); Cin % 32 == 0. */
int b200_op_tc_linear_f32(const float* x_dev, const float* w_dev, float* y_dev, int M, int N, int K, void* stream);
int b200_op_tc_conv1d(const float* x_dev, const float* w_dev, const float* bias_dev, float* prev_dev, const uint8_t* exec_mask_dev,
                      float* y_dev, int B, int Cin, int Cout, int T, int K, int stride, int dilation, int elu_in, int transposed,
                      void* stream);
/* One temporal attention step, as the LM launches it (transformer.py:557-597): qkv bf16 [B,3*H*128] (rows q|k|v),
 * RoPE(q,k) at pos[b], K/V appended to the rings [B,H,cap,128] at pos % cap for rows with exec_mask, attention over
 * the min(pos + exec, cap) valid slots, out bf16 [B,H*128].  One kernel (rope + append + split-KV + merge). */
int b200_op_attn_step(const void* qkv_dev, void* k_dev, void* v_dev, void* out_dev, const int64_t* pos_dev,
                      const uint8_t* exec_mask_dev, int B, int H, int cap, int nsplit, float max_period, void* stream);
/* The same step over paged rings (b200_lm_set_kv_pool): k_pool / v_pool bf16 [n_pages,H,page_slots,128], page_table int32
 * [B,ceil(cap / page_slots)]; slot s of row b is page page_table[b][s / page_slots], offset s % page_slots.  Every slot the
 * step reads or writes (those below min(pos + exec, cap)) must be mapped.  Bit-identical to b200_op_attn_step on a ring
 * holding the same keys, for the same nsplit (<= 0: the LM's choice for (B, H, cap)). */
int b200_op_attn_step_paged(const void* qkv_dev, void* k_pool_dev, void* v_pool_dev, const int32_t* page_table_dev, void* out_dev,
                            const int64_t* pos_dev, const uint8_t* exec_mask_dev, int B, int H, int cap, int page_slots, int nsplit,
                            float max_period, void* stream);
/* The same step over an opt-in 8-bit ring (b200_lm_set_kv_dtype): k8 / v8 u8 [B,H,cap,128] (e4m3 bytes, or
 * round(x * 127 / absmax) + 128), ks / vs f32 [B,H,cap] = absmax / 448 (or / 127) of the row.  The q.k products are summed
 * in fp16 four at a time: queries are supported up to |q| = 256 per element (see lm_kernels.cuh). */
int b200_op_attn_step_q8(const void* qkv_dev, void* k8_dev, void* v8_dev, float* ks_dev, float* vs_dev, void* out_dev,
                         const int64_t* pos_dev, const uint8_t* exec_mask_dev, int B, int H, int cap, int nsplit, float max_period,
                         int kv_dtype, void* stream);
/* One depformer attention sub-step, as the LM launches it: qkv bf16 [B,3*H*64] (rows q|k|v), the new k / v written to slot
 * `step` of the per-frame caches [B,H,cap,64], attention over slots 0..step with scale 1/8 and no positional embedding,
 * out bf16 [B,H*64].  cap <= 16, step < cap. */
int b200_op_dep_attn_step(const void* qkv_dev, void* k_dev, void* v_dev, void* out_dev, int B, int H, int cap, int step, void* stream);
/* One attention step of a Mimi bottleneck transformer layer, as the Mimi handle launches it (ring_attn_step_kernel, D = 64):
 * qkv f32 [B,T,3*H*64] (rows q|k|v, each (h d)), RoPE at position offset[b] + t (fp32 angle), the T new keys / values
 * appended at slots (offset[b] + t) % cap of the rings k / v f32 [B,H,cap,64] for rows with exec_mask (paused rows write
 * nothing), attention of the T queries over the ring with the reference's mask (slot positions of RingKVCache.complete,
 * 0 <= q_pos - k_pos < context), out = out_hi + out_lo f32 [B,T,H*64] (a tf32 hi / lo pair).  offset is not advanced.
 * B200_ERR_SHAPE for T > 4 (one warp per query, 4 warps) or (T*64 + T*cap)*4 bytes of shared memory above 48 KB.  The qkv
 * layout is implied by H and T, not checked: the entry receives bare pointers, so a qkv row narrower than 3*H*64 floats cannot be
 * detected. */
int b200_op_mimi_ring_attn(const float* qkv_dev, float* k_dev, float* v_dev, float* out_hi_dev, float* out_lo_dev, const int64_t* offset_dev,
                           const uint8_t* exec_mask_dev, int B, int H, int T, int cap, int context, float max_period, void* stream);
/* RMSNorm of the LM (transformer.py:45-58, eps 1e-8): y = bf16(x * alpha * rsqrt(eps + mean(x^2))), x / y bf16 [M,dim],
 * alpha bf16 [dim], dim even. */
int b200_op_rmsnorm(const void* x_dev, const void* alpha_dev, void* y_dev, int M, int dim, void* stream);
/* LayerNorm of the cross-attention layers (norm_cross, nn.LayerNorm eps 1e-5): y = bf16((x - mean) * rstd * w + b) with fp32
 * statistics, x / y bf16 [M,dim], w / b bf16 [dim], dim even. */
int b200_op_layernorm(const void* x_dev, const void* w_dev, const void* b_dev, void* y_dev, int M, int dim, void* stream);
/* One cross-attention step, as the LM launches it: q bf16 [B,H*128], attention over all T keys of k / v bf16 [B,H,T,128]
 * (no RoPE, no mask), out bf16 [B,H*128].  nsplit <= 0: the LM's choice of splits. */
int b200_op_cross_attn_step(const void* q_dev, const void* k_dev, const void* v_dev, void* out_dev, int B, int H, int T, int nsplit,
                            void* stream);
/* b200_op_linear_sk on rmsnorm(x, alpha) with the norm folded into the GEMV kernel's activation staging (the LM's path for one
 * or two sessions).  Only the GEMV path takes a norm: where the plan takes another kernel (for M above
 * b200_op_set_gemv_max_rows) it returns B200_ERR_STATE. */
int b200_op_linear_sk_norm(const void* x_dev, const void* alpha_dev, const void* w_tiles_dev, void* y_dev, const void* res_dev, int M,
                           int N, int K, int epi, int gate_rows, void* stream);
/* sample_token (sampling.py:86-106): logits bf16 [B,card], noise f32 [B,min(k,card)] -> i64 [B]. */
int b200_op_sample(const void* logits_bf16_dev, const float* noise_dev, int64_t* out_dev, int B,
                   int card, int use_sampling, float temp, int top_k, void* stream);
/* The Exp(1) noise the LM step draws itself (b200_lm_seed_noise), as the step launches it: out f32 [n], element i from word
 * i % 4 of Philox4x32-10 block i / 4 with counter (i / 4 low, high, ctr low, high) and key (seed low, high).  Nothing past n is
 * written.  The counter is staged in a device word shared by all calls: calls must not overlap. */
int b200_op_lm_noise(float* out_dev, int64_t n, uint64_t seed, uint64_t ctr, void* stream);
/* The per-session text sampler of the LM step (b200_lm_set_session_sampling) on B rows: logits bf16 [B,card], noise f32 rows of
 * noise_ld floats, settings p[B] (host, every row with its own settings; NULL: every row follows use_sampling / temp / top_k),
 * history int32 [B,history] and counts int32 [B] on the device, updated in place as the step updates them (every row executes)
 * -> i64 [B]. */
int b200_op_sample_text_rows(const void* logits_bf16_dev, const float* noise_dev, int64_t noise_ld, int64_t* out_dev, int B, int card,
                             int use_sampling, float temp, int top_k, const b200_row_sampling* p, int32_t* history_dev,
                             int32_t* count_dev, int history, void* stream);
/* The step's bits -> Exp(1) transform on given 32-bit words: out[i] = -log(((words[i] >> 8) + 1) * 2^-24), and 2^-24 for the top
 * two 24-bit patterns (u >= 1 - 2^-24, as torch's exponential_ on CUDA); every output is finite and strictly positive. */
int b200_op_exp1(const uint32_t* words_dev, float* out_dev, int64_t n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MOSHI_B200_H */
