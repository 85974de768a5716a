// Mimi handle: weight ingestion (reference state-dict names), streaming state, encode / decode.
// Reference orchestration: moshi/moshi/models/compression.py:338-433.
//
// Everything between the PCM frame and the latent is TOKEN-MAJOR ([session][step][channel]): every SEANet conv / transposed
// conv and every transformer linear is one launch of mimi_tc_kernel (TMA + wgmma tf32 with 3xTF32 split products,
// mimi_tc.cuh); a layer's epilogue writes its consumer's activation (ELU applied, hi / lo pair) straight behind the
// consumer's carried left context, so that `cat(previous, x)` (conv.py:261) is an address, the streaming-state update
// (conv.py:263-267) is a P-row shift inside that buffer, and ProjectedTransformer.conv_layout (transformer.py:972-981)
// costs nothing.  The degenerate convs (Cin = 1, Cout = 1), the learnt 2x down-sampling conv (replicate padding), the
// depth-wise up-sampling, LayerNorm / RoPE / ring attention and the residual VQ are small SIMT kernels.
#include "mimi_kernels.cuh"
#include "mimi_tc.cuh"
#include "mimi_tm_kernels.cuh"
#include "tc_host.cuh"

using namespace b200;
using namespace b200::mimi;

namespace {

struct SeaLayer {
  int kind = 0;              // 0 = StreamingConv1d, 1 = StreamingConvTranspose1d
  std::string key;           // state-dict prefix of the nn.Conv1d / nn.ConvTranspose1d
  std::string tap;           // debug name of the raw output (empty: not stored)
  int cin = 0, cout = 0, k = 0, stride = 1, dil = 1;
  bool elu_in = false;
  int res_from = -1;         // index of the layer whose raw output is added in the epilogue (residual block second conv)
  bool simt_first = false, simt_last = false;   // Cin = 1 / Cout = 1: memory-bound SIMT kernels
  // per-frame geometry
  int t_in = 0, t_out = 0;   // steps per frame in / out
  int P = 0;                 // carried input rows: conv (k-1)*dil + 1 - stride; convtr 1 (the previous input step)
  int N = 0;                 // GEMM output features: conv Cout; convtr S * Cout, ordered (phase, channel)
  // weights
  float* w_simt = nullptr;   // first conv [Cout][K]; last conv [K][Cin]
  float* bias = nullptr;
  // streaming buffers
  float *ext_hi = nullptr, *ext_lo = nullptr;   // [B][P + t_in][cin] (SIMT layers: ext_hi is plain fp32, ext_lo null)
  float* y = nullptr;                           // raw output, token-major [B][t_out * (convtr: S)][cout]
  mtc::TcLayer tc;
};

struct TrLayer {
  const float *n1w, *n1b, *n2w, *n2b, *ls1, *ls2;
  mtc::TcLayer in_proj, out_proj, l1, l2;
  float *kc = nullptr, *vc = nullptr;
};

struct Transformer {
  std::vector<TrLayer> layers;
  long long* offset = nullptr;   // [B] tokens seen (== RingKVCache.end_offset == _MHAState.offset)
};

struct Tap { const float* p; int C, T; bool transpose; };   // transpose: stored [B][T][C], reported [B][C][T]

struct DownLayer {             // ConvDownsample1d (resample.py:14-65): k = 2 * stride, no bias, replicate padding
  std::string key;
  int cin = 0, cout = 0, k = 0, stride = 1;
  int t_in = 0, t_out = 0, P = 0;
  float* w = nullptr;          // [Cout][K * Cin]
  float* state = nullptr;      // previous [B][Cin][P]
  uint8_t* first = nullptr;    // replicate flags [B]
};

// what the configuration fixes (plan_seanet): frame geometry, layer lists, the tensor-core layers' shapes
struct MimiShape {
  b200_mimi_config cfg;
  int frame_size = 0, hop = 0, rs = 0;       // rs = resample stride (2)
  std::vector<SeaLayer> enc, dec;
  DownLayer down;                            // learnt down-sampling conv (replicate padding): split-K fp32 SIMT kernels
  mtc::TcShape in_proj, out_proj, linear1, linear2;   // every layer of both transformers
};

// what one frame of B sessions launches (plan_mimi)
struct MimiPlan {
  std::vector<mtc::TcSchedule> enc, dec;     // per SEANet layer (the SIMT layers' entries stay empty)
  mtc::TcSchedule in_proj, out_proj, linear1, linear2;   // both transformers run rs tokens per session
  int down_ksplit = 0;                       // K slices of the down-sampling conv
  size_t ws_bytes = 0;                       // split-K workspace
  int enc_launches = 0, dec_launches = 0;    // kernels of one encode frame (RVQ included) and of one decode frame
};

}  // namespace

struct b200_mimi : StreamCore, MimiShape {     // graphs[ENC_GRAPH] / graphs[DEC_GRAPH]: one frame's encode / decode
  TensorStore store;
  Arena weights;
  int num_codebooks = 8;

  // up-sampling (depth-wise convtr)
  float *up_w = nullptr, *up_partial = nullptr, *up_scratch = nullptr;
  Transformer enc_tr, dec_tr;
  // quantizer
  float *wT[2] = {nullptr, nullptr}, *woT[2] = {nullptr, nullptr};
  float *cb[2] = {nullptr, nullptr}, *cbT[2] = {nullptr, nullptr}, *cnorm[2] = {nullptr, nullptr};
  int stored_levels[2] = {0, 0};
  // per-batch buffers
  float *tok_in_enc = nullptr, *tok_enc = nullptr, *latent = nullptr;     // [B][T][C], [B][T][C], [B][C]
  float *latent_q = nullptr, *tok_in_dec = nullptr, *tok_dec = nullptr;
  float *tr_xn_hi = nullptr, *tr_xn_lo = nullptr, *tr_qkv = nullptr, *tr_ao_hi = nullptr,
        *tr_ao_lo = nullptr, *tr_h_hi = nullptr, *tr_h_lo = nullptr;
  uint8_t* exec_mask = nullptr;
  TmCommit *enc_tm = nullptr, *dec_tm = nullptr; int n_enc_tm = 0, n_dec_tm = 0; long long max_enc_tm = 0, max_dec_tm = 0;
  float* rvq_res[2] = {nullptr, nullptr};      // RVQ workspace for B queries: residuals, per-chunk partial argmin
  float* rvq_best[2] = {nullptr, nullptr};
  int* rvq_idx[2] = {nullptr, nullptr};
  float* splitk_ws = nullptr;                            // split-K partial sums of the deep / skinny layers
  // one-frame encode / decode as CUDA graphs over static buffers (frame in enc[0].ext -> enc_codes, dec_codes -> out_frame)
  int dec_graph_ncb = 0;
  long long *enc_codes = nullptr, *dec_codes = nullptr;   // [B][K], [B][q_n_q]
  float* out_frame = nullptr;                              // [B][frame_size]
  // staging of the host variants: pinned and device buffers of pin_pcm_n samples and pin_codes_n codes, grown on demand
  Arena staging;
  float *pin_pcm = nullptr; long long* pin_codes = nullptr; size_t pin_pcm_n = 0, pin_codes_n = 0;
  float* dev_pcm = nullptr; long long* dev_codes = nullptr;
  std::map<std::string, Tap> taps;
  int64_t weight_bytes = 0;
  // session records: the [B]-leading slice of every marked state entry, in marking order
  RowSlice* slices_dev = nullptr;
  int n_slices = 0;
  long long session_bytes = 0, slices_max = 0;
};

namespace {

enum { ENC_GRAPH, DEC_GRAPH };

// ---------------------------------------------------------------------------------------------
// structure (seanet.py:170-236, 323-388; resample.py; loaders.py:38-88)
// ---------------------------------------------------------------------------------------------
// Everything the configuration fixes, or why mimi_create refuses it: frame geometry, both SEANets' layers with their steps
// per frame in and out, carried rows P and GEMM widths N, the down-sampling conv and the tensor-core layers' shapes.
int plan_seanet(const b200_mimi_config& c, MimiShape* g) {
  if (c.n_ratios < 1 || c.n_ratios > 8) B200_FAIL(B200_ERR_INVALID, "mimi_create: n_ratios out of range");
  if (c.channels != 1) B200_FAIL(B200_ERR_INVALID, "mimi_create: only mono audio is on the hot path");
  if (c.q_dimension % 8) B200_FAIL(B200_ERR_INVALID, "mimi_create: codebook dimension must be a multiple of 8");
  if (c.tr_d_model / c.tr_num_heads != 64) B200_FAIL(B200_ERR_INVALID, "mimi_create: head dim must be 64");
  if (c.tr_d_model != c.dimension) B200_FAIL(B200_ERR_INVALID, "mimi_create: projected transformer unsupported");
  if (c.n_filters % 32 || c.compress != 2 || c.n_filters / c.compress % 32)
    B200_FAIL(B200_ERR_INVALID, "mimi_create: SEANet channel counts must be multiples of 32 (tensor-core k-blocks)");
  g->cfg = c;
  g->hop = 1;
  for (int i = 0; i < c.n_ratios; ++i) g->hop *= c.ratios[i];
  g->frame_size = (int)(c.sample_rate / c.frame_rate);
  const double enc_rate = (double)c.sample_rate / g->hop;
  g->rs = (int)(enc_rate / c.frame_rate);
  if (g->rs < 1 || g->frame_size != g->hop * g->rs) B200_FAIL(B200_ERR_INVALID, "mimi_create: frame size %d is not hop*stride", g->frame_size);
  g->enc.clear();
  g->dec.clear();
  auto conv = [](const std::string& key, int cin, int cout, int k, int stride, int dil, bool elu) {
    SeaLayer l;
    l.kind = 0; l.key = key; l.cin = cin; l.cout = cout; l.k = k; l.stride = stride; l.dil = dil; l.elu_in = elu;
    return l;
  };
  int idx = 0, mult = 1;
  {
    auto l = conv("encoder.model.0.conv.conv", c.channels, mult * c.n_filters, c.kernel_size, 1, 1, false);
    l.tap = "enc.0";
    g->enc.push_back(l);
  }
  idx = 1;
  for (int ri = c.n_ratios - 1; ri >= 0; --ri) {
    const int ratio = c.ratios[ri];
    const int ch = mult * c.n_filters;
    for (int j = 0; j < c.n_residual_layers; ++j) {
      int dil = 1;
      for (int q = 0; q < j; ++q) dil *= c.dilation_base;
      const std::string base = "encoder.model." + std::to_string(idx);
      auto a = conv(base + ".block.1.conv.conv", ch, ch / c.compress, c.residual_kernel_size, 1, dil, true);
      auto b = conv(base + ".block.3.conv.conv", ch / c.compress, ch, 1, 1, 1, true);
      b.res_from = (int)g->enc.size() - 1;      // skip connection: the input of the block = the previous module's raw output
      b.tap = "enc." + std::to_string(idx);
      g->enc.push_back(a);
      g->enc.push_back(b);
      ++idx;
    }
    ++idx;  // ELU
    auto l = conv("encoder.model." + std::to_string(idx) + ".conv.conv", ch, ch * 2, 2 * ratio, ratio, 1, true);
    l.tap = "enc." + std::to_string(idx);
    g->enc.push_back(l);
    ++idx;
    mult *= 2;
  }
  ++idx;  // ELU
  {
    auto l = conv("encoder.model." + std::to_string(idx) + ".conv.conv", mult * c.n_filters, c.dimension,
                  c.last_kernel_size, 1, 1, true);
    l.tap = "enc." + std::to_string(idx);
    g->enc.push_back(l);
  }

  idx = 0;
  mult = 1 << c.n_ratios;
  {
    auto l = conv("decoder.model.0.conv.conv", c.dimension, mult * c.n_filters, c.kernel_size, 1, 1, false);
    l.tap = "dec.0";
    g->dec.push_back(l);
  }
  idx = 1;
  for (int ri = 0; ri < c.n_ratios; ++ri) {
    const int ratio = c.ratios[ri];
    const int ch = mult * c.n_filters;
    ++idx;  // ELU
    SeaLayer t;
    t.kind = 1; t.key = "decoder.model." + std::to_string(idx) + ".convtr.convtr";
    t.cin = ch; t.cout = ch / 2; t.k = 2 * ratio; t.stride = ratio; t.elu_in = true;
    t.tap = "dec." + std::to_string(idx);
    g->dec.push_back(t);
    ++idx;
    for (int j = 0; j < c.n_residual_layers; ++j) {
      int dil = 1;
      for (int q = 0; q < j; ++q) dil *= c.dilation_base;
      const std::string base = "decoder.model." + std::to_string(idx);
      auto a = conv(base + ".block.1.conv.conv", ch / 2, ch / 2 / c.compress, c.residual_kernel_size, 1, dil, true);
      auto b = conv(base + ".block.3.conv.conv", ch / 2 / c.compress, ch / 2, 1, 1, 1, true);
      b.res_from = (int)g->dec.size() - 1;
      b.tap = "dec." + std::to_string(idx);
      g->dec.push_back(a);
      g->dec.push_back(b);
      ++idx;
    }
    mult /= 2;
  }
  ++idx;  // ELU
  {
    auto l = conv("decoder.model." + std::to_string(idx) + ".conv.conv", c.n_filters, c.channels,
                  c.last_kernel_size, 1, 1, true);
    l.tap = "dec." + std::to_string(idx);
    g->dec.push_back(l);
  }
  for (auto* layers : {&g->enc, &g->dec}) {
    int t = layers == &g->enc ? g->frame_size : g->rs;
    for (auto& l : *layers) {
      l.simt_first = l.kind == 0 && l.cin == 1;
      l.simt_last = l.kind == 0 && l.cout == 1;
      l.N = l.kind == 1 ? l.stride * l.cout : l.cout;
      l.P = l.kind == 1 ? 1 : (l.k - 1) * l.dil + 1 - l.stride;
      l.t_in = t;
      if (l.kind == 0) {
        if (t % l.stride) B200_FAIL(B200_ERR_INVALID, "%s: %d samples not divisible by stride %d", l.key.c_str(), t, l.stride);
        l.t_out = t / l.stride;
      } else {
        l.t_out = t;                            // GEMM rows per session; each row holds `stride` output steps
      }
      t = l.kind == 1 ? l.t_out * l.stride : l.t_out;
      if (!l.simt_first && !l.simt_last)
        l.tc.s = l.kind == 0 ? mtc::tc_shape(mtc::TC_CONV, l.N, l.cin, l.k, l.dil, l.stride, l.cout)
                             : mtc::tc_shape(mtc::TC_CONVTR, l.N, l.cin, 2, 1, 1, l.cout);
    }
    if (layers == &g->enc && t != g->rs) B200_FAIL(B200_ERR_INVALID, "encoder yields %d tokens/frame, expected %d", t, g->rs);
  }
  if (g->dec.back().t_out != g->frame_size) B200_FAIL(B200_ERR_INVALID, "decoder yields %d samples/frame", g->dec.back().t_out);
  g->down = DownLayer();
  g->down.key = "downsample.conv.conv.conv"; g->down.cin = c.dimension; g->down.cout = c.dimension;
  g->down.k = 2 * g->rs; g->down.stride = g->rs;
  g->down.t_in = g->rs; g->down.t_out = 1; g->down.P = g->down.k - g->down.stride;   // the encoder transformer's rs tokens -> one frame
  const int d = c.tr_d_model, ff = c.tr_dim_feedforward;
  g->in_proj = mtc::tc_shape(mtc::TC_LINEAR, 3 * d, d, 1);
  g->out_proj = mtc::tc_shape(mtc::TC_LINEAR, d, d, 1);
  g->linear1 = mtc::tc_shape(mtc::TC_LINEAR, ff, d, 1);
  g->linear2 = mtc::tc_shape(mtc::TC_LINEAR, d, ff, 1);
  return B200_OK;
}

// The schedule of every tensor-core layer at B sessions, the split-K workspace and the kernels one frame launches
// (encode_body + quantize_frame, dequantize_cols + decode_latent_body; a split layer adds its reduction); no CUDA call.
int plan_mimi(const MimiShape& g, int B, int sms, int num_codebooks, MimiPlan* out) {
  const auto& c = g.cfg;
  MimiPlan q;
  int sea[2] = {0, 0}, commit[2] = {0, 0};
  for (int w = 0; w < 2; ++w) {
    const std::vector<SeaLayer>& layers = w == 0 ? g.enc : g.dec;
    std::vector<mtc::TcSchedule>& s = w == 0 ? q.enc : q.dec;
    s.resize(layers.size());
    for (size_t i = 0; i < layers.size(); ++i) {
      const SeaLayer& l = layers[i];
      if (!l.simt_first && !l.simt_last) B200_TRY(mtc::plan_tc(l.tc.s, B, l.t_out, sms, mtc::TC_SPLIT_BYTES, &s[i]));
      sea[w] += 1 + (s[i].ksplit > 1);
      if (l.P > 0) commit[w] = 1;             // tm_commit_kernel
    }
  }
  B200_TRY(mtc::plan_tc(g.in_proj, B, g.rs, sms, mtc::TC_SPLIT_BYTES, &q.in_proj));
  B200_TRY(mtc::plan_tc(g.out_proj, B, g.rs, sms, mtc::TC_SPLIT_BYTES, &q.out_proj));
  B200_TRY(mtc::plan_tc(g.linear1, B, g.rs, sms, mtc::TC_SPLIT_BYTES, &q.linear1));
  B200_TRY(mtc::plan_tc(g.linear2, B, g.rs, sms, mtc::TC_SPLIT_BYTES, &q.linear2));
  // per layer: two LayerNorms, the attention step and four linears; then advance_offsets
  int tr = 7;
  for (const auto* s : {&q.in_proj, &q.out_proj, &q.linear1, &q.linear2}) tr += s->ksplit > 1;
  tr = c.tr_num_layers * tr + 1;
  // the down-sampling conv's partials outgrow the tensor-core layers' budget above 1024 sessions
  q.down_ksplit = ds_splits(g.down.cin * g.down.k);
  const size_t down_bytes = (size_t)q.down_ksplit * B * g.down.t_out * g.down.cout * 4;
  q.ws_bytes = down_bytes > mtc::TC_SPLIT_BYTES ? down_bytes : mtc::TC_SPLIT_BYTES;
  const int semantic = std::min(c.q_n_semantic, num_codebooks), levels = std::max(semantic, num_codebooks - semantic);
  // encode: SEANet, transformer, down conv + reduction, conv_commit (+ tm_commit), RVQ projection + search / pick per level
  q.enc_launches = sea[0] + tr + 2 + 1 + commit[0] + 1 + 2 * levels;
  // decode: RVQ decode, up-sampling, transformer, SEANet, (tm_commit +) convtr_commit
  q.dec_launches = 2 + tr + sea[1] + commit[1] + 1;
  *out = q;
  return B200_OK;
}

int get_f32(b200_mimi* h, const std::string& name, std::vector<int64_t> shape, const float** out) {
  const Tensor* t = h->store.find(name);
  if (!t) B200_FAIL(B200_ERR_MISSING, "mimi finalize: tensor '%s' was not loaded", name.c_str());
  if (t->dtype != B200_F32) B200_FAIL(B200_ERR_SHAPE, "mimi tensor '%s' must be float32", name.c_str());
  if (!shape.empty() && t->shape != shape) {
    std::string got;
    for (auto s : t->shape) got += std::to_string(s) + ",";
    B200_FAIL(B200_ERR_SHAPE, "mimi tensor '%s' has shape [%s]", name.c_str(), got.c_str());
  }
  *out = static_cast<const float*>(t->data);
  return B200_OK;
}

// nn.Linear-shaped weight [N][n_taps * Cin] (fp32, device) -> packed hi / lo tiles of L's shape owned by the handle
int pack_tc(b200_mimi* h, mtc::TcLayer& L, const float* w_ntc) {
  const mtc::TcShape& s = L.s;
  if (s.Cin % mtc::TC_KB || s.N % 16 || (s.N > mtc::TC_MAX_NT && s.N % mtc::TC_MAX_NT))
    B200_FAIL(B200_ERR_INVALID, "mimi: a %d x %d (x %d taps) contraction does not tile on the tensor-core kernel", s.N, s.Cin, s.n_taps);
  const size_t bytes = mtc::tc_packed_bytes(s);
  void* out = nullptr;
  B200_TRY(h->weights.alloc(&out, bytes, false));
  B200_TRY(mtc::tc_pack_weights(w_ntc, out, s, nullptr));
  L.wt = static_cast<uint8_t*>(out);
  h->weight_bytes += (int64_t)bytes;
  return B200_OK;
}

int pack_sea(b200_mimi* h, SeaLayer& l) {
  const float* w = nullptr;
  const long long n = (long long)l.cout * l.cin * l.k;
  if (l.kind == 0) B200_TRY(get_f32(h, l.key + ".weight", {l.cout, l.cin, l.k}, &w));
  else {
    if (l.k != 2 * l.stride) B200_FAIL(B200_ERR_INVALID, "convtr %s: kernel must be 2*stride", l.key.c_str());
    B200_TRY(get_f32(h, l.key + ".weight", {l.cin, l.cout, l.k}, &w));
  }
  if (l.simt_first) {                       // [Cout][1][K] is already [Cout][K]
    if (l.k > 8 || l.stride != 1 || l.cout % 4) B200_FAIL(B200_ERR_INVALID, "%s: unsupported first conv", l.key.c_str());
    B200_TRY(h->weights.alloc_t(&l.w_simt, (size_t)n, false));
    B200_CUDA(cudaMemcpy(l.w_simt, w, (size_t)n * 4, cudaMemcpyDeviceToDevice));
    h->weight_bytes += n * 4;
  } else if (l.simt_last) {                 // [1][Cin][K] -> [K][Cin]
    if (l.stride != 1 || l.cin % 4) B200_FAIL(B200_ERR_INVALID, "%s: unsupported last conv", l.key.c_str());
    B200_TRY(h->weights.alloc_t(&l.w_simt, (size_t)n, false));
    B200_LAUNCH(tm_weight_conv_kernel, (unsigned)ceil_div64(n, 256), 256, 0, 0, w, l.w_simt, 1, l.cin, l.k);
    h->weight_bytes += n * 4;
  } else {
    Arena tmp;
    float* wk = nullptr;
    B200_TRY(tmp.alloc_t(&wk, (size_t)n, false));
    if (l.kind == 0) B200_LAUNCH(tm_weight_conv_kernel, (unsigned)ceil_div64(n, 256), 256, 0, 0, w, wk, l.cout, l.cin, l.k);
    else B200_LAUNCH(tm_weight_convtr_kernel, (unsigned)ceil_div64(n, 256), 256, 0, 0, w, wk, l.cin, l.cout, l.stride);
    B200_TRY(pack_tc(h, l.tc, wk));
    B200_CUDA(cudaDeviceSynchronize());
  }
  const float* b = nullptr;
  B200_TRY(get_f32(h, l.key + ".bias", {l.cout}, &b));
  B200_TRY(h->weights.alloc_t(&l.bias, l.cout, false));
  B200_CUDA(cudaMemcpy(l.bias, b, l.cout * 4, cudaMemcpyDeviceToDevice));
  h->weight_bytes += l.cout * 4;
  l.tc.bias = l.bias;
  B200_CUDA(cudaDeviceSynchronize());
  h->store.release(l.key + ".weight");
  h->store.release(l.key + ".bias");
  return check_launch("pack_sea");
}

// the down-sampling conv's weights for conv_splitk_kernel: [Cout][K * Cin]
int pack_down(b200_mimi* h, DownLayer& l) {
  const float* w = nullptr;
  B200_TRY(get_f32(h, l.key + ".weight", {l.cout, l.cin, l.k}, &w));
  const long long n = (long long)l.cout * l.cin * l.k;
  B200_TRY(h->weights.alloc_t(&l.w, n, false));
  B200_LAUNCH(tm_weight_conv_kernel, (unsigned)ceil_div64(n, 256), 256, 0, 0, w, l.w, l.cout, l.cin, l.k);
  h->weight_bytes += n * 4;
  B200_CUDA(cudaDeviceSynchronize());
  h->store.release(l.key + ".weight");
  return check_launch("pack_down");
}

int keep(b200_mimi* h, const std::string& name, std::vector<int64_t> shape, const float** out) {
  const float* src = nullptr;
  B200_TRY(get_f32(h, name, shape, &src));
  long long n = 1;
  for (auto s : shape) n *= s;
  float* dst = nullptr;
  B200_TRY(h->weights.alloc_t(&dst, n, false));
  B200_CUDA(cudaMemcpy(dst, src, n * 4, cudaMemcpyDeviceToDevice));
  h->store.release(name);
  h->weight_bytes += n * 4;
  *out = dst;
  return B200_OK;
}

int keep_linear(b200_mimi* h, const std::string& name, const mtc::TcShape& s, mtc::TcLayer& L) {
  const float* src = nullptr;
  B200_TRY(get_f32(h, name, {s.N, s.Cin}, &src));
  L.s = s;
  B200_TRY(pack_tc(h, L, src));                // nn.Linear weight [out][in] is already [N][K]
  B200_CUDA(cudaDeviceSynchronize());
  h->store.release(name);
  return B200_OK;
}

int pack_transformer(b200_mimi* h, const std::string& prefix, Transformer& tr) {
  const auto& c = h->cfg;
  const int d = c.tr_d_model;
  tr.layers.resize(c.tr_num_layers);
  for (int li = 0; li < c.tr_num_layers; ++li) {
    const std::string p = prefix + ".transformer.layers." + std::to_string(li);
    TrLayer& L = tr.layers[li];
    B200_TRY(keep_linear(h, p + ".self_attn.in_projs.0.weight", h->in_proj, L.in_proj));
    B200_TRY(keep_linear(h, p + ".self_attn.out_projs.0.weight", h->out_proj, L.out_proj));
    B200_TRY(keep(h, p + ".norm1.weight", {d}, &L.n1w));
    B200_TRY(keep(h, p + ".norm1.bias", {d}, &L.n1b));
    B200_TRY(keep(h, p + ".norm2.weight", {d}, &L.n2w));
    B200_TRY(keep(h, p + ".norm2.bias", {d}, &L.n2b));
    B200_TRY(keep_linear(h, p + ".linear1.weight", h->linear1, L.l1));
    B200_TRY(keep_linear(h, p + ".linear2.weight", h->linear2, L.l2));
    B200_TRY(keep(h, p + ".layer_scale_1.scale", {d}, &L.ls1));
    B200_TRY(keep(h, p + ".layer_scale_2.scale", {d}, &L.ls2));
  }
  return B200_OK;
}

int pack_quantizer(b200_mimi* h) {
  const auto& c = h->cfg;
  const char* names[2] = {"rvq_first", "rvq_rest"};
  h->stored_levels[0] = c.q_n_semantic;
  h->stored_levels[1] = c.q_n_q - c.q_n_semantic;
  for (int w = 0; w < 2; ++w) {
    const std::string p = std::string("quantizer.") + names[w];
    const float* src = nullptr;
    B200_TRY(get_f32(h, p + ".input_proj.weight", {c.q_dimension, c.dimension, 1}, &src));
    B200_TRY(h->weights.alloc_t(&h->wT[w], (size_t)c.q_dimension * c.dimension, false));
    B200_LAUNCH(transpose_kernel, (unsigned)ceil_div64((long long)c.q_dimension * c.dimension, 256), 256, 0, 0, src,
                h->wT[w], c.q_dimension, c.dimension);
    B200_TRY(get_f32(h, p + ".output_proj.weight", {c.dimension, c.q_dimension, 1}, &src));
    B200_TRY(h->weights.alloc_t(&h->woT[w], (size_t)c.q_dimension * c.dimension, false));
    B200_LAUNCH(transpose_kernel, (unsigned)ceil_div64((long long)c.q_dimension * c.dimension, 256), 256, 0, 0, src,
                h->woT[w], c.dimension, c.q_dimension);
    const int L = h->stored_levels[w];
    const size_t per = (size_t)c.q_bins * c.q_dimension;
    B200_TRY(h->weights.alloc_t(&h->cb[w], per * L, false));
    B200_TRY(h->weights.alloc_t(&h->cbT[w], per * L, false));
    B200_TRY(h->weights.alloc_t(&h->cnorm[w], (size_t)c.q_bins * L, false));
    for (int l = 0; l < L; ++l) {
      const std::string cbp = p + ".vq.layers." + std::to_string(l) + "._codebook";
      const float *es = nullptr, *us = nullptr;
      B200_TRY(get_f32(h, cbp + ".embedding_sum", {c.q_bins, c.q_dimension}, &es));
      B200_TRY(get_f32(h, cbp + ".cluster_usage", {c.q_bins}, &us));
      B200_LAUNCH(build_codebook_kernel, c.q_bins, 128, 0, 0, es, us, h->cb[w] + per * l, h->cbT[w] + per * l,
                  h->cnorm[w] + (size_t)c.q_bins * l, c.q_bins, c.q_dimension);
    }
    B200_CUDA(cudaDeviceSynchronize());
    for (int l = 0; l < L; ++l) {
      const std::string cbp = p + ".vq.layers." + std::to_string(l) + "._codebook";
      h->store.release(cbp + ".embedding_sum");
      h->store.release(cbp + ".cluster_usage");
      h->store.release(cbp + "._initialized");
    }
    h->store.release(p + ".input_proj.weight");
    h->store.release(p + ".output_proj.weight");
  }
  return check_launch("pack_quantizer");
}

// ---------------------------------------------------------------------------------------------
// launches
// ---------------------------------------------------------------------------------------------
int launch_tc(b200_mimi* h, const mtc::TcLayer& L) { return mtc::tc_launch(L, h->body); }

// StreamingTransformer.forward for T tokens per row (transformer.py:894-929, layer :752-802)
int run_transformer(b200_mimi* h, Transformer& tr, const float* x_in, float* x, int T) {
  const auto& c = h->cfg;
  const int B = h->batch, ntok = B * T, d = c.tr_d_model, H = c.tr_num_heads, D = d / H;
  const float nl = -logf(c.tr_max_period) * 2.f / (float)D;
  const size_t attn_smem = (size_t)(T * D + T * c.tr_context) * sizeof(float);
  for (size_t li = 0; li < tr.layers.size(); ++li) {
    TrLayer& L = tr.layers[li];
    const float* cur = li == 0 ? x_in : x;
    B200_LAUNCH(layernorm_split_kernel, ceil_div(ntok * 32, 256), 256, 0, h->body, cur, L.n1w, L.n1b, h->tr_xn_hi, h->tr_xn_lo, ntok, d, 1e-5f);
    B200_TRY(launch_tc(h, L.in_proj));
    B200_LAUNCH((ring_attn_step_kernel<64>), B * H, 128, attn_smem, h->body, h->tr_qkv, L.kc, L.vc, h->tr_ao_hi, h->tr_ao_lo, tr.offset,
                h->exec_mask, T, H, c.tr_context, c.tr_context, nl);
    B200_TRY(launch_tc(h, L.out_proj));       // x = cur + layer_scale_1 * out_proj(attention)
    B200_LAUNCH(layernorm_split_kernel, ceil_div(ntok * 32, 256), 256, 0, h->body, x, L.n2w, L.n2b, h->tr_xn_hi, h->tr_xn_lo, ntok, d, 1e-5f);
    B200_TRY(launch_tc(h, L.l1));             // h = gelu(linear1(xn)) as a hi / lo pair
    B200_TRY(launch_tc(h, L.l2));             // x = x + layer_scale_2 * linear2(h)
  }
  B200_LAUNCH(advance_offsets_kernel, ceil_div(B, 128), 128, 0, h->body, tr.offset, h->exec_mask, B, T);
  return check_launch("mimi transformer");
}

int run_seanet(b200_mimi* h, std::vector<SeaLayer>& layers) {
  const int B = h->batch;
  for (size_t i = 0; i < layers.size(); ++i) {
    SeaLayer& l = layers[i];
    if (l.simt_first) {
      const SeaLayer& nx = layers[i + 1];
      ConvFirst q;
      q.ext = l.ext_hi; q.E = l.P + l.t_in; q.P = l.P; q.w = l.w_simt; q.bias = l.bias;
      q.y = l.y; q.y_sb = (long long)l.t_out * l.cout;
      q.a_hi = nx.ext_hi + (long long)nx.P * nx.cin; q.a_lo = nx.ext_lo + (long long)nx.P * nx.cin;
      q.a_sb = (long long)(nx.P + nx.t_in) * nx.cin; q.a_elu = nx.elu_in;
      q.B = B; q.Cout = l.cout; q.K = l.k; q.T = l.t_out;
      const long long n = (long long)B * l.t_out;
      if (l.cout % 4 || 128 % (l.cout / 4) || l.k > 8) B200_FAIL(B200_ERR_INVALID, "mimi: first conv with %d channels / %d taps", l.cout, l.k);
      const int per_pass = 128 / (l.cout / 4);
      q.tok_per_block = per_pass * 16;           // 16 passes per CTA: the 4 x K weights of a thread are loaded once
      B200_LAUNCH(conv_first_tm_kernel, (unsigned)ceil_div64(n, q.tok_per_block), 128, 0, h->body, q);
    } else if (l.simt_last) {
      ConvLast q;
      q.ext = l.ext_hi; q.e_sb = (long long)(l.P + l.t_in) * l.cin; q.Cin = l.cin; q.w = l.w_simt; q.bias = l.bias;
      q.y = l.y; q.y_sb = l.t_out; q.B = B; q.K = l.k; q.dil = l.dil; q.T = l.t_out;
      const long long n = (long long)B * l.t_out;
      B200_LAUNCH(conv_last_tm_kernel, (unsigned)ceil_div64(n, 128), 128, (size_t)l.k * l.cin * 4, h->body, q);
    } else {
      B200_TRY(launch_tc(h, l.tc));
    }
  }
  return check_launch("mimi seanet");
}

// the down-sampling conv reads tok_enc token-major and writes latent [B][C] (replicate padding on a session's first frame)
ConvSplitK down_conv(b200_mimi* h) {
  const DownLayer& l = h->down;
  const int d = h->cfg.dimension;
  ConvSplitK p;
  p.x = h->tok_enc; p.xb = (long long)l.t_in * d; p.xc = 1; p.xt = d; p.Tin = l.t_in;
  p.st = l.state; p.P = l.P; p.first = l.first;
  p.w = l.w; p.bias = nullptr;
  p.y = h->latent; p.yb = d; p.yc = 1; p.yt = 1;
  p.Cin = l.cin; p.stride = l.stride; p.dil = 1; p.Tout = l.t_out; p.elu_in = 0;
  p.M = l.cout; p.N = h->batch * l.t_out; p.Kd = l.cin * l.k;
  return p;
}

int commit_states(b200_mimi* h, bool encoder) {
  const int B = h->batch;
  if (encoder) {
    B200_LAUNCH(conv_commit_kernel, B, 128, 0, h->body, down_conv(h), h->exec_mask);   // the down-sampling conv
    if (h->n_enc_tm) {
      dim3 grid((unsigned)ceil_div64(h->max_enc_tm, 128), h->n_enc_tm);
      B200_LAUNCH(tm_commit_kernel, grid, 128, 0, h->body, h->enc_tm, h->exec_mask, B);
    }
  } else {
    if (h->n_dec_tm) {
      dim3 grid((unsigned)ceil_div64(h->max_dec_tm, 128), h->n_dec_tm);
      B200_LAUNCH(tm_commit_kernel, grid, 128, 0, h->body, h->dec_tm, h->exec_mask, B);
    }
    const int per_row = h->cfg.dimension * h->rs;                                 // the depth-wise up-sampling's overlap-add carry
    B200_LAUNCH(convtr_commit_kernel, (unsigned)ceil_div64((long long)B * per_row, 256), 256, 0, h->body, h->up_partial, h->up_scratch,
                per_row, h->exec_mask, B);
  }
  return check_launch("commit_states");
}

// frame in enc[0].ext -> latent [B][C]   (static buffers only: this is what gets captured into a graph)
int encode_body(b200_mimi* h) {
  const int T = h->frame_size / h->hop;   // encoder tokens per frame (2)
  B200_TRY(run_seanet(h, h->enc));        // the last conv's raw output is tok_in_enc, token-major [B][T][C]
  B200_TRY(run_transformer(h, h->enc_tr, h->tok_in_enc, h->tok_enc, T));
  {
    // deep and skinny (2048 reduction steps, N = sessions): the reduction cut over KS CTAs per 64 outputs, slices added in order
    const ConvSplitK p = down_conv(h);
    const int KS = ds_splits(p.Kd);
    dim3 g1(ceil_div(p.M, DS_CO), KS);
    B200_LAUNCH(conv_splitk_kernel, g1, 256, 0, h->body, p, h->splitk_ws, KS);
    B200_LAUNCH(conv_splitk_reduce_kernel, (unsigned)ceil_div64((long long)p.N * p.M, 256), 256, 0, h->body, p, h->splitk_ws, KS);
  }
  B200_TRY(commit_states(h, true));
  return B200_OK;
}

// the PCM frame lands right behind the first conv's carried samples
int load_frame(b200_mimi* h, const float* pcm, int n_frames, int f) {
  const int fs = h->frame_size;
  const SeaLayer& l = h->enc[0];
  B200_CUDA(cudaMemcpy2DAsync(l.ext_hi + l.P, (size_t)(l.P + fs) * 4, pcm + (size_t)f * fs, (size_t)fs * n_frames * 4,
                              (size_t)fs * 4, h->batch, cudaMemcpyDeviceToDevice, h->stream));
  return B200_OK;
}

// One frame's latent [B][C] (row b at lat + b * lb, channel c at + c * lc) -> codes[b * cs_b + k * cs_k], B queries.
int quantize_frame(b200_mimi* h, const float* lat, long long lb, long long lc, long long* codes, long long cs_b, long long cs_k) {
  const auto& c = h->cfg;
  const int Q = h->batch, Dq = c.q_dimension, bins = c.q_bins;
  const int n_chunks = ceil_div(bins, RVQ_CHUNK);
  int levels[2];
  levels[0] = c.q_n_semantic < h->num_codebooks ? c.q_n_semantic : h->num_codebooks;
  levels[1] = h->num_codebooks - levels[0];
  {
    dim3 grid(ceil_div(Q, RVQ_PQ), 2, ceil_div(Dq, 64));
    B200_LAUNCH(rvq_project_kernel, grid, 256, (size_t)(RVQ_PQ * c.dimension + 4 * RVQ_PQ * 64) * 4, h->body, lat, lb, lc, 1LL, 1, Q,
                h->wT[0], h->wT[1], h->rvq_res[0], h->rvq_res[1], c.dimension, Dq);
  }
  const int max_levels = levels[0] > levels[1] ? levels[0] : levels[1];
  const size_t per = (size_t)bins * Dq;
  for (int level = 0; level < max_levels; ++level) {
    RvqLevelArgs a;
    for (int w = 0; w < 2; ++w) {
      a.res[w] = h->rvq_res[w];
      a.cbT[w] = h->cbT[w] + per * level; a.cb[w] = h->cb[w] + per * level; a.cnorm[w] = h->cnorm[w] + (size_t)bins * level;
      a.part_best[w] = h->rvq_best[w]; a.part_idx[w] = h->rvq_idx[w];
      a.active[w] = level < levels[w];
      a.code_index[w] = (w == 0 ? 0 : levels[0]) + level;
    }
    a.codes = codes; a.cs_b = cs_b; a.cs_k = cs_k; a.cs_f = 1;
    a.n_query = Q; a.n_frames = 1; a.Dq = Dq; a.bins = bins; a.n_chunks = n_chunks;
    dim3 g1(n_chunks, ceil_div(Q, RVQ_QT), 2);
    B200_LAUNCH(rvq_search_kernel, g1, RVQ_CHUNK, (size_t)RVQ_QT * Dq * 4, h->body, a);
    dim3 g2(Q, 2);
    B200_LAUNCH(rvq_pick_kernel, g2, 128, 0, h->body, a);
  }
  return check_launch("rvq_encode");
}

int dequantize_cols(b200_mimi* h, const long long* codes, long long cs_b, long long cs_k, long long cs_f, int n_codebooks,
                    int n_cols, float* out, long long ob, long long oc, long long ot) {
  const auto& c = h->cfg;
  if (n_codebooks < 1 || n_codebooks > c.q_n_q) B200_FAIL(B200_ERR_SHAPE, "decode: %d codebooks", n_codebooks);
  RvqDecArgs a;
  a.codes = codes; a.cs_b = cs_b; a.cs_k = cs_k; a.cs_f = cs_f; a.n_frames = n_cols;
  for (int w = 0; w < 2; ++w) { a.cb[w] = h->cb[w]; a.woT[w] = h->woT[w]; }
  a.levels[0] = c.q_n_semantic < n_codebooks ? c.q_n_semantic : n_codebooks;
  a.levels[1] = n_codebooks - a.levels[0];
  a.level_offset[0] = 0; a.level_offset[1] = a.levels[0];
  a.out = out; a.ob = ob; a.oc = oc; a.ot = ot;
  a.Dq = c.q_dimension; a.Cout = c.dimension; a.bins = c.q_bins; a.err = h->err;
  dim3 grid(h->batch * n_cols, (c.dimension + 63) / 64);
  B200_LAUNCH(rvq_decode_kernel, grid, 256, (2 * c.q_dimension + 256) * sizeof(float), h->body, a);
  return check_launch("rvq_decode");
}

// latent_q [B][C] -> out_frame [B][frame]   (static buffers only)
int decode_latent_body(b200_mimi* h) {
  const int B = h->batch, d = h->cfg.dimension, S = h->rs;
  const int T = S;   // tokens per frame after up-sampling
  {
    const long long total = (long long)B * 2 * S * d;   // (T_in + 1) * S * C with T_in = 1
    B200_LAUNCH(upsample_dw_kernel, (unsigned)ceil_div64(total, 256), 256, 0, h->body, h->latent_q, (long long)d, 1LL, 1LL, 1,
                h->up_w, h->up_partial, h->up_scratch, h->tok_in_dec, B, d, S);
  }
  B200_TRY(run_transformer(h, h->dec_tr, h->tok_in_dec, h->tok_dec, T));   // its last linear also fills dec[0]'s ext
  B200_TRY(run_seanet(h, h->dec));
  B200_TRY(commit_states(h, false));
  return B200_OK;
}

void register_tap(b200_mimi* h, const std::string& name, const float* p, int C, int T, bool transpose) { h->taps[name] = Tap{p, C, T, transpose}; }

// A SEANet's buffers for B sessions: every layer owns its extended input; raw outputs where something reads them
int alloc_seanet(b200_mimi* h, std::vector<SeaLayer>& layers, int B, bool is_dec, std::vector<TmCommit>& commits, long long& max_rows) {
  Arena& A = h->state;
  for (size_t i = 0; i < layers.size(); ++i) {
    SeaLayer& l = layers[i];
    const size_t ext_n = (size_t)B * (l.P + l.t_in) * l.cin;
    B200_TRY(A.alloc_t(&l.ext_hi, ext_n));
    if (!l.simt_first && !l.simt_last) B200_TRY(A.alloc_t(&l.ext_lo, ext_n));
    else l.ext_lo = nullptr;
    if (l.P > 0) {
      TmCommit cm;
      cm.hi = l.ext_hi; cm.lo = l.ext_lo; cm.P = l.P; cm.T = l.t_in; cm.rowlen = l.cin; cm.sb = (long long)(l.P + l.t_in) * l.cin;
      commits.push_back(cm);
      if ((long long)B * l.cin > max_rows) max_rows = (long long)B * l.cin;
    }
    const int steps_out = l.kind == 1 ? l.t_out * l.stride : l.t_out;
    const bool is_last = i + 1 == layers.size();
    l.y = nullptr;
    if (is_last && !is_dec) l.y = h->tok_in_enc;                       // transformer input
    else if (is_last && is_dec) l.y = h->out_frame;
    else if (!l.tap.empty()) B200_TRY(A.alloc_t(&l.y, (size_t)B * steps_out * l.cout));
    if (!l.tap.empty() && l.y) register_tap(h, l.tap, l.y, l.cout, steps_out, !(is_last && !is_dec));
  }
  return B200_OK;
}

// the activation a tensor-core layer writes for its consumer nx (ELU applied where nx wants it) behind nx's carried rows;
// a_row = the producer's N (= stride * nx.cin for a convtr: `stride` consumer rows per GEMM row)
void feed(mtc::TcParams& e, const SeaLayer& nx, int a_row) {
  e.act_mode = nx.simt_last ? mtc::TC_ACT_FULL : mtc::TC_ACT_SPLIT;
  e.act_elu = nx.elu_in ? 1 : 0;
  e.a_hi = nx.ext_hi + (long long)nx.P * nx.cin;
  e.a_lo = nx.ext_lo ? nx.ext_lo + (long long)nx.P * nx.cin : nullptr;
  e.a_sb = (long long)(nx.P + nx.t_in) * nx.cin;
  e.a_row = a_row;
}

// Binds a SEANet's tensor-core layers to their schedules: layer i writes its raw output and the activation layer i + 1 reads.
// conv: GEMM row t reads ext rows t * stride + tap * dil (ext row 0 = oldest carried sample)
// convtr: GEMM row t reads ext rows t + slot, slot 0 = x[t-1] (ext row 0 = the carried previous step)
int bind_seanet(b200_mimi* h, std::vector<SeaLayer>& layers, const std::vector<mtc::TcSchedule>& sched) {
  for (size_t i = 0; i < layers.size(); ++i) {
    SeaLayer& l = layers[i];
    if (l.simt_first || l.simt_last) continue;
    mtc::TcParams e{};
    e.epi = mtc::TC_EPI_CONV;
    e.y = l.y; e.y_sb = (long long)l.t_out * l.N; e.y_row = l.N;      // convtr: a GEMM row is `stride` consecutive output steps
    if (l.res_from >= 0) {
      const SeaLayer& r = layers[l.res_from];
      if (!r.y) B200_FAIL(B200_ERR_INVALID, "bad residual plan");
      e.res = r.y; e.r_sb = (long long)l.t_out * l.N; e.r_row = l.N;
    }
    if (i + 1 < layers.size()) feed(e, layers[i + 1], l.N);
    B200_TRY(mtc::tc_bind(l.tc, sched[i], e, l.ext_hi, l.ext_lo, l.P + l.t_in, h->splitk_ws));
  }
  return B200_OK;
}

}  // namespace

int b200::mimi_frame_view(b200_mimi* h, MimiFrameView* v) {
  B200_TRY(check_streaming(h, "mimi_frame_view"));
  *v = MimiFrameView{h->batch, h->num_codebooks, h->frame_size};
  return B200_OK;
}

// =============================================================================================
// C ABI
// =============================================================================================
extern "C" {

int b200_mimi_create(const b200_mimi_config* cfg, b200_mimi** out) {
  if (!cfg || !out) B200_FAIL(B200_ERR_INVALID, "mimi_create: null argument");
  MimiShape g;
  B200_TRY(plan_seanet(*cfg, &g));
  b200_mimi* h = new b200_mimi();
  static_cast<MimiShape&>(*h) = std::move(g);
  cudaGetDevice(&h->device);
  h->session_kind = SESSION_MIMI;
  h->fingerprint = config_fingerprint(&h->cfg, sizeof(h->cfg));
  h->num_codebooks = cfg->num_codebooks;
  *out = h;
  return B200_OK;
}

int b200_mimi_load_tensor(b200_mimi* h, const char* name, const void* data_dev, int dtype, int ndim,
                          const int64_t* shape) {
  if (!h) B200_FAIL(B200_ERR_INVALID, "mimi_load_tensor: null handle");
  if (h->finalized) B200_FAIL(B200_ERR_STATE, "mimi_load_tensor: already finalized");
  DeviceGuard g(h->device);
  return h->store.put(name, data_dev, dtype, ndim, shape);
}

int b200_mimi_finalize(b200_mimi* h) {
  if (!h) B200_FAIL(B200_ERR_INVALID, "mimi_finalize: null handle");
  if (h->finalized) return B200_OK;
  DeviceGuard g(h->device);
  B200_TRY(mtc::tc_init());
  for (auto& l : h->enc) B200_TRY(pack_sea(h, l));
  for (auto& l : h->dec) B200_TRY(pack_sea(h, l));
  B200_TRY(pack_down(h, h->down));
  {
    const float* w = nullptr;
    B200_TRY(keep(h, "upsample.convtr.convtr.convtr.weight", {h->cfg.dimension, 1, 2 * h->rs}, &w));
    h->up_w = const_cast<float*>(w);
  }
  B200_TRY(pack_transformer(h, "encoder_transformer", h->enc_tr));
  B200_TRY(pack_transformer(h, "decoder_transformer", h->dec_tr));
  B200_TRY(pack_quantizer(h));
  B200_CUDA(cudaDeviceSynchronize());
  h->store.release_all();   // anything left is not used on the hot path
  h->finalized = true;
  return B200_OK;
}

int b200_mimi_destroy(b200_mimi* h) {
  if (!h) return B200_OK;
  DeviceGuard g(h->device);
  b200_mimi_streaming_end(h);
  h->store.release_all();
  h->weights.free_all();
  delete h;
  return B200_OK;
}

int b200_mimi_set_num_codebooks(b200_mimi* h, int n) {
  if (!h) B200_FAIL(B200_ERR_INVALID, "set_num_codebooks: null handle");
  if (n < h->cfg.q_n_semantic || n > h->cfg.q_n_q)   // vq.py:315-317 assertion
    B200_FAIL(B200_ERR_SHAPE, "set_num_codebooks(%d): must be in [%d, %d]", n, h->cfg.q_n_semantic, h->cfg.q_n_q);
  h->num_codebooks = n;
  h->graphs[ENC_GRAPH].drop();
  return B200_OK;
}

int b200_mimi_streaming_begin(b200_mimi* h, int batch, void* stream) {
  B200_TRY(check_begin(h, batch, "streaming_begin"));
  DeviceGuard guard_dev(h->device);
  const auto& c = h->cfg;
  const int B = batch, d = c.dimension;
  h->stream = static_cast<cudaStream_t>(stream);
  h->taps.clear();
  Arena& A = h->state;
  struct Cleanup { b200_mimi* h; bool armed = true; ~Cleanup() { if (armed) b200_mimi_streaming_end(h); } } cleanup{h};
  MimiPlan plan;
  B200_TRY(plan_mimi(*h, B, num_sms(), h->num_codebooks, &plan));
  B200_TRY(A.alloc_t(&h->exec_mask, B, false));
  B200_CUDA(cudaMemset(h->exec_mask, 1, B));
  B200_TRY(A.alloc_t(&h->err, 1));
  B200_TRY(A.alloc(reinterpret_cast<void**>(&h->splitk_ws), plan.ws_bytes, false));

  const int T = h->rs;   // transformer tokens per frame on both sides
  B200_TRY(A.alloc_t(&h->tok_in_enc, (size_t)B * T * d));   // written by the last encoder conv
  B200_TRY(A.alloc_t(&h->tok_enc, (size_t)B * T * d));
  B200_TRY(A.alloc_t(&h->latent, (size_t)B * d));
  B200_TRY(A.alloc_t(&h->latent_q, (size_t)B * d));
  B200_TRY(A.alloc_t(&h->tok_in_dec, (size_t)B * T * d));
  B200_TRY(A.alloc_t(&h->tok_dec, (size_t)B * T * d));
  B200_TRY(A.alloc_t(&h->out_frame, (size_t)B * h->frame_size));

  std::vector<TmCommit> enc_tm, dec_tm;
  h->max_enc_tm = h->max_dec_tm = 0;
  B200_TRY(alloc_seanet(h, h->enc, B, false, enc_tm, h->max_enc_tm));
  B200_TRY(alloc_seanet(h, h->dec, B, true, dec_tm, h->max_dec_tm));
  B200_TRY(bind_seanet(h, h->enc, plan.enc));
  B200_TRY(bind_seanet(h, h->dec, plan.dec));
  register_tap(h, "enc.tr", h->tok_enc, d, T, false);
  register_tap(h, "enc.latent", h->latent, d, 1, false);
  register_tap(h, "dec.latent", h->latent_q, d, 1, false);
  register_tap(h, "dec.up", h->tok_in_dec, d, T, false);
  register_tap(h, "dec.tr", h->tok_dec, d, T, false);

  // down-sampling conv (replicate pad): carried input and first-frame flags
  B200_TRY(A.alloc_t(&h->down.state, (size_t)B * h->down.cin * h->down.P));
  B200_TRY(A.alloc_t(&h->down.first, B, false));
  B200_CUDA(cudaMemset(h->down.first, 1, B));
  // up-sampling depth-wise convtr
  B200_TRY(A.alloc_t(&h->up_partial, (size_t)B * d * h->rs));
  B200_TRY(A.alloc_t(&h->up_scratch, (size_t)B * d * h->rs));
  h->n_enc_tm = (int)enc_tm.size();
  h->n_dec_tm = (int)dec_tm.size();
  B200_TRY(A.alloc_t(&h->enc_tm, enc_tm.size() ? enc_tm.size() : 1, false));
  B200_TRY(A.alloc_t(&h->dec_tm, dec_tm.size() ? dec_tm.size() : 1, false));
  if (!enc_tm.empty()) B200_CUDA(cudaMemcpy(h->enc_tm, enc_tm.data(), enc_tm.size() * sizeof(TmCommit), cudaMemcpyHostToDevice));
  if (!dec_tm.empty()) B200_CUDA(cudaMemcpy(h->dec_tm, dec_tm.data(), dec_tm.size() * sizeof(TmCommit), cudaMemcpyHostToDevice));

  // transformers
  const int H = c.tr_num_heads, D = d / H, ff = c.tr_dim_feedforward;
  const size_t ntok = (size_t)B * T;
  B200_TRY(A.alloc_t(&h->tr_xn_hi, ntok * d));
  B200_TRY(A.alloc_t(&h->tr_xn_lo, ntok * d));
  B200_TRY(A.alloc_t(&h->tr_qkv, ntok * 3 * d));
  B200_TRY(A.alloc_t(&h->tr_ao_hi, ntok * d));
  B200_TRY(A.alloc_t(&h->tr_ao_lo, ntok * d));
  B200_TRY(A.alloc_t(&h->tr_h_hi, ntok * ff));
  B200_TRY(A.alloc_t(&h->tr_h_lo, ntok * ff));
  for (int which = 0; which < 2; ++which) {
    Transformer* tr = which == 0 ? &h->enc_tr : &h->dec_tr;
    const float* x_in = which == 0 ? h->tok_in_enc : h->tok_in_dec;
    float* x = which == 0 ? h->tok_enc : h->tok_dec;
    B200_TRY(A.alloc_t(&tr->offset, B));
    for (size_t li = 0; li < tr->layers.size(); ++li) {
      TrLayer& L = tr->layers[li];
      B200_TRY(A.alloc_t(&L.kc, (size_t)B * H * c.tr_context * D));
      B200_TRY(A.alloc_t(&L.vc, (size_t)B * H * c.tr_context * D));
      const float* cur = li == 0 ? x_in : x;
      const long long sb = (long long)T * d;
      float* ws = h->splitk_ws;
      mtc::TcParams e{};                      // in_proj: qkv = W_in xn
      e.epi = mtc::TC_EPI_CONV; e.y = h->tr_qkv; e.y_sb = 3 * sb; e.y_row = 3 * d;
      B200_TRY(mtc::tc_bind(L.in_proj, plan.in_proj, e, h->tr_xn_hi, h->tr_xn_lo, T, ws));
      e = mtc::TcParams{};                    // out_proj: x = cur + layer_scale_1 * (W_out ao)   (transformer.py:769)
      e.epi = mtc::TC_EPI_RES_SCALE; e.y = x; e.y_sb = sb; e.y_row = d; e.res = cur; e.r_sb = sb; e.r_row = d; e.scale = L.ls1;
      B200_TRY(mtc::tc_bind(L.out_proj, plan.out_proj, e, h->tr_ao_hi, h->tr_ao_lo, T, ws));
      e = mtc::TcParams{};                    // linear1 + GELU -> h as a hi / lo pair (never stored raw)
      e.epi = mtc::TC_EPI_GELU; e.y_sb = (long long)T * ff; e.y_row = ff;
      e.act_mode = mtc::TC_ACT_SPLIT; e.a_hi = h->tr_h_hi; e.a_lo = h->tr_h_lo; e.a_sb = (long long)T * ff; e.a_row = ff;
      B200_TRY(mtc::tc_bind(L.l1, plan.linear1, e, h->tr_xn_hi, h->tr_xn_lo, T, ws));
      // linear2: x = x + layer_scale_2 * (W_2 h)   (transformer.py:777); the decoder's last layer also feeds dec[0]
      e = mtc::TcParams{};
      e.epi = mtc::TC_EPI_RES_SCALE; e.y = x; e.y_sb = sb; e.y_row = d; e.res = x; e.r_sb = sb; e.r_row = d; e.scale = L.ls2;
      if (which == 1 && li + 1 == tr->layers.size()) feed(e, h->dec[0], d);
      B200_TRY(mtc::tc_bind(L.l2, plan.linear2, e, h->tr_h_hi, h->tr_h_lo, T, ws));
    }
  }
  B200_TRY(A.alloc_t(&h->enc_codes, (size_t)B * c.q_n_q));
  B200_TRY(A.alloc_t(&h->dec_codes, (size_t)B * c.q_n_q));
  B200_TRY(h->open_streams());
  h->body = h->stream;
  // what a streaming-state snapshot holds (streaming.py:158-181): masks, carried conv rows (the transposed convs' carry is
  // their previous input step), both transformers' KV rings and offsets
  A.mark_state(h->exec_mask, B, "exec_mask", B200_U8, {B});
  A.mark_state(h->down.first, B, "downsample.first", B200_U8, {B});
  for (int which = 0; which < 2; ++which)
    for (auto& l : which == 0 ? h->enc : h->dec) {
      const std::string nm = (which == 0 ? "encoder." : "decoder.") + l.key.substr(l.key.find("model."));
      const int64_t E = l.P + l.t_in;
      // the whole extended buffer is registered (the frame part is scratch); the shim slices the first P rows out
      A.mark_state(l.ext_hi, (size_t)B * E * l.cin * 4, nm + ".ext_hi", B200_F32, {B, E, l.cin});
      if (l.ext_lo) A.mark_state(l.ext_lo, (size_t)B * E * l.cin * 4, nm + ".ext_lo", B200_F32, {B, E, l.cin});
    }
  A.mark_state(h->down.state, (size_t)B * h->down.cin * h->down.P * 4, "downsample.previous", B200_F32, {B, h->down.cin, h->down.P});
  A.mark_state(h->up_partial, (size_t)B * d * h->rs * 4, "upsample.partial", B200_F32, {B, d, h->rs});
  for (int which = 0; which < 2; ++which) {
    Transformer* tr = which == 0 ? &h->enc_tr : &h->dec_tr;
    const std::string tp = which == 0 ? "encoder_transformer" : "decoder_transformer";
    A.mark_state(tr->offset, (size_t)B * 8, tp + ".offset", B200_I64, {B});
    for (size_t li = 0; li < tr->layers.size(); ++li) {
      auto& L = tr->layers[li];
      const std::string p = tp + ".layers." + std::to_string(li);
      A.mark_state(L.kc, (size_t)B * H * c.tr_context * D * 4, p + ".k", B200_F32, {B, H, c.tr_context, D});
      A.mark_state(L.vc, (size_t)B * H * c.tr_context * D * 4, p + ".v", B200_F32, {B, H, c.tr_context, D});
    }
  }
  {
    std::vector<RowSlice> s;
    for (auto& e : A.snap) s.push_back({static_cast<char*>(e.ptr), (long long)(e.bytes / B), 0, 0});
    h->session_bytes = layout_row_slices(s, sizeof(SessionHeader));
    h->slices_max = 0;
    for (auto& e : s) h->slices_max = std::max(h->slices_max, e.row_bytes);
    h->n_slices = (int)s.size();
    B200_TRY(A.alloc_t(&h->slices_dev, s.size(), false));
    B200_CUDA(cudaMemcpy(h->slices_dev, s.data(), s.size() * sizeof(RowSlice), cudaMemcpyHostToDevice));
  }
  {
    const int n_chunks = ceil_div(c.q_bins, RVQ_CHUNK);
    for (int w = 0; w < 2; ++w) {
      B200_TRY(A.alloc_t(&h->rvq_res[w], (size_t)B * c.q_dimension, false));
      B200_TRY(A.alloc_t(&h->rvq_best[w], (size_t)B * n_chunks, false));
      B200_TRY(A.alloc_t(&h->rvq_idx[w], (size_t)B * n_chunks, false));
    }
  }
  B200_CUDA(cudaDeviceSynchronize());
  h->batch = B;
  cleanup.armed = false;
  return B200_OK;
}

int b200_mimi_streaming_end(b200_mimi* h) {
  if (!h) return B200_OK;
  DeviceGuard g(h->device);
  h->end_streaming();
  h->taps.clear();
  return B200_OK;
}

int b200_mimi_reset(b200_mimi* h, const uint8_t* reset_mask_dev) {
  B200_STREAMING_ENTRY(h, "mimi_reset");
  const int B = h->batch;
  auto zero = [&](float* buf, long long per_row) {
    if (!buf || per_row <= 0) return;
    B200_LAUNCH(zero_rows_kernel, (unsigned)ceil_div64((long long)B * per_row, 256), 256, 0, h->stream, buf, per_row,
                reset_mask_dev, B);
  };
  for (auto* layers : {&h->enc, &h->dec})
    for (auto& l : *layers)
      if (l.P > 0)
        B200_LAUNCH(tm_zero_kernel, (unsigned)ceil_div64((long long)B * l.P * l.cin, 256), 256, 0, h->stream, l.ext_hi, l.ext_lo, l.P,
                    l.cin, (long long)(l.P + l.t_in) * l.cin, reset_mask_dev, B);
  zero(h->down.state, (long long)h->down.cin * h->down.P);
  zero(h->up_partial, (long long)h->cfg.dimension * h->rs);
  B200_LAUNCH(reset_flags_kernel, ceil_div(B, 128), 128, 0, h->stream, h->down.first, h->enc_tr.offset, h->dec_tr.offset,
              h->exec_mask, reset_mask_dev, B);
  return check_launch("mimi_reset");
}

int b200_mimi_set_exec_mask(b200_mimi* h, const uint8_t* exec_mask_dev) {
  B200_STREAMING_ENTRY(h, "mimi_set_exec_mask");
  if (!exec_mask_dev) B200_FAIL(B200_ERR_INVALID, "mimi_set_exec_mask: null mask");
  B200_CUDA(cudaMemcpyAsync(h->exec_mask, exec_mask_dev, h->batch, cudaMemcpyDeviceToDevice, h->stream));
  return B200_OK;
}

int b200_mimi_encode_to_latent(b200_mimi* h, const float* pcm_dev, int n_frames, float* latent_dev) {
  B200_STREAMING_ENTRY(h, "mimi_encode_to_latent");
  if (!pcm_dev || !latent_dev || n_frames < 1) B200_FAIL(B200_ERR_SHAPE, "mimi_encode_to_latent: bad arguments");
  const int d = h->cfg.dimension;
  for (int f = 0; f < n_frames; ++f) {
    B200_TRY(load_frame(h, pcm_dev, n_frames, f));
    h->body = h->stream;
    B200_TRY(encode_body(h));
    B200_CUDA(cudaMemcpy2DAsync(latent_dev + f, (size_t)n_frames * 4, h->latent, 4, 4, (size_t)h->batch * d,
                                cudaMemcpyDeviceToDevice, h->stream));
  }
  return B200_OK;
}

int b200_mimi_quantize(b200_mimi* h, const float* latent_dev, int n_frames, int64_t* codes_dev) {
  B200_STREAMING_ENTRY(h, "mimi_quantize");
  if (!latent_dev || !codes_dev || n_frames < 1) B200_FAIL(B200_ERR_SHAPE, "mimi_quantize: bad arguments");
  const int d = h->cfg.dimension, K = h->num_codebooks;
  h->body = h->stream;
  for (int f = 0; f < n_frames; ++f)       // latent [B][C][n_frames] -> codes [B][K][n_frames], the pass encode runs per frame
    B200_TRY(quantize_frame(h, latent_dev + f, (long long)d * n_frames, n_frames, reinterpret_cast<long long*>(codes_dev) + f,
                            (long long)K * n_frames, n_frames));
  return B200_OK;
}

int b200_mimi_encode(b200_mimi* h, const float* pcm_dev, int n_frames, int64_t* codes_dev) {
  B200_STREAMING_ENTRY(h, "mimi_encode");
  if (!pcm_dev || !codes_dev || n_frames < 1) B200_FAIL(B200_ERR_SHAPE, "mimi_encode: bad arguments");
  const int d = h->cfg.dimension, K = h->num_codebooks;
  for (int f = 0; f < n_frames; ++f) {
    B200_TRY(load_frame(h, pcm_dev, n_frames, f));
    B200_TRY(h->run(h->graphs[ENC_GRAPH], "a Mimi frame", [&]() -> int {
      B200_TRY(encode_body(h));
      return quantize_frame(h, h->latent, d, 1, h->enc_codes, K, 1);
    }));
    // enc_codes [B][K] -> codes[b][k][f]
    B200_CUDA(cudaMemcpy2DAsync(reinterpret_cast<long long*>(codes_dev) + f, (size_t)n_frames * 8, h->enc_codes, 8, 8,
                                (size_t)h->batch * K, cudaMemcpyDeviceToDevice, h->stream));
  }
  return B200_OK;
}

int b200_mimi_decode_latent(b200_mimi* h, const int64_t* codes_dev, int n_codebooks, int n_frames, float* latent_dev) {
  B200_STREAMING_ENTRY(h, "mimi_decode_latent");
  if (!codes_dev || !latent_dev || n_frames < 1) B200_FAIL(B200_ERR_SHAPE, "mimi_decode_latent: bad arguments");
  const int d = h->cfg.dimension;
  h->body = h->stream;
  return dequantize_cols(h, reinterpret_cast<const long long*>(codes_dev), (long long)n_codebooks * n_frames, n_frames, 1,
                         n_codebooks, n_frames, latent_dev, (long long)d * n_frames, n_frames, 1);
}

int b200_mimi_decode(b200_mimi* h, const int64_t* codes_dev, int n_codebooks, int n_frames, float* pcm_dev) {
  B200_STREAMING_ENTRY(h, "mimi_decode");
  if (!codes_dev || !pcm_dev || n_frames < 1) B200_FAIL(B200_ERR_SHAPE, "mimi_decode: bad arguments");
  if (n_codebooks < 1 || n_codebooks > h->cfg.q_n_q) B200_FAIL(B200_ERR_SHAPE, "decode: %d codebooks", n_codebooks);
  const int d = h->cfg.dimension, fs = h->frame_size;
  if (h->dec_graph_ncb != n_codebooks) h->graphs[DEC_GRAPH].drop();
  h->dec_graph_ncb = n_codebooks;
  for (int f = 0; f < n_frames; ++f) {
    // codes[b][k][f] -> dec_codes [B][n_codebooks]
    B200_CUDA(cudaMemcpy2DAsync(h->dec_codes, 8, reinterpret_cast<const long long*>(codes_dev) + f, (size_t)n_frames * 8, 8,
                                (size_t)h->batch * n_codebooks, cudaMemcpyDeviceToDevice, h->stream));
    B200_TRY(h->run(h->graphs[DEC_GRAPH], "a Mimi frame", [&]() -> int {
      B200_TRY(dequantize_cols(h, h->dec_codes, n_codebooks, 1, 1, n_codebooks, 1, h->latent_q, d, 1, 1));
      return decode_latent_body(h);
    }));
    B200_CUDA(cudaMemcpy2DAsync(pcm_dev + (size_t)f * fs, (size_t)fs * n_frames * 4, h->out_frame, (size_t)fs * 4,
                                (size_t)fs * 4, h->batch, cudaMemcpyDeviceToDevice, h->stream));
  }
  return B200_OK;
}

/* get_streaming_state / set_streaming_state (streaming.py:158-181) as one opaque device blob */
int64_t b200_mimi_state_bytes(b200_mimi* h) { return (h && h->batch > 0) ? (int64_t)h->state.state_bytes() : 0; }

int b200_mimi_get_state(b200_mimi* h, void* dst_dev, int64_t capacity) {
  B200_STREAMING_ENTRY(h, "mimi_get_state");
  return h->save_state(dst_dev, capacity, 0, "mimi_get_state");
}

int b200_mimi_set_state(b200_mimi* h, const void* src_dev, int64_t nbytes) {
  B200_STREAMING_ENTRY(h, "mimi_set_state");
  B200_TRY(h->check_blob(src_dev, nbytes, 0, "mimi_set_state"));
  return h->load_state(src_dev);
}

/* One session as a record: the 256-byte SessionHeader, then row `row` of every marked state entry in marking order, each
 * 16-byte aligned.  The size depends on the configuration only. */
int b200_mimi_session_bytes(b200_mimi* h, int64_t* nbytes) {
  B200_TRY(check_streaming(h, "mimi_session_bytes"));
  if (nbytes) *nbytes = h->session_bytes;
  return B200_OK;
}

int b200_mimi_session_export(b200_mimi* h, int row, void* dst_dev, int64_t capacity) {
  B200_STREAMING_ENTRY(h, "mimi_session_export");
  B200_TRY(h->check_row(row, "mimi_session_export"));
  if (!dst_dev) B200_FAIL(B200_ERR_INVALID, "mimi_session_export: null destination");
  if (capacity < h->session_bytes)
    B200_FAIL(B200_ERR_SHAPE, "mimi_session_export: the record takes %lld bytes, capacity %lld", h->session_bytes, (long long)capacity);
  const SessionHeader s = h->session_header(h->session_bytes);
  char* rec = static_cast<char*>(dst_dev);
  B200_CUDA(cudaMemcpyAsync(rec, &s, sizeof(s), cudaMemcpyHostToDevice, h->stream));
  B200_TRY(row_slice_copy(h->slices_dev, h->n_slices, h->slices_max, rec, row, true, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200_OK;
}

int b200_mimi_session_import(b200_mimi* h, int row, const void* src_dev, int64_t nbytes) {
  B200_STREAMING_ENTRY(h, "mimi_session_import");
  B200_TRY(h->check_row(row, "mimi_session_import"));
  SessionHeader s;
  B200_TRY(h->read_session_header(src_dev, nbytes, "mimi_session_import", &s));
  if (s.bytes != h->session_bytes || nbytes != h->session_bytes)
    B200_FAIL(B200_ERR_SHAPE, "mimi_session_import: the record takes %lld bytes, header says %lld, caller passed %lld", h->session_bytes,
              (long long)s.bytes, (long long)nbytes);
  B200_TRY(row_slice_copy(h->slices_dev, h->n_slices, h->slices_max, const_cast<char*>(static_cast<const char*>(src_dev)), row, false,
                          h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200_OK;
}

int b200_mimi_set_graph(b200_mimi* h, int enable) {
  if (!h) B200_FAIL(B200_ERR_INVALID, "mimi_set_graph: null handle");
  h->set_graph(enable);
  return B200_OK;
}

static int ensure_host_staging(b200_mimi* h, size_t pcm_n, size_t codes_n) {
  if (pcm_n <= h->pin_pcm_n && codes_n <= h->pin_codes_n) return B200_OK;
  const size_t pn = std::max(pcm_n, h->pin_pcm_n), cn = std::max(codes_n, h->pin_codes_n);
  h->staging.free_all();
  h->pin_pcm_n = h->pin_codes_n = 0;
  B200_TRY(h->staging.alloc_host(&h->pin_pcm, pn));
  B200_TRY(h->staging.alloc_t(&h->dev_pcm, pn, false));
  B200_TRY(h->staging.alloc_host(&h->pin_codes, cn));
  B200_TRY(h->staging.alloc_t(&h->dev_codes, cn, false));
  h->pin_pcm_n = pn;
  h->pin_codes_n = cn;
  return B200_OK;
}

int b200_mimi_encode_host(b200_mimi* h, const float* pcm_host, int n_frames, int64_t* codes_host) {
  B200_STREAMING_ENTRY(h, "mimi_encode_host");
  if (!pcm_host || !codes_host || n_frames < 1) B200_FAIL(B200_ERR_SHAPE, "mimi_encode_host: bad arguments");
  const size_t pn = (size_t)h->batch * h->frame_size * n_frames, cn = (size_t)h->batch * h->num_codebooks * n_frames;
  B200_TRY(ensure_host_staging(h, pn, cn));
  memcpy(h->pin_pcm, pcm_host, pn * 4);
  B200_CUDA(cudaMemcpyAsync(h->dev_pcm, h->pin_pcm, pn * 4, cudaMemcpyHostToDevice, h->stream));
  B200_TRY(b200_mimi_encode(h, h->dev_pcm, n_frames, reinterpret_cast<int64_t*>(h->dev_codes)));
  B200_CUDA(cudaMemcpyAsync(h->pin_codes, h->dev_codes, cn * 8, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  memcpy(codes_host, h->pin_codes, cn * 8);
  return B200_OK;
}

int b200_mimi_decode_host(b200_mimi* h, const int64_t* codes_host, int n_codebooks, int n_frames, float* pcm_host) {
  B200_STREAMING_ENTRY(h, "mimi_decode_host");
  if (!pcm_host || !codes_host || n_frames < 1) B200_FAIL(B200_ERR_SHAPE, "mimi_decode_host: bad arguments");
  const size_t pn = (size_t)h->batch * h->frame_size * n_frames, cn = (size_t)h->batch * n_codebooks * n_frames;
  B200_TRY(ensure_host_staging(h, pn, cn));
  memcpy(h->pin_codes, codes_host, cn * 8);
  B200_CUDA(cudaMemcpyAsync(h->dev_codes, h->pin_codes, cn * 8, cudaMemcpyHostToDevice, h->stream));
  B200_TRY(b200_mimi_decode(h, reinterpret_cast<const int64_t*>(h->dev_codes), n_codebooks, n_frames, h->dev_pcm));
  B200_CUDA(cudaMemcpyAsync(h->pin_pcm, h->dev_pcm, pn * 4, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  memcpy(pcm_host, h->pin_pcm, pn * 4);
  return B200_OK;
}

/* the same state entry by entry (names in include/moshi_b200.h) */
int b200_mimi_state_count(b200_mimi* h) { return (h && h->batch > 0) ? (int)h->state.snap.size() : 0; }
int b200_mimi_state_entry(b200_mimi* h, int index, const char** name, int* dtype, int* ndim, int64_t* shape8, int64_t* nbytes) {
  B200_TRY(check_streaming(h, "mimi_state_entry"));
  return h->state_entry_info(index, name, dtype, ndim, shape8, nbytes);
}
int b200_mimi_state_read(b200_mimi* h, const char* name, void* dst_dev, int64_t nbytes) {
  B200_STREAMING_ENTRY(h, "mimi_state_read");
  return h->state_entry(name, dst_dev, nullptr, nbytes, "mimi_state_read");
}
int b200_mimi_state_write(b200_mimi* h, const char* name, const void* src_dev, int64_t nbytes) {
  B200_STREAMING_ENTRY(h, "mimi_state_write");
  return h->state_entry(name, nullptr, src_dev, nbytes, "mimi_state_write");
}

int b200_mimi_error_flags(b200_mimi* h, int* flags_out) {
  B200_STREAMING_ENTRY(h, "mimi_error_flags");
  return h->error_flags(flags_out);
}

int b200_mimi_read_buffer(b200_mimi* h, const char* name, float* dst_dev, int64_t capacity, int64_t* numel) {
  B200_STREAMING_ENTRY(h, "mimi_read_buffer");
  auto it = h->taps.find(name ? name : "");
  if (it == h->taps.end()) B200_FAIL(B200_ERR_INVALID, "mimi_read_buffer: unknown buffer '%s'", name ? name : "(null)");
  const Tap& t = it->second;
  const int64_t n = (int64_t)h->batch * t.C * t.T;
  const bool transpose = t.transpose && t.T > 1;     // stored token-major [B][T][C], reported in the reference's [B][C][T]
  B200_TRY(copy_out(t.p, n, transpose ? 0 : n * 4, dst_dev, capacity, numel, h->stream, "mimi_read_buffer"));
  if (!transpose || !dst_dev) return B200_OK;
  B200_LAUNCH(tm_to_bct_kernel, (unsigned)ceil_div64(n, 256), 256, 0, h->stream, t.p, dst_dev, h->batch, t.C, t.T);
  return check_launch("mimi_read_buffer");
}

int64_t b200_mimi_algorithmic_bytes(b200_mimi* h) {
  if (!h || h->batch <= 0) return 0;
  const auto& c = h->cfg;
  // weights once per step (encode + decode; the tensor-core layers hold a hi and a lo copy: 8 bytes per parameter) + active
  // codebooks (row-major for decode, transposed for encode)
  int64_t bytes = h->weight_bytes;
  bytes += (int64_t)2 * h->num_codebooks * c.q_bins * c.q_dimension * 4 + (int64_t)4 * c.q_dimension * c.dimension * 4;
  // per session: both transformer KV rings read once, carried conv rows read + written (hi and lo), PCM in/out
  int64_t per_row = (int64_t)2 * c.tr_num_layers * 2 * c.tr_context * c.tr_d_model * 4;
  int64_t st = 0;
  for (auto* layers : {&h->enc, &h->dec})
    for (auto& l : *layers) st += (int64_t)l.cin * l.P * (l.ext_lo ? 2 : 1);
  st += (int64_t)h->down.cin * h->down.P + (int64_t)c.dimension * h->rs;
  per_row += 2 * st * 4 + (int64_t)2 * h->frame_size * 4 + h->num_codebooks * 8;
  return bytes + per_row * h->batch;
}

int b200_op_mimi_plan(const b200_mimi_config* cfg, int batch, int sms, int num_codebooks, int64_t* out, int capacity) {
  constexpr int HEAD = 6, F = 21;
  if (!cfg || !out) B200_FAIL(B200_ERR_INVALID, "op_mimi_plan: null argument");
  MimiShape g;
  B200_TRY(plan_seanet(*cfg, &g));
  if (batch < 1 || sms < 1 || num_codebooks < cfg->q_n_semantic || num_codebooks > cfg->q_n_q)
    B200_FAIL(B200_ERR_INVALID, "op_mimi_plan: batch %d, %d SMs, %d codebooks", batch, sms, num_codebooks);
  MimiPlan P;
  B200_TRY(plan_mimi(g, batch, sms, num_codebooks, &P));
  int n_tc[2] = {0, 0};
  for (int w = 0; w < 2; ++w)
    for (const SeaLayer& l : w ? g.dec : g.enc) n_tc[w] += !l.simt_first && !l.simt_last;
  const int n = n_tc[0] + n_tc[1] + 4;
  if (capacity < HEAD + F * n) B200_FAIL(B200_ERR_INVALID, "op_mimi_plan: %d layers need %d slots", n, HEAD + F * n);
  const long long head[HEAD] = {n_tc[0], n_tc[1], P.down_ksplit, (long long)P.ws_bytes, P.enc_launches, P.dec_launches};
  int k = 0;
  for (long long v : head) out[k++] = v;
  auto put = [&](int layer, const mtc::TcShape& s, const mtc::TcSchedule& q) {
    const long long v[F] = {layer, s.kind, s.Cin, s.N, s.n_taps, s.dil, s.stride, s.NT, s.n_tiles_n, s.num_kb, q.tt, q.bb, q.T,
                            q.n_sessions, q.m_tiles, q.ksplit, q.kb_per_split, q.stages, q.stage_bytes, q.grid, (long long)q.smem};
    for (long long x : v) out[k++] = x;
  };
  for (int w = 0; w < 2; ++w) {
    const std::vector<SeaLayer>& ls = w ? g.dec : g.enc;
    for (size_t i = 0; i < ls.size(); ++i)
      if (!ls[i].simt_first && !ls[i].simt_last) put((int)i, ls[i].tc.s, (w ? P.dec : P.enc)[i]);
  }
  put(0, g.in_proj, P.in_proj);
  put(1, g.out_proj, P.out_proj);
  put(2, g.linear1, P.linear1);
  put(3, g.linear2, P.linear2);
  return B200_OK;
}

}  // extern "C"
