// dcb200 engine: C-ABI implementation (include/dcb200.h) -- configuration, weight packing into
// the device operand images, workspace management and the per-chunk launch sequence.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <functional>
#include <map>
#include <string>
#include <vector>

#include "../../include/dcb200.h"
#include "../../include/dcb200_debug.h"
#include "kernels.h"

using namespace dcb;

namespace {

thread_local std::string g_create_error;

// One embedding table of the checkpoint (networks.py:375-421) and its element offset in the table blob.  The blob's
// tables start 16-byte aligned as bf16 (the embed kernel's width-8 fast path); the float32 blob uses the same offsets.
struct EmbedTable {
  const char* layer;
  int vocab, width, off;
};

struct LayerDev {
  __nv_bfloat16* wqkv = nullptr;  // 6 groups x split-bf16 [72][144][8]: q_h0, q_h1, k_h0, k_h1, v_h0, v_h1
  __nv_bfloat16* wo = nullptr;    // split-bf16 [72][288][8]
  __nv_bfloat16* w1 = nullptr;    // ff / kFFChunk groups x [36][kFFChunk][8]
  __nv_bfloat16* w2 = nullptr;    // [ff/8][288][8] (ReZero alpha folded in)
  float* b1 = nullptr;            // [ff] (both paths)
  float* b2 = nullptr;            // [288] (gain folded)
  float* ln_g[2] = {nullptr, nullptr};  // [288] pre-norm gamma/beta of the attention / FFN sub-layer (both paths)
  float* ln_b[2] = {nullptr, nullptr};
  struct {   // strict-fp32 path (strict_kernels.cu): float32 in the reference's own shapes
    float *wq = nullptr, *wk = nullptr, *wv = nullptr, *wo = nullptr, *w1 = nullptr, *w2 = nullptr, *b2 = nullptr;
    float alpha[2] = {1.f, 1.f};
  } strict;
};

// The device copy of one checkpoint.  dcb_load_weights builds a complete new set before it frees the previous one.
struct Weights {
  EmbedCol* cols = nullptr;
  EmbedRow* rowmeta = nullptr;
  __nv_bfloat16* tables = nullptr;
  __nv_bfloat16* wc = nullptr;   // split-bf16 condenser [2 Epad / 8][288][8]
  float* pe = nullptr;           // positional table [Lw][288]
  float* pe_img = nullptr;       // same table in residual-image order (window-aligned layout only)
  std::vector<LayerDev> layers;
  float *fln_g = nullptr, *fln_b = nullptr, *wfc = nullptr, *bfc = nullptr;   // final LayerNorm [288], fc1 (both paths)
  float *head_gw8 = nullptr, *head_ab = nullptr;   // head_kernel: gamma * Wfc (padded to 8) and the A / B sums
  struct {   // strict-fp32 path
    StrictEmbedRow* embed = nullptr;
    float *tables = nullptr, *wc = nullptr, *pe = nullptr;   // pe: [L][280]
  } strict;
  std::vector<void*> owned;
};

}  // namespace

struct dcb_engine {
  dcb_config cfg{};
  std::string err;
  int R = 0, L = 0, Lw = 0, E = 0, Epad = 0, echunks = 0;   // Lw: tokens per window in the layout (>= L)
  PackedLayout pl{};
  int chunk_tiles = 0, chunk_windows = 0;
  int num_sms = 132;
  cudaStream_t stream = nullptr;        // compute (+ result D2H)
  cudaStream_t copy_stream = nullptr;   // H2D of the rows of the NEXT submission, overlapping the kernels of the current one
  cudaStream_t out_stream = nullptr;    // D2H of the results of the PREVIOUS submission, off the compute stream
  // Two-deep submission pipeline (dcb_submit / dcb_wait): only the input rows and the status word are per slot; every
  // other buffer is reused in stream order.
  struct Slot {
    float* d_rows = nullptr;
    uint8_t* d_packed = nullptr;        // packed rows of a dcb_submit_packed call (allocated on first use)
    uint8_t *d_bases = nullptr, *d_quals = nullptr;   // per slot: the results of batch i are copied out on `out_stream`
    float *d_probs = nullptr, *d_logits = nullptr;    // while the kernels of batch i+1 already write the other slot's
    int* d_status = nullptr;
    int* h_status = nullptr;            // pinned
    cudaEvent_t rows_ready = nullptr, ev0 = nullptr, ev1 = nullptr, done = nullptr;
    bool busy = false, used = false;
    int64_t ticket = -1;
    int launches = 0;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> prof_events;  // around every launch when profiling
    std::vector<int> prof_kind;                                    // kernel class of each event pair
    size_t prof_used = 0;
  } slots[2];
  int64_t next_ticket = 0;
  bool weights_loaded = false;
  bool debug = false;
  bool profile = false;
  float prof_ms[6] = {0, 0, 0, 0, 0, 0};   // embed, gemm_row, qkv, attention, ffn, head
  int prof_n[6] = {0, 0, 0, 0, 0, 0};
  float prof_ffn_ms = 0.f;
  int prof_ffn_launches = 0;
  long long prof_ffn_tokens = 0;
  float last_ms = 0.f;
  int last_launches = 0;
  int last_chunk_tokens = 0;
  // model: the embedding layout follows from the configuration (dcb_create), the weights from the checkpoint
  std::vector<EmbedTable> tables;
  std::vector<StrictEmbedRow> embed;   // per input row, in concat order; table_off into the table blob
  int table_elems = 0;
  Weights w;
  // workspace
  __nv_bfloat16* d_embqkv = nullptr;
  float* d_x = nullptr;
  __nv_bfloat16* d_xb = nullptr;
  __nv_bfloat16* d_att = nullptr;
  __nv_bfloat16* d_hid = nullptr;   // FFN hidden activation, bf16 operand image [tile][ff/8][128][8]
  // stitch scratch (grown on demand)
  uint8_t *d_st_in = nullptr, *d_st_out = nullptr;   // [2][cap] each: bases|quals, seq|qual
  int32_t *d_st_start = nullptr, *d_st_len = nullptr;
  size_t st_cap = 0, st_zcap = 0;
  // post-model stage scratch (dcb_stitch_fastq / dcb_skip_mask / dcb_fill_skipped), grown on demand
  double* d_p10 = nullptr;           // 10^(-q/10), q = 0..255 (host libm pow, as NumPy)
  struct Scratch { void* p = nullptr; size_t cap = 0; } sc_pos, sc_names, sc_nameoff, sc_outcome, sc_avg, sc_recoff, sc_fastq,
      sc_bq, sc_mask, sc_ids, sc_dst, sc_tmpb, sc_tmpq,
      sc_ev_probs, sc_ev_in, sc_ev_out,   // dcb_evaluate: host probs, labels | ccs ids, loss | counts | flags
      sc_ds_in, sc_ds_out,                // dcb_distill_loss: host teacher | student logits, loss
      sc_lg_in, sc_lg_out, sc_lg_dp,      // dcb_alignment_loss_grad: host probs | labels, loss | grad | matches, DP tables
      sc_he_in, sc_he_out;                // dcb_debug_head_epilogue: logits + zero bias | probs, bases, quals
  cudaEvent_t ev_eval0 = nullptr, ev_eval1 = nullptr;
  float* d_dbg = nullptr;  // [stages][chunk_tiles * x_image]
  __nv_bfloat16* d_dbg_op = nullptr;   // bf16 operand images per stage (dbg_operand_slot)
  // strict-fp32 path (strict_kernels.cu): row-major workspace, allocated on the first strict call
  struct Strict {
    float *emb = nullptr, *x = nullptr, *y = nullptr, *q = nullptr, *k = nullptr, *v = nullptr, *att = nullptr, *hid = nullptr;
    int chunk_windows = 0;
  } strict;
  std::vector<void*> owned;   // workspace
};

namespace {

int fail(dcb_engine* e, int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (e) e->err = buf; else g_create_error = buf;
  return code;
}

// the head epilogue's calibration and cap, from the configuration
void set_head_quality(HeadParams& hp, const dcb_config& c) {
  hp.calib_enabled = c.calibration_enabled;
  hp.calib_thr = (float)c.calibration_threshold; hp.calib_w = (float)c.calibration_w; hp.calib_b = (float)c.calibration_b;
  hp.calib_thr64 = c.calibration_threshold; hp.calib_w64 = c.calibration_w; hp.calib_b64 = c.calibration_b;
  hp.max_q = (float)c.max_base_quality;
}

#define CU(e, call)                                                                     \
  do {                                                                                  \
    cudaError_t _st = (call);                                                           \
    if (_st != cudaSuccess)                                                             \
      return fail(e, DCB_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_st), \
                  __FILE__, __LINE__);                                                  \
  } while (0)

// n zeroed elements, freed with the allocations in `owned` (the engine's workspace or one weight set)
template <typename T>
int dev_alloc(dcb_engine* e, std::vector<void*>& owned, T** p, size_t n) {
  CU(e, cudaMalloc(reinterpret_cast<void**>(p), n * sizeof(T)));
  owned.push_back(*p);
  CU(e, cudaMemset(*p, 0, n * sizeof(T)));
  return DCB_OK;
}

template <typename T>
int dev_alloc(dcb_engine* e, T** p, size_t n) {
  return dev_alloc(e, e->owned, p, n);
}

template <typename T>
int upload(dcb_engine* e, std::vector<void*>& owned, T** p, const std::vector<T>& h) {
  int rc = dev_alloc(e, owned, p, h.size());
  if (rc) return rc;
  CU(e, cudaMemcpy(*p, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
  return DCB_OK;
}

// B-operand image [K/8][N][8] bf16 from a getter W(k, n) (zero outside the real extents).
std::vector<__nv_bfloat16> pack_b(int kpad, int n, const std::function<float(int, int)>& w) {
  std::vector<__nv_bfloat16> img((size_t)kpad * n);
  for (int kc = 0; kc < kpad / 8; ++kc)
    for (int r = 0; r < n; ++r)
      for (int j = 0; j < 8; ++j)
        img[((size_t)kc * n + r) * 8 + j] = __float2bfloat16(w(kc * 8 + j, r));
  return img;
}

// Split-bf16 B image [2 * kpad / 8][N][8]: the pack_b image of bf16(W), then that of bf16(W - bf16(W)).  The GEMM reads
// its A k-steps twice against it, so the product carries the weight to ~16 mantissa bits.
std::vector<__nv_bfloat16> pack_b_split(int kpad, int n, const std::function<float(int, int)>& w) {
  std::vector<__nv_bfloat16> img = pack_b(kpad, n, w);
  auto lo = pack_b(kpad, n, [&](int k, int nn) {
    const float v = w(k, nn);
    return v - __bfloat162float(__float2bfloat16(v));
  });
  img.insert(img.end(), lo.begin(), lo.end());
  return img;
}

std::vector<float> pad288(const float* src, float scale = 1.f) {
  std::vector<float> v(kDP, 0.f);
  for (int i = 0; i < kD; ++i) v[i] = src[i] * scale;
  return v;
}

// The checkpoint's variables, each looked up and shape-checked once: host pointers into the caller's tensors.
struct Checkpoint {
  struct Layer {
    float alpha[2] = {1.f, 1.f};   // ReZero
    const float *ln_g[2] = {}, *ln_b[2] = {};   // pre-LN
    const float *wq, *wk, *wv, *wo, *w1, *b1, *w2, *b2;
  };
  std::vector<const float*> tables;   // per dcb_engine::tables entry
  const float* wc;
  std::vector<Layer> layers;
  const float *fln_g, *fln_b, *wfc, *bfc;
};

int read_checkpoint(dcb_engine* e, const dcb_tensor* tensors, int n, Checkpoint* ck) {
  std::map<std::string, const dcb_tensor*> m;
  for (int i = 0; i < n; ++i)
    if (tensors[i].name) m[tensors[i].name] = &tensors[i];
  int rc = DCB_OK;   // the first failure: later lookups are skipped, so its message is the one reported
  auto get = [&](const std::string& name, std::initializer_list<int64_t> shape) -> const float* {
    if (rc) return nullptr;
    auto it = m.find(name);
    if (it == m.end()) { rc = fail(e, DCB_ERR_WEIGHTS, "missing variable %s", name.c_str()); return nullptr; }
    const dcb_tensor* t = it->second;
    bool ok = t->ndim == (int)shape.size() && t->data != nullptr;
    int i = 0;
    for (int64_t s : shape) { if (ok && t->shape[i] != s) ok = false; ++i; }
    if (!ok) { rc = fail(e, DCB_ERR_WEIGHTS, "variable %s has the wrong shape/ndim", name.c_str()); return nullptr; }
    return t->data;
  };
  const dcb_config& c = e->cfg;
  const int ff = c.filter_size;
  for (const EmbedTable& tb : e->tables)
    ck->tables.push_back(get(std::string("model/") + tb.layer + "/embeddings", {tb.vocab, tb.width}));
  ck->wc = get("model/transformer_input_condenser/kernel", {e->E, kD});
  ck->layers.resize(c.num_hidden_layers);
  for (int n_ = 0; n_ < c.num_hidden_layers; ++n_) {
    Checkpoint::Layer& l = ck->layers[n_];
    const std::string pre = "model/encoder_stack/layers/" + std::to_string(n_);
    const std::string P0 = pre + "/0", P1 = pre + "/1";
    for (int s = 0; s < 2; ++s) {
      const std::string& P = s ? P1 : P0;
      if (c.rezero) {
        if (const float* a = get(P + "/alpha", {})) l.alpha[s] = *a;
      } else {
        l.ln_g[s] = get(P + "/layer_norm/gamma", {kD});
        l.ln_b[s] = get(P + "/layer_norm/beta", {kD});
      }
    }
    l.wq = get(P0 + "/layer/query_dense_layer/kernel", {kD, kHeads, kDH});
    l.wk = get(P0 + "/layer/key_dense_layer/kernel", {kD, kHeads, kDH});
    l.wv = get(P0 + "/layer/value_dense_layer/kernel", {kD, kHeads, kDH});
    l.wo = get(P0 + "/layer/output_dense_layer/kernel", {kHeads, kDH, kD});
    l.w1 = get(P1 + "/layer/filter_dense_layer/kernel", {kD, ff});
    l.b1 = get(P1 + "/layer/filter_dense_layer/bias", {ff});
    l.w2 = get(P1 + "/layer/output_dense_layer/kernel", {ff, kD});
    l.b2 = get(P1 + "/layer/output_dense_layer/bias", {kD});
  }
  ck->fln_g = get("model/encoder_stack/output_normalization/gamma", {kD});
  ck->fln_b = get("model/encoder_stack/output_normalization/beta", {kD});
  ck->wfc = get("model/fc1/kernel", {kD, kVocab});
  ck->bfc = get("model/fc1/bias", {kVocab});
  return rc;
}

void free_weights(Weights& w) {
  for (void* p : w.owned) cudaFree(p);
  w = Weights();
}

// Both paths' device weights from a validated checkpoint, allocated in w->owned.
int upload_weights(dcb_engine* e, const Checkpoint& ck, Weights* w) {
  const dcb_config& c = e->cfg;
  int rc = DCB_OK;   // the first failure: later uploads are skipped
  auto up = [&](auto** p, const auto& h) { if (!rc) rc = upload(e, w->owned, p, h); };
  auto copy = [&](float** p, const float* src, size_t n) { up(p, std::vector<float>(src, src + n)); };

  // ---- embedding tables (networks.py:375-421), pre-scaled by sqrt(width), row 0 zeroed
  //      (ModifiedOnDeviceEmbedding, networks.py:42-63); the bf16 blob is the float32 blob rounded
  std::vector<float> blob(e->table_elems, 0.f);
  for (size_t t = 0; t < e->tables.size(); ++t) {
    const EmbedTable& tb = e->tables[t];
    const float scale = sqrtf((float)tb.width);
    for (int i = tb.width; i < tb.vocab * tb.width; ++i) blob[tb.off + i] = ck.tables[t][i] * scale;
  }
  std::vector<__nv_bfloat16> blob16(blob.size());
  for (size_t i = 0; i < blob.size(); ++i) blob16[i] = __float2bfloat16(blob[i]);
  // ---- the embed kernel's per-row id rules and per-column gather descriptors (columns E..Epad: src_row -1)
  std::vector<EmbedRow> rowmeta;
  std::vector<EmbedCol> cols(e->Epad, EmbedCol{-1, 0, 0, 0, 0, 0, 0.f});
  for (int r = 0; r < e->R; ++r) {
    const StrictEmbedRow& m = e->embed[r];
    rowmeta.push_back(EmbedRow{m.clip_hi, m.shift, m.vocab});
    for (int j = 0; j < m.width; ++j)
      cols[m.col0 + j] = EmbedCol{(int16_t)r, (int16_t)m.width, (int16_t)j, (int16_t)m.shift, m.table_off, m.vocab, m.clip_hi};
  }
  up(&w->tables, blob16);
  up(&w->rowmeta, rowmeta);
  up(&w->cols, cols);
  up(&w->strict.tables, blob);
  up(&w->strict.embed, e->embed);
  // ---- condenser (networks.py:426-434): B image [Epad/8][288][8]
  {
    const int E = e->E;
    auto img = pack_b_split(e->Epad, kDP, [&](int k, int nn) { return (k < E && nn < kD) ? ck.wc[(size_t)k * kD + nn] : 0.f; });
    up(&w->wc, img);
    copy(&w->strict.wc, ck.wc, (size_t)E * kD);
  }
  // ---- positional encoding table [Lw][288] (tf-models RelativePositionEmbedding; networks.py:301-323)
  {
    std::vector<float> pe((size_t)e->Lw * kDP, 0.f);
    if (c.add_pos_encoding) {
      const int nt = kD / 2;
      const float inc = (float)(log(1e4 / 1.0) / (double)(nt - 1));
      for (int l = 0; l < e->L; ++l)
        for (int k = 0; k < nt; ++k) {
          const float inv = expf((float)k * -inc);
          const float sc = (float)l * inv;
          pe[(size_t)l * kDP + k] = sinf(sc);
          pe[(size_t)l * kDP + nt + k] = cosf(sc);
        }
    }
    up(&w->pe, pe);
    if (e->Lw == kTileM) {
      // window-aligned layout: every tile sees positions 0..127, so the table can also be laid out like the residual
      // image [72][128][4] -- a warp of the row epilogue then reads 512 contiguous bytes instead of 32 scattered rows
      std::vector<float> img((size_t)kTileM * kDP, 0.f);
      for (int l = 0; l < kTileM; ++l)
        for (int col = 0; col < kDP; ++col) img[((size_t)(col / 4) * kTileM + l) * 4 + (col & 3)] = pe[(size_t)l * kDP + col];
      up(&w->pe_img, img);
    }
    std::vector<float> pe_strict((size_t)e->L * kD);   // the strict GEMM epilogue reads [L][280]
    for (int l = 0; l < e->L; ++l) std::copy_n(&pe[(size_t)l * kDP], kD, &pe_strict[(size_t)l * kD]);
    up(&w->strict.pe, pe_strict);
  }
  // ---- encoder layers
  const int ff = c.filter_size;
  w->layers.assign(c.num_hidden_layers, LayerDev());
  for (int n_ = 0; n_ < c.num_hidden_layers; ++n_) {
    LayerDev& ld = w->layers[n_];
    const Checkpoint::Layer& l = ck.layers[n_];
    const float alpha0 = l.alpha[0], alpha1 = l.alpha[1];
    for (int s = 0; s < 2 && !c.rezero; ++s) {
      up(&ld.ln_g[s], pad288(l.ln_g[s]));
      up(&ld.ln_b[s], pad288(l.ln_b[s]));
    }
    const float qscale = 1.0f / sqrtf((float)kDH);  // query *= depth**-0.5 (attention_layer.py:196-197)
    {
      // kQKVN / kQKVGroup n-groups of 288 columns: [q_h0 q_h1 | k_h0 k_h1 | v_h0 v_h1], each slot 144 wide (140 + 4 zero)
      std::vector<__nv_bfloat16> img;
      for (int grp = 0; grp < kQKVN / kQKVGroup; ++grp) {
        auto part = pack_b_split(kDP, kQKVGroup, [&](int k, int nn) {
          const int colg = grp * kQKVGroup + nn;
          const int slot = colg / kDHP, dd = colg % kDHP;
          if (k >= kD || dd >= kDH) return 0.f;
          const int proj = slot / kHeads, head = slot % kHeads;
          const float* wp = proj == 0 ? l.wq : (proj == 1 ? l.wk : l.wv);
          const float v = wp[((size_t)k * kHeads + head) * kDH + dd];
          return proj == 0 ? v * qscale : v;
        });
        img.insert(img.end(), part.begin(), part.end());
      }
      up(&ld.wqkv, img);
    }
    {
      // out-proj: K index = head*144 + dd, N = e; ReZero alpha folded in (encoder_stack.py:88-90)
      auto img = pack_b_split(kDP, kDP, [&](int k, int nn) {
        const int head = k / kDHP, dd = k % kDHP;
        if (dd >= kDH || nn >= kD) return 0.f;
        return l.wo[((size_t)head * kDH + dd) * kD + nn] * alpha0;
      });
      up(&ld.wo, img);
    }
    {
      // W1 in n-groups of kFFChunk hidden units, W2 as one [ff/8][288][8] image (ReZero alpha folded in)
      const int gw = kFFChunk;
      std::vector<__nv_bfloat16> img;
      img.reserve((size_t)ff * kDP);
      for (int grp = 0; grp < ff / gw; ++grp) {
        auto part = pack_b(kDP, gw, [&](int k, int nn) { return k < kD ? l.w1[(size_t)k * ff + grp * gw + nn] : 0.f; });
        img.insert(img.end(), part.begin(), part.end());
      }
      up(&ld.w1, img);
      auto img2 = pack_b(ff, kDP, [&](int k, int nn) { return nn < kD ? l.w2[(size_t)k * kD + nn] * alpha1 : 0.f; });
      up(&ld.w2, img2);
    }
    copy(&ld.b1, l.b1, ff);
    up(&ld.b2, pad288(l.b2, alpha1));
    // the strict path: every matrix once more as float32, in the reference's own shapes
    ld.strict.alpha[0] = alpha0;
    ld.strict.alpha[1] = alpha1;
    copy(&ld.strict.wq, l.wq, (size_t)kD * kD);
    copy(&ld.strict.wk, l.wk, (size_t)kD * kD);
    copy(&ld.strict.wv, l.wv, (size_t)kD * kD);
    copy(&ld.strict.wo, l.wo, (size_t)kD * kD);
    copy(&ld.strict.w1, l.w1, (size_t)kD * ff);
    copy(&ld.strict.w2, l.w2, (size_t)ff * kD);
    copy(&ld.strict.b2, l.b2, kD);
  }
  // ---- head
  up(&w->fln_g, pad288(ck.fln_g));
  up(&w->fln_b, pad288(ck.fln_b));
  copy(&w->wfc, ck.wfc, kD * kVocab);
  copy(&w->bfc, ck.bfc, kVocab);
  {
    // head_kernel folds the final LayerNorm into the fc1 sums (one pass over the row): logits_j = rstd * (sum_c y_c g_c W_cj
    // - mean_y * A_j) + B_j + bfc_j.  The products are formed here once, in float32.
    const float *g = ck.fln_g, *b = ck.fln_b, *wf = ck.wfc;
    std::vector<float> gw8((size_t)kD * 8, 0.f), ab(16, 0.f);
    for (int cc = 0; cc < kD; ++cc)
      for (int j = 0; j < kVocab; ++j) gw8[(size_t)cc * 8 + j] = g[cc] * wf[cc * kVocab + j];
    for (int j = 0; j < kVocab; ++j) {
      float a = 0.f, bsum = 0.f;
      for (int cc = 0; cc < kD; ++cc) { a += g[cc] * wf[cc * kVocab + j]; bsum += b[cc] * wf[cc * kVocab + j]; }
      ab[j] = a; ab[8 + j] = bsum;
    }
    up(&w->head_gw8, gw8);
    up(&w->head_ab, ab);
  }
  if (rc) return rc;
  // the uploads have landed before any kernel on the engine's (non-blocking) streams reads them, and no kernel still
  // reads the previous set when the caller frees it
  CU(e, cudaDeviceSynchronize());
  return DCB_OK;
}

}  // namespace

extern "C" {

const char* dcb_version(void) { return "dcb200 0.1.0 (sm_90a)"; }

const char* dcb_last_error(const dcb_engine* e) { return e ? e->err.c_str() : g_create_error.c_str(); }

int dcb_create(const dcb_config* cfg, dcb_engine** out) {
  if (!cfg || !out) return fail(nullptr, DCB_ERR_INVALID, "null argument");
  if (cfg->struct_size != (int32_t)sizeof(dcb_config))
    return fail(nullptr, DCB_ERR_INVALID, "dcb_config size mismatch: got %d, built with %zu",
                cfg->struct_size, sizeof(dcb_config));
  if (cfg->hidden_size != kD || cfg->num_heads != kHeads)
    return fail(nullptr, DCB_ERR_INVALID, "unsupported model: hidden_size=%d num_heads=%d (engine is built for %d/%d)",
                cfg->hidden_size, cfg->num_heads, kD, kHeads);
  if (!cfg->condense_transformer_input)
    return fail(nullptr, DCB_ERR_INVALID, "condense_transformer_input must be true");
  if (cfg->filter_size <= 0 || cfg->filter_size % kFFChunk || cfg->filter_size > 2048)
    return fail(nullptr, DCB_ERR_INVALID, "filter_size must be a multiple of %d and <= 2048", kFFChunk);
  if (cfg->max_passes <= 0 || cfg->max_length <= 0 || cfg->max_length > 256 || cfg->num_hidden_layers <= 0 ||
      cfg->max_batch <= 0)
    return fail(nullptr, DCB_ERR_INVALID, "bad max_passes/max_length(<=256)/num_hidden_layers/max_batch");
  if (cfg->precision != DCB_PRECISION_BF16 && cfg->precision != DCB_PRECISION_FP32)
    return fail(nullptr, DCB_ERR_INVALID, "precision must be DCB_PRECISION_BF16 or DCB_PRECISION_FP32");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail(nullptr, DCB_ERR_CUDA, "no CUDA device available (the dcb200 engine has no CPU fallback)");
  if (cfg->device < 0 || cfg->device >= ndev) return fail(nullptr, DCB_ERR_INVALID, "bad device ordinal %d", cfg->device);
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, cfg->device) != cudaSuccess || prop.major != 9)
    return fail(nullptr, DCB_ERR_CUDA, "device %d is not an sm_90 GPU (compute capability %d.%d)", cfg->device,
                prop.major, prop.minor);

  dcb_engine* e = new dcb_engine();
  e->cfg = *cfg;
  e->num_sms = prop.multiProcessorCount;
  e->L = cfg->max_length;
  e->Lw = e->L;
  bool align = true;
  int ct = cfg->chunk_tiles;
#ifdef DCB_DEV_SWITCHES
  // Developer build only (libdcb200_dev.so, csrc/build.sh): environment switches that select the alternative token
  // layout and chunking.  The product library ignores the environment.
  if (const char* env = getenv("DCB_ALIGN")) align = atoi(env) != 0;
  if (const char* env = getenv("DCB_CHUNK_TILES")) ct = atoi(env);
#endif
  // window-aligned tiling: one window per 128-token tile when it fits (the positional table is then read in residual-
  // image order); otherwise windows are packed back to back
  if (align && e->L <= kTileM) e->Lw = kTileM;
  e->R = 4 * cfg->max_passes + (cfg->use_ccs_bq ? 6 : 5);  // data_providers.py:61-78
  e->pl = make_packed_layout(cfg->max_passes, cfg->max_length, cfg->use_ccs_bq ? 1 : 0);
  {
    // the embedding in concat order (networks.py:457-506): each table once in the blob, then each input row with its
    // table, clip (data_providers.py:151-162), id shift and first column; E is the sum of the rows' widths
    auto table = [&](const char* layer, int vocab, int width) {
      const int off = (e->table_elems + 7) / 8 * 8;
      e->tables.push_back(EmbedTable{layer, vocab, width, off});
      e->table_elems = off + vocab * width;
      return e->tables.back();
    };
    auto rows = [&](const EmbedTable& tb, int n, float clip, int shift) {
      for (int r = 0; r < n; ++r) {
        e->embed.push_back(StrictEmbedRow{clip, shift, tb.vocab, tb.width, e->E, tb.off});
        e->E += tb.width;
      }
    };
    const int P = cfg->max_passes;
    const EmbedTable bases = table("bases_embedding_layer", kVocab, cfg->per_base_hidden_size);
    rows(bases, P, 0.f, 0);
    rows(table("pw_embedding_layer", cfg->pw_max + 1, cfg->pw_hidden_size), P, (float)cfg->pw_max, 0);
    rows(table("ip_embedding_layer", cfg->ip_max + 1, cfg->ip_hidden_size), P, (float)cfg->ip_max, 0);
    rows(table("strand_embedding_layer", cfg->strand_max + 1, cfg->strand_hidden_size), P, 0.f, 0);
    rows(bases, 1, 0.f, 0);                                                  // ccs shares the bases table (networks.py:485-489)
    if (cfg->use_ccs_bq)                                                     // +1 shift (networks.py:495)
      rows(table("ccs_base_quality_scores_embedding_layer", cfg->ccs_bq_max, cfg->ccs_bq_hidden_size), 1, 0.f, 1);
    rows(table("sn_embedding_layer", cfg->sn_max + 1, cfg->sn_hidden_size), 4, (float)cfg->sn_max, 0);
  }
  e->Epad = (e->E + 15) / 16 * 16;
  e->echunks = e->Epad / 8;
  if (ct <= 0) ct = 8 * e->num_sms;   // measured: larger chunks win (kernels are not DRAM-bound)
  const int max_tiles = (int)(((int64_t)cfg->max_batch * e->Lw + kTileM - 1) / kTileM);
  e->chunk_windows = std::max(1, std::min(cfg->max_batch, ct * kTileM / e->Lw));
  e->chunk_tiles = std::min(max_tiles, (e->chunk_windows * e->Lw + kTileM - 1) / kTileM);

  auto bail = [&](int rc) { std::string m = e->err; dcb_destroy(e); g_create_error = m; return rc; };
#define TRY(x) do { int _rc = (x); if (_rc) return bail(_rc); } while (0)
#define CUC(call) do { cudaError_t _s = (call); if (_s != cudaSuccess) { fail(e, DCB_ERR_CUDA, "%s: %s", #call, cudaGetErrorString(_s)); return bail(DCB_ERR_CUDA); } } while (0)
  CUC(cudaSetDevice(cfg->device));
  CUC(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
  CUC(cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking));
  CUC(cudaStreamCreateWithFlags(&e->out_stream, cudaStreamNonBlocking));
  for (auto& sl : e->slots) {
    CUC(cudaEventCreateWithFlags(&sl.rows_ready, cudaEventDisableTiming));
    CUC(cudaEventCreate(&sl.ev0));
    CUC(cudaEventCreate(&sl.ev1));
    CUC(cudaEventCreateWithFlags(&sl.done, cudaEventDisableTiming));
    CUC(cudaMallocHost(reinterpret_cast<void**>(&sl.h_status), sizeof(int)));
  }
  CUC(kernels_init());
  {
    std::vector<double> p10(256);
    for (int q = 0; q < 256; ++q) p10[q] = pow(10.0, (double)q / -10.0);    // utils.py:103: 10 ** (q / -10.0)
    TRY(upload(e, e->owned, &e->d_p10, p10));
  }
  const size_t T = e->chunk_tiles;
  for (auto& sl : e->slots) {
    TRY(dev_alloc(e, &sl.d_rows, (size_t)cfg->max_batch * e->R * e->L));
    TRY(dev_alloc(e, &sl.d_status, 1));
  }
  TRY(dev_alloc(e, &e->d_embqkv, T * kTileM * (size_t)std::max(e->Epad, kQKVN)));
  TRY(dev_alloc(e, &e->d_x, T * x_image_elems()));
  TRY(dev_alloc(e, &e->d_xb, T * act_image_elems(kDP)));
  TRY(dev_alloc(e, &e->d_att, T * act_image_elems(kDP)));
  TRY(dev_alloc(e, &e->d_hid, T * act_image_elems(cfg->filter_size)));
  const size_t mtok = (size_t)cfg->max_batch * e->L;
  for (auto& sl : e->slots) {
    TRY(dev_alloc(e, &sl.d_bases, mtok));
    TRY(dev_alloc(e, &sl.d_quals, mtok));
  }
#undef TRY
#undef CUC
  *out = e;
  return DCB_OK;
}

void dcb_destroy(dcb_engine* e) {
  if (!e) return;
  cudaSetDevice(e->cfg.device);
  if (e->copy_stream) cudaStreamSynchronize(e->copy_stream);
  if (e->stream) cudaStreamSynchronize(e->stream);
  if (e->out_stream) cudaStreamSynchronize(e->out_stream);
  for (void* p : e->owned) cudaFree(p);
  free_weights(e->w);
  if (e->d_st_in) cudaFree(e->d_st_in);
  if (e->d_st_out) cudaFree(e->d_st_out);
  if (e->d_st_start) cudaFree(e->d_st_start);
  if (e->d_st_len) cudaFree(e->d_st_len);
  for (dcb_engine::Scratch* sc : {&e->sc_pos, &e->sc_names, &e->sc_nameoff, &e->sc_outcome, &e->sc_avg, &e->sc_recoff,
                                  &e->sc_fastq, &e->sc_bq, &e->sc_mask, &e->sc_ids, &e->sc_dst, &e->sc_tmpb, &e->sc_tmpq,
                                  &e->sc_ev_probs, &e->sc_ev_in, &e->sc_ev_out, &e->sc_ds_in, &e->sc_ds_out,
                                  &e->sc_lg_in, &e->sc_lg_out, &e->sc_lg_dp, &e->sc_he_in, &e->sc_he_out})
    if (sc->p) cudaFree(sc->p);
  if (e->ev_eval0) cudaEventDestroy(e->ev_eval0);
  if (e->ev_eval1) cudaEventDestroy(e->ev_eval1);
  for (auto& sl : e->slots)
    for (auto& pr : sl.prof_events) { cudaEventDestroy(pr.first); cudaEventDestroy(pr.second); }
  if (e->copy_stream) cudaStreamSynchronize(e->copy_stream);
  for (auto& sl : e->slots) {
    if (sl.rows_ready) cudaEventDestroy(sl.rows_ready);
    if (sl.ev0) cudaEventDestroy(sl.ev0);
    if (sl.ev1) cudaEventDestroy(sl.ev1);
    if (sl.done) cudaEventDestroy(sl.done);
    if (sl.h_status) cudaFreeHost(sl.h_status);
  }
  if (e->copy_stream) cudaStreamDestroy(e->copy_stream);
  if (e->out_stream) cudaStreamDestroy(e->out_stream);
  if (e->stream) cudaStreamDestroy(e->stream);
  delete e;
}

int dcb_load_weights(dcb_engine* e, const dcb_tensor* tensors, int32_t n) {
  if (!e || !tensors) return fail(e, DCB_ERR_INVALID, "null argument");
  CU(e, cudaSetDevice(e->cfg.device));
  if (embed_smem_bytes(e->R, e->echunks, e->table_elems) > 160 * 1024)
    return fail(e, DCB_ERR_INVALID, "embedding tables + ids do not fit the embed kernel's shared memory");
  // every variable is checked before the first allocation, and the previous weights stay in use until the new set is
  // complete: a failed load changes nothing
  Checkpoint ck;
  int rc = read_checkpoint(e, tensors, n, &ck);
  if (rc) return rc;
  Weights w;
  if ((rc = upload_weights(e, ck, &w))) {
    free_weights(w);
    return rc;
  }
  free_weights(e->w);
  e->w = std::move(w);
  e->weights_loaded = true;
  return DCB_OK;
}

// One chunk of the strict-fp32 forward (strict_kernels.cu): rows [bw, R, L] -> outputs via hp.  Returns launches.
static int strict_forward_chunk(dcb_engine* e, const float* rows_chunk, int bw, const HeadParams& hp, int* d_status,
                                cudaStream_t st) {
  const dcb_config& c = e->cfg;
  dcb_engine::Strict& S = e->strict;
  const Weights& W = e->w;
  const int L = e->L, M = bw * L, ff = c.filter_size;
  int launches = 0;
  launch_strict_embed(rows_chunk, e->R, L, e->E, bw, W.strict.embed, W.strict.tables, S.emb, d_status, st); ++launches;
  {
    StrictEpi ep;
    if (c.add_pos_encoding) { ep.pe = W.strict.pe; ep.pe_L = L; }
    launch_strict_gemm(S.emb, W.strict.wc, S.x, M, kD, e->E, ep, st); ++launches;            // networks.py:509-516, :319-323
  }
  const float qscale = 1.0f / sqrtf((float)kDH);                                       // attention_layer.py:196-197
  for (int n_ = 0; n_ < c.num_hidden_layers; ++n_) {
    const LayerDev& ld = W.layers[n_];
    const float* yin = S.x;
    if (!c.rezero) { launch_strict_layernorm(S.x, S.y, M, ld.ln_g[0], ld.ln_b[0], st); ++launches; yin = S.y; }
    StrictEpi eq; eq.scale = qscale;
    launch_strict_gemm(yin, ld.strict.wq, S.q, M, kD, kD, eq, st);
    launch_strict_gemm(yin, ld.strict.wk, S.k, M, kD, kD, StrictEpi(), st);
    launch_strict_gemm(yin, ld.strict.wv, S.v, M, kD, kD, StrictEpi(), st);
    launch_strict_attention(S.q, S.k, S.v, S.att, bw, L, c.attn_win_size, st);
    StrictEpi eo; eo.residual = S.x; eo.scale = c.rezero ? ld.strict.alpha[0] : 1.f;         // encoder_stack.py:88-92
    launch_strict_gemm(S.att, ld.strict.wo, S.x, M, kD, kD, eo, st);
    launches += 5;
    yin = S.x;
    if (!c.rezero) { launch_strict_layernorm(S.x, S.y, M, ld.ln_g[1], ld.ln_b[1], st); ++launches; yin = S.y; }
    StrictEpi e1; e1.bias = ld.b1; e1.relu = 1;                                        // ffn_layer.py:83-86
    launch_strict_gemm(yin, ld.strict.w1, S.hid, M, ff, kD, e1, st);
    StrictEpi e2; e2.bias = ld.strict.b2; e2.residual = S.x; e2.scale = c.rezero ? ld.strict.alpha[1] : 1.f;
    launch_strict_gemm(S.hid, ld.strict.w2, S.x, M, kD, ff, e2, st);
    launches += 2;
  }
  HeadParams h = hp;
  h.x = S.x; h.M = M; h.L = L; h.Lw = L;
  launch_strict_head(S.x, M, h, st); ++launches;
  return launches;
}

// Where the debug capture keeps bf16 operand image `which` (DCB_DEBUG_*) of stage `stage`: element offset into d_dbg_op
// per tile row of 128 tokens and the image width.  Per stage the images are stored back to back, each chunk_tiles
// tiles long.  Returns false for a pair that is not captured.
//   stage 0     : EMBED (Epad), XB (layer 0's q/k/v operand)
//   stage 1 + 2n: QKV (864), ATT (288), XB (the FFN's operand)
//   stage 2 + 2n: HID (ff), XB (layer n + 1's q/k/v operand; not after the last layer)
static bool dbg_operand_slot(const dcb_engine* e, int stage, int which, size_t* off_cols, int* width) {
  const int layers = e->cfg.num_hidden_layers, ff = e->cfg.filter_size;
  if (stage < 0 || stage > 2 * layers) return false;
  size_t cols = 0;
  for (int s = 0; s < stage; ++s) cols += s == 0 ? e->Epad + kDP : (s & 1) ? kQKVN + 2 * kDP : ff + kDP;
  int w = -1;
  if (stage == 0) {
    if (which == DCB_DEBUG_EMBED) w = e->Epad;
    else if (which == DCB_DEBUG_XB) { cols += e->Epad; w = kDP; }
  } else if (stage & 1) {
    if (which == DCB_DEBUG_QKV) w = kQKVN;
    else if (which == DCB_DEBUG_ATT) { cols += kQKVN; w = kDP; }
    else if (which == DCB_DEBUG_XB) { cols += kQKVN + kDP; w = kDP; }
  } else {
    if (which == DCB_DEBUG_HID) w = ff;
    else if (which == DCB_DEBUG_XB && stage < 2 * layers) { cols += ff; w = kDP; }
  }
  if (w < 0) return false;
  *off_cols = cols;
  *width = w;
  return true;
}

int dcb_set_debug(dcb_engine* e, int32_t enabled) {
  if (!e) return DCB_ERR_INVALID;
  e->debug = enabled != 0;
  if (e->debug && !e->d_dbg) {
    CU(e, cudaSetDevice(e->cfg.device));
    const size_t stages = 1 + 2 * (size_t)e->cfg.num_hidden_layers;
    int rc = dev_alloc(e, &e->d_dbg, stages * e->chunk_tiles * x_image_elems());
    if (rc) return rc;
    size_t cols = 0;
    int w = 0;
    dbg_operand_slot(e, (int)stages - 1, DCB_DEBUG_HID, &cols, &w);   // the last stage holds HID only
    rc = dev_alloc(e, &e->d_dbg_op, (cols + w) * e->chunk_tiles * kTileM);
    if (rc) return rc;
  }
  return DCB_OK;
}

static int submit_impl(dcb_engine* e, const float* rows, const uint8_t* packed, int32_t batch, uint32_t flags,
                       uint8_t* bases_out, uint8_t* quals_out, float* probs_out, float* logits_out, int64_t* ticket_out) {
  if (!e || !ticket_out) return DCB_ERR_INVALID;
  if (!e->weights_loaded) return fail(e, DCB_ERR_STATE, "dcb_forward before dcb_load_weights");
  // any free slot (preferring the alternating one): a blocking dcb_forward between two submissions must not collide
  // with the slot of the one still outstanding
  int si = (int)(e->next_ticket & 1);
  if (e->slots[si].busy) si ^= 1;
  dcb_engine::Slot& sl = e->slots[si];
  if (sl.busy) return fail(e, DCB_ERR_STATE, "two submissions in flight: dcb_wait(ticket %lld) first",
                           (long long)std::min(e->slots[0].ticket, e->slots[1].ticket));
  if (batch < 0 || batch > e->cfg.max_batch) return fail(e, DCB_ERR_INVALID, "batch %d outside [0, max_batch=%d]", batch, e->cfg.max_batch);
  sl.launches = 0;
  sl.ticket = e->next_ticket;
  if (batch == 0) { sl.busy = true; sl.used = false; *ticket_out = e->next_ticket++; return DCB_OK; }
  if ((!rows && !packed) || !bases_out || !quals_out) return fail(e, DCB_ERR_INVALID, "null rows / output buffer");
  CU(e, cudaSetDevice(e->cfg.device));
  const dcb_config& c = e->cfg;
  if (packed && (c.pw_max > 255 || c.ip_max > 255)) return fail(e, DCB_ERR_INVALID, "packed rows need PW_MAX, IP_MAX <= 255");
  const int L = e->L, R = e->R;
  const size_t mtok = (size_t)c.max_batch * L;
  if (probs_out && !sl.d_probs) { int rc = dev_alloc(e, &sl.d_probs, mtok * kVocab); if (rc) return rc; }
  if (logits_out && !sl.d_logits) { int rc = dev_alloc(e, &sl.d_logits, mtok * kVocab); if (rc) return rc; }
  const bool rows_dev = flags & DCB_ROWS_ON_DEVICE;
  const bool out_dev = flags & DCB_OUT_ON_DEVICE;
  if ((flags & DCB_STRICT_FP32) && (flags & DCB_FAST_BF16)) return fail(e, DCB_ERR_INVALID, "DCB_STRICT_FP32 and DCB_FAST_BF16 are exclusive");
  const bool strict = (flags & DCB_STRICT_FP32) || (c.precision == DCB_PRECISION_FP32 && !(flags & DCB_FAST_BF16));
  if (rows_dev && ((reinterpret_cast<uintptr_t>(rows) | reinterpret_cast<uintptr_t>(packed)) & 15))
    return fail(e, DCB_ERR_INVALID, "device-resident rows must be 16-byte aligned");
  if (strict && !e->strict.emb) {
    // workspace of the strict path, on first use: ~16 k tokens per chunk
    dcb_engine::Strict& S = e->strict;
    S.chunk_windows = std::max(1, std::min(c.max_batch, 16384 / L));
    const size_t Mc = (size_t)S.chunk_windows * L;
    int rc = 0;
    if ((rc = dev_alloc(e, &S.emb, Mc * e->E)) || (rc = dev_alloc(e, &S.x, Mc * kD)) || (rc = dev_alloc(e, &S.y, Mc * kD)) ||
        (rc = dev_alloc(e, &S.q, Mc * kD)) || (rc = dev_alloc(e, &S.k, Mc * kD)) || (rc = dev_alloc(e, &S.v, Mc * kD)) ||
        (rc = dev_alloc(e, &S.att, Mc * kD)) || (rc = dev_alloc(e, &S.hid, Mc * c.filter_size)))
      return rc;
  }
  cudaStream_t st = e->stream;
  if (packed && !rows_dev && !sl.d_packed) {
    int rc = dev_alloc(e, &sl.d_packed, (size_t)c.max_batch * e->pl.stride);
    if (rc) return rc;
  }
  if (!rows_dev) {
    // The slot's previous forward (two submissions ago) was waited for before the slot was handed out again, so its
    // rows buffer is free; the copy overlaps whatever the compute stream is still running for the other slot.
    if (packed) CU(e, cudaMemcpyAsync(sl.d_packed, packed, (size_t)batch * e->pl.stride, cudaMemcpyHostToDevice, e->copy_stream));
    else CU(e, cudaMemcpyAsync(sl.d_rows, rows, (size_t)batch * R * L * sizeof(float), cudaMemcpyHostToDevice, e->copy_stream));
    CU(e, cudaEventRecord(sl.rows_ready, e->copy_stream));
    CU(e, cudaStreamWaitEvent(st, sl.rows_ready, 0));
  }
  const uint8_t* packed_base = packed ? (rows_dev ? packed : sl.d_packed) : nullptr;
  // the default path's embedding kernel reads packed rows directly; the strict path gets the float32 rows they stand for
  if (packed_base && strict) launch_unpack_rows(packed_base, e->pl, batch, sl.d_rows, st);
  const float* rows_base = packed ? sl.d_rows : (rows_dev ? rows : sl.d_rows);
  CU(e, cudaMemsetAsync(sl.d_status, 0, sizeof(int), st));
  CU(e, cudaEventRecord(sl.ev0, st));
  int launches = (packed_base && strict) ? 1 : 0;
  const size_t ximg = x_image_elems();
  bool prof_err = false;
  auto pbegin = [&](int kind) {
    if (!e->profile) return;
    if (sl.prof_used == sl.prof_events.size()) {
      cudaEvent_t a, b;
      if (cudaEventCreate(&a) != cudaSuccess || cudaEventCreate(&b) != cudaSuccess) { prof_err = true; return; }
      sl.prof_events.emplace_back(a, b);
    }
    if (sl.prof_kind.size() <= sl.prof_used) sl.prof_kind.resize(sl.prof_used + 1);
    sl.prof_kind[sl.prof_used] = kind;
    cudaEventRecord(sl.prof_events[sl.prof_used].first, st);
  };
  auto pend = [&]() {
    if (!e->profile || prof_err) return;
    cudaEventRecord(sl.prof_events[sl.prof_used].second, st);
    ++sl.prof_used;
  };
  auto make_head_at = [&](int w0) {
    HeadParams hp{};
    hp.x = e->d_x; hp.ln_g = e->w.fln_g; hp.ln_b = e->w.fln_b; hp.wfc = e->w.wfc; hp.bfc = e->w.bfc;
    hp.gw8 = e->w.head_gw8; hp.ab = e->w.head_ab;
    const size_t t0 = (size_t)w0 * L;
    hp.bases = (out_dev ? bases_out : sl.d_bases) + t0;
    hp.quals = (out_dev ? quals_out : sl.d_quals) + t0;
    hp.probs = probs_out ? ((out_dev ? probs_out : sl.d_probs) + t0 * kVocab) : nullptr;
    hp.logits = logits_out ? ((out_dev ? logits_out : sl.d_logits) + t0 * kVocab) : nullptr;
    set_head_quality(hp, c);
    return hp;
  };
  if (strict) {
    for (int w0 = 0; w0 < batch; w0 += e->strict.chunk_windows) {
      const int bw = std::min(e->strict.chunk_windows, batch - w0);
      launches += strict_forward_chunk(e, rows_base + (size_t)w0 * R * L, bw, make_head_at(w0), sl.d_status, st);
    }
  }
  for (int w0 = 0; !strict && w0 < batch; w0 += e->chunk_windows) {
    const int bw = std::min(e->chunk_windows, batch - w0);
    const int Lw = e->Lw;
    const int M = bw * Lw;          // tokens in the (possibly window-aligned) layout
    const int T = (M + kTileM - 1) / kTileM;
    const float* rows_chunk = rows_base + (size_t)w0 * R * L;
    int stage = 0;
    auto snap = [&]() {
      if (e->debug) {
        cudaMemcpyAsync(e->d_dbg + (size_t)stage * e->chunk_tiles * ximg, e->d_x, (size_t)T * ximg * sizeof(float), cudaMemcpyDeviceToDevice, st);
        // the bf16 operand images the launches since the previous snapshot wrote (stream-ordered copies only)
        const __nv_bfloat16* src[5] = {e->d_embqkv, e->d_xb, e->d_embqkv, e->d_att, e->d_hid};   // DCB_DEBUG_* order
        for (int which = 0; which < 5; ++which) {
          size_t cols = 0;
          int w = 0;
          if (dbg_operand_slot(e, stage, which, &cols, &w))
            cudaMemcpyAsync(e->d_dbg_op + cols * e->chunk_tiles * kTileM, src[which], (size_t)T * kTileM * w * sizeof(__nv_bfloat16),
                            cudaMemcpyDeviceToDevice, st);
        }
      }
      ++stage;
    };
    auto make_head = [&]() {
      HeadParams hp = make_head_at(w0);
      hp.M = M; hp.L = L; hp.Lw = Lw;
      return hp;
    };
    {
      RowEpi epi{};
      epi.x = e->d_x; epi.xb = e->d_xb; epi.bias = nullptr;
      epi.pe = c.add_pos_encoding ? e->w.pe : nullptr;
      epi.pe_img = c.add_pos_encoding ? e->w.pe_img : nullptr;
      epi.ln_g = c.rezero ? nullptr : e->w.layers[0].ln_g[0];
      epi.ln_b = c.rezero ? nullptr : e->w.layers[0].ln_b[0];
      epi.has_xold = 0; epi.L = Lw;
      pbegin(0);
      launch_embed(packed_base ? nullptr : rows_chunk, packed_base ? packed_base + (size_t)w0 * e->pl.stride : nullptr, e->pl,
                   R, L, Lw, M, T, e->echunks, e->w.cols, e->w.rowmeta, e->w.tables, e->table_elems, e->d_embqkv, sl.d_status, st);
      pend();
      pbegin(1);
      launch_gemm_row(e->d_embqkv, e->w.wc, e->Epad / 16, 2 * (e->Epad / 16), T, epi, st);
      pend();
      launches += 2;
      snap();
    }
    for (int n_ = 0; n_ < c.num_hidden_layers; ++n_) {
      const LayerDev& ld = e->w.layers[n_];
      const bool last = n_ + 1 == c.num_hidden_layers;
      pbegin(2);
      launch_gemm_qkv(e->d_xb, ld.wqkv, T, e->d_embqkv, st);
      pend();
      pbegin(3);
      launch_attention(e->d_embqkv, e->d_att, L, Lw, c.attn_win_size, bw, st);
      pend();
      // attention out-projection + residual; xb = the FFN sub-layer's input (pre-LayerNorm or identity)
      RowEpi ea{};
      ea.x = e->d_x; ea.xb = e->d_xb; ea.bias = nullptr; ea.pe = nullptr;
      ea.ln_g = c.rezero ? nullptr : ld.ln_g[1];
      ea.ln_b = c.rezero ? nullptr : ld.ln_b[1];
      ea.has_xold = 1; ea.L = Lw;
      pbegin(1);
      launch_gemm_row(e->d_att, ld.wo, kDP / 16, 2 * (kDP / 16), T, ea, st);
      pend();
      snap();
      // FFN: hidden = relu(xb W1 + b1), then hidden W2 + b2 + residual; xb = the next layer's input
      RowEpi ef{};
      ef.x = e->d_x; ef.xb = last ? nullptr : e->d_xb; ef.bias = ld.b2; ef.pe = nullptr;
      ef.ln_g = (c.rezero || last) ? nullptr : e->w.layers[n_ + 1].ln_g[0];
      ef.ln_b = (c.rezero || last) ? nullptr : e->w.layers[n_ + 1].ln_b[0];
      ef.has_xold = 1; ef.L = Lw;
      pbegin(4);
      launch_ffn_up(e->d_xb, ld.w1, ld.b1, c.filter_size, T, e->d_hid, st);
      launch_gemm_row(e->d_hid, ld.w2, c.filter_size / 16, c.filter_size / 16, T, ef, st);
      pend();
      if (e->profile) e->prof_ffn_tokens += (long long)bw * L;   // valid tokens (layout padding is not algorithmic work)
      snap();
      launches += 5;
    }
    pbegin(5);
    launch_head(make_head(), T, st);
    pend();
    ++launches;
    e->last_chunk_tokens = M;
  }
  CU(e, cudaEventRecord(sl.ev1, st));
  // results and status go back on their own stream: the compute stream is free for the next submission's kernels
  cudaStream_t os = e->out_stream;
  CU(e, cudaStreamWaitEvent(os, sl.ev1, 0));
  if (!out_dev) {
    const size_t ntok = (size_t)batch * L;
    CU(e, cudaMemcpyAsync(bases_out, sl.d_bases, ntok, cudaMemcpyDeviceToHost, os));
    CU(e, cudaMemcpyAsync(quals_out, sl.d_quals, ntok, cudaMemcpyDeviceToHost, os));
    if (probs_out) CU(e, cudaMemcpyAsync(probs_out, sl.d_probs, ntok * kVocab * sizeof(float), cudaMemcpyDeviceToHost, os));
    if (logits_out) CU(e, cudaMemcpyAsync(logits_out, sl.d_logits, ntok * kVocab * sizeof(float), cudaMemcpyDeviceToHost, os));
  }
  CU(e, cudaMemcpyAsync(sl.h_status, sl.d_status, sizeof(int), cudaMemcpyDeviceToHost, os));
  CU(e, cudaEventRecord(sl.done, os));
  CU(e, cudaGetLastError());
  sl.launches = launches;
  sl.busy = true;
  sl.used = true;
  *ticket_out = e->next_ticket++;
  return DCB_OK;
}

int dcb_submit(dcb_engine* e, const float* rows, int32_t batch, uint32_t flags, uint8_t* bases_out,
               uint8_t* quals_out, float* probs_out, float* logits_out, int64_t* ticket_out) {
  return submit_impl(e, rows, nullptr, batch, flags, bases_out, quals_out, probs_out, logits_out, ticket_out);
}

int dcb_submit_packed(dcb_engine* e, const uint8_t* packed, int32_t batch, uint32_t flags, uint8_t* bases_out,
                      uint8_t* quals_out, float* probs_out, float* logits_out, int64_t* ticket_out) {
  return submit_impl(e, nullptr, packed, batch, flags, bases_out, quals_out, probs_out, logits_out, ticket_out);
}

int dcb_forward_packed(dcb_engine* e, const uint8_t* packed, int32_t batch, uint32_t flags, uint8_t* bases_out,
                       uint8_t* quals_out, float* probs_out, float* logits_out) {
  int64_t ticket = -1;
  int rc = dcb_submit_packed(e, packed, batch, flags, bases_out, quals_out, probs_out, logits_out, &ticket);
  if (rc) return rc;
  return dcb_wait(e, ticket);
}

size_t dcb_packed_window_bytes(const dcb_config* cfg) {
  if (!cfg || cfg->max_passes <= 0 || cfg->max_length <= 0) return 0;
  return (size_t)make_packed_layout(cfg->max_passes, cfg->max_length, cfg->use_ccs_bq ? 1 : 0).stride;
}

// float32 rows [B, R, L] -> packed rows (include/dcb200.h).  Host code (no GPU, no engine): the producer side of the path.
int dcb_pack_rows(const dcb_config* cfg, const float* rows, int32_t batch, uint8_t* out) {
  if (!cfg || !rows || !out || batch < 0 || cfg->max_passes <= 0 || cfg->max_length <= 0)
    return fail(nullptr, DCB_ERR_INVALID, "dcb_pack_rows: bad argument");
  const dcb_config& c = *cfg;
  dcb_engine* e = nullptr;   // messages go to the engine-less error slot (dcb_last_error(NULL))
  if (c.pw_max > 255 || c.ip_max > 255) return fail(e, DCB_ERR_INVALID, "packed rows need PW_MAX, IP_MAX <= 255");
  const PackedLayout pl = make_packed_layout(c.max_passes, c.max_length, c.use_ccs_bq ? 1 : 0);
  const int P = pl.P, L = pl.L, R = pl.R;
  bool bad = false;
  auto trunc_clip = [](float v, int hi, bool* flag) {   // clip to [0, hi] as format_rows, then truncate as tf.cast
    if (!(v >= 0.f)) { if (v < 0.f || v != v) { if (flag) *flag = true; } return 0; }
    if (v > (float)hi) { if (flag) *flag = true; return hi; }
    return (int)v;
  };
  for (int b = 0; b < batch; ++b) {
    const float* w = rows + (size_t)b * R * L;
    uint8_t* o = out + (size_t)b * pl.stride;
    memset(o, 0, pl.stride);
    for (int p_ = 0; p_ < P; ++p_)
      for (int l = 0; l < L; ++l) {
        const int base = trunc_clip(w[(size_t)p_ * L + l], kVocab - 1, &bad);               // outside 0..4: TF raises
        const int strand = trunc_clip(w[(size_t)(3 * P + p_) * L + l], c.strand_max, &bad);
        o[p_ * L + l] = (uint8_t)(base | (strand << 3));
        o[(P + p_) * L + l] = (uint8_t)trunc_clip(w[(size_t)(P + p_) * L + l], 255, nullptr);       // clip, not an error
        o[(2 * P + p_) * L + l] = (uint8_t)trunc_clip(w[(size_t)(2 * P + p_) * L + l], 255, nullptr);
      }
    for (int l = 0; l < L; ++l) o[3 * P * L + l] = (uint8_t)trunc_clip(w[(size_t)4 * P * L + l], kVocab - 1, &bad);
    if (pl.bq)
      for (int l = 0; l < L; ++l)
        o[(3 * P + 1) * L + l] = (uint8_t)trunc_clip(w[(size_t)(4 * P + 1) * L + l] + 1.f, c.ccs_bq_max - 1, &bad);
    float* sn = reinterpret_cast<float*>(o + pl.sn_off);
    for (int i = 0; i < 4; ++i) {
      const float* row = w + (size_t)(R - 4 + i) * L;
      sn[i] = row[0];
      for (int l = 1; l < L; ++l)
        if (row[l] != row[0]) bad = true;
    }
  }
  if (bad) return fail(e, DCB_ERR_INPUT_RANGE, "dcb_pack_rows: value outside its vocabulary (clamped) or SN row not constant");
  return DCB_OK;
}

int dcb_wait(dcb_engine* e, int64_t ticket) {
  if (!e) return DCB_ERR_INVALID;
  int si = -1;
  for (int i = 0; i < 2; ++i)
    if (e->slots[i].busy && e->slots[i].ticket == ticket) si = i;
  if (ticket < 0 || si < 0) return fail(e, DCB_ERR_STATE, "dcb_wait: ticket %lld is not in flight", (long long)ticket);
  dcb_engine::Slot& sl = e->slots[si];
  sl.busy = false;
  if (!sl.used) { e->last_ms = 0.f; e->last_launches = 0; return DCB_OK; }   // empty batch
  CU(e, cudaSetDevice(e->cfg.device));
  CU(e, cudaEventSynchronize(sl.done));
  CU(e, cudaGetLastError());
  CU(e, cudaEventElapsedTime(&e->last_ms, sl.ev0, sl.ev1));
  e->last_launches = sl.launches;
  const int status = *sl.h_status;
  {
    for (size_t i = 0; i < sl.prof_used; ++i) {
      float ms = 0.f;
      CU(e, cudaEventElapsedTime(&ms, sl.prof_events[i].first, sl.prof_events[i].second));
      const int kind = sl.prof_kind[i];
      e->prof_ms[kind] += ms;
      ++e->prof_n[kind];
      if (kind == 4) { e->prof_ffn_ms += ms; ++e->prof_ffn_launches; }
    }
    sl.prof_used = 0;
  }
  if (status & 1) return fail(e, DCB_ERR_INPUT_RANGE, "embedding id out of range in the input rows (clamped)");
  return DCB_OK;
}

int dcb_forward(dcb_engine* e, const float* rows, int32_t batch, uint32_t flags, uint8_t* bases_out,
                uint8_t* quals_out, float* probs_out, float* logits_out) {
  int64_t ticket = -1;
  int rc = dcb_submit(e, rows, batch, flags, bases_out, quals_out, probs_out, logits_out, &ticket);
  if (rc) return rc;
  return dcb_wait(e, ticket);
}

int dcb_last_forward_ms(dcb_engine* e, float* ms) {
  if (!e || !ms) return DCB_ERR_INVALID;
  *ms = e->last_ms;
  return DCB_OK;
}

int dcb_last_forward_launches(dcb_engine* e, int32_t* n) {
  if (!e || !n) return DCB_ERR_INVALID;
  *n = e->last_launches;
  return DCB_OK;
}

int dcb_set_profile(dcb_engine* e, int32_t enabled) {
  if (!e) return DCB_ERR_INVALID;
  e->profile = enabled != 0;
  e->prof_ffn_ms = 0.f;
  e->prof_ffn_launches = 0;
  e->prof_ffn_tokens = 0;
  for (auto& sl : e->slots) sl.prof_used = 0;
  for (int i = 0; i < 6; ++i) { e->prof_ms[i] = 0.f; e->prof_n[i] = 0; }
  return DCB_OK;
}

int dcb_get_profile(dcb_engine* e, float* ffn_ms_total, int32_t* ffn_launches, int64_t* ffn_tokens) {
  if (!e || !ffn_ms_total || !ffn_launches || !ffn_tokens) return DCB_ERR_INVALID;
  *ffn_ms_total = e->prof_ffn_ms;
  *ffn_launches = e->prof_ffn_launches;
  *ffn_tokens = e->prof_ffn_tokens;
  return DCB_OK;
}

int dcb_get_profile_kernels(dcb_engine* e, float* ms6, int32_t* n6) {
  if (!e || !ms6 || !n6) return DCB_ERR_INVALID;
  for (int i = 0; i < 6; ++i) { ms6[i] = e->prof_ms[i]; n6[i] = e->prof_n[i]; }
  return DCB_OK;
}

int dcb_debug_residual(dcb_engine* e, int32_t stage, float* out, int64_t out_elems) {
  if (!e || !out) return DCB_ERR_INVALID;
  if (!e->debug || !e->d_dbg) return fail(e, DCB_ERR_STATE, "debug capture not enabled");
  const int stages = 1 + 2 * e->cfg.num_hidden_layers;
  if (stage < 0 || stage >= stages) return fail(e, DCB_ERR_INVALID, "stage %d outside [0,%d)", stage, stages);
  const int Mlay = e->last_chunk_tokens;               // tokens in the layout
  const int M = Mlay / e->Lw * e->L;                   // valid tokens
  if (out_elems < (int64_t)M * kD) return fail(e, DCB_ERR_INVALID, "output too small: need %lld", (long long)M * kD);
  CU(e, cudaSetDevice(e->cfg.device));
  const int T = (Mlay + kTileM - 1) / kTileM;
  std::vector<float> img((size_t)T * x_image_elems());
  CU(e, cudaMemcpy(img.data(), e->d_dbg + (size_t)stage * e->chunk_tiles * x_image_elems(), img.size() * sizeof(float), cudaMemcpyDeviceToHost));
  for (int t = 0; t < M; ++t) {
    const int tl = t / e->L * e->Lw + t % e->L;        // position of valid token t in the layout
    const int tile = tl / kTileM, r = tl % kTileM;
    for (int col = 0; col < kD; ++col)
      out[(size_t)t * kD + col] = img[(((size_t)tile * kXChunks + col / 4) * kTileM + r) * 4 + col % 4];
  }
  return DCB_OK;
}

int dcb_debug_operand(dcb_engine* e, int32_t stage, int32_t which, uint16_t* out, int64_t out_elems) {
  if (!e || !out) return DCB_ERR_INVALID;
  if (!e->debug || !e->d_dbg_op) return fail(e, DCB_ERR_STATE, "debug capture not enabled");
  size_t cols = 0;
  int w = 0;
  if (!dbg_operand_slot(e, stage, which, &cols, &w))
    return fail(e, DCB_ERR_INVALID, "operand %d is not captured at stage %d", which, stage);
  const int Mlay = e->last_chunk_tokens;               // tokens in the layout
  const int M = Mlay / e->Lw * e->L;                   // valid tokens
  if (out_elems < (int64_t)M * w) return fail(e, DCB_ERR_INVALID, "output too small: need %lld", (long long)M * w);
  CU(e, cudaSetDevice(e->cfg.device));
  const int T = (Mlay + kTileM - 1) / kTileM;
  std::vector<uint16_t> img((size_t)T * kTileM * w);
  CU(e, cudaMemcpy(img.data(), e->d_dbg_op + cols * e->chunk_tiles * kTileM, img.size() * sizeof(uint16_t), cudaMemcpyDeviceToHost));
  const int chunks = w / 8;
  for (int t = 0; t < M; ++t) {
    const int tl = t / e->L * e->Lw + t % e->L;        // position of valid token t in the layout
    const int tile = tl / kTileM, r = tl % kTileM;
    for (int col = 0; col < w; ++col)
      out[(size_t)t * w + col] = img[(((size_t)tile * chunks + col / 8) * kTileM + r) * 8 + col % 8];
  }
  return DCB_OK;
}

int dcb_stitch(dcb_engine* e, const uint8_t* bases, const uint8_t* quals, int32_t n_windows, int32_t L,
               const int32_t* zmw_start, int32_t n_zmw, uint32_t flags,
               uint8_t* seq_out, uint8_t* qual_out, int32_t* len_out) {
  if (!e) return DCB_ERR_INVALID;
  if (n_windows < 0 || L <= 0 || n_zmw < 0) return fail(e, DCB_ERR_INVALID, "dcb_stitch: negative size");
  if (n_zmw == 0 || n_windows == 0) return DCB_OK;
  if (!bases || !quals || !zmw_start || !seq_out || !qual_out || !len_out) return fail(e, DCB_ERR_INVALID, "dcb_stitch: null pointer");
  if (zmw_start[0] < 0 || zmw_start[n_zmw] > n_windows) return fail(e, DCB_ERR_INVALID, "dcb_stitch: zmw_start outside [0, n_windows]");
  for (int z = 0; z < n_zmw; ++z)
    if (zmw_start[z + 1] < zmw_start[z]) return fail(e, DCB_ERR_INVALID, "dcb_stitch: zmw_start must be non-decreasing");
  CU(e, cudaSetDevice(e->cfg.device));
  const size_t nbytes = (size_t)n_windows * L;
  const bool in_dev = flags & DCB_ROWS_ON_DEVICE, out_dev = flags & DCB_OUT_ON_DEVICE;
  cudaStream_t st = e->stream;
  if (nbytes > e->st_cap) {
    CU(e, cudaStreamSynchronize(st));
    if (e->d_st_in) cudaFree(e->d_st_in);
    if (e->d_st_out) cudaFree(e->d_st_out);
    e->d_st_in = e->d_st_out = nullptr;
    e->st_cap = 0;
    CU(e, cudaMalloc(reinterpret_cast<void**>(&e->d_st_in), 2 * nbytes));
    CU(e, cudaMalloc(reinterpret_cast<void**>(&e->d_st_out), 2 * nbytes));
    e->st_cap = nbytes;
  }
  if ((size_t)n_zmw + 1 > e->st_zcap) {
    CU(e, cudaStreamSynchronize(st));
    if (e->d_st_start) cudaFree(e->d_st_start);
    if (e->d_st_len) cudaFree(e->d_st_len);
    e->d_st_start = e->d_st_len = nullptr;
    e->st_zcap = 0;
    CU(e, cudaMalloc(reinterpret_cast<void**>(&e->d_st_start), ((size_t)n_zmw + 1) * sizeof(int32_t)));
    CU(e, cudaMalloc(reinterpret_cast<void**>(&e->d_st_len), ((size_t)n_zmw + 1) * sizeof(int32_t)));
    e->st_zcap = (size_t)n_zmw + 1;
  }
  const uint8_t *db = bases, *dq = quals;
  if (!in_dev) {
    CU(e, cudaMemcpyAsync(e->d_st_in, bases, nbytes, cudaMemcpyHostToDevice, st));
    CU(e, cudaMemcpyAsync(e->d_st_in + e->st_cap, quals, nbytes, cudaMemcpyHostToDevice, st));
    db = e->d_st_in; dq = e->d_st_in + e->st_cap;
  }
  CU(e, cudaMemcpyAsync(e->d_st_start, zmw_start, ((size_t)n_zmw + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  uint8_t* ds = out_dev ? seq_out : e->d_st_out;
  uint8_t* dqo = out_dev ? qual_out : e->d_st_out + e->st_cap;
  int32_t* dl = out_dev ? len_out : e->d_st_len;
  launch_stitch(db, dq, L, e->d_st_start, n_zmw, ds, dqo, dl, st);
  if (!out_dev) {
    CU(e, cudaMemcpyAsync(seq_out, ds, nbytes, cudaMemcpyDeviceToHost, st));
    CU(e, cudaMemcpyAsync(qual_out, dqo, nbytes, cudaMemcpyDeviceToHost, st));
    CU(e, cudaMemcpyAsync(len_out, dl, (size_t)n_zmw * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  }
  CU(e, cudaStreamSynchronize(st));
  CU(e, cudaGetLastError());
  return DCB_OK;
}

namespace {
// grow-on-demand device scratch; contents are not preserved
int ensure(dcb_engine* e, dcb_engine::Scratch& sc, size_t bytes) {
  if (bytes <= sc.cap) return DCB_OK;
  CU(e, cudaStreamSynchronize(e->stream));
  if (sc.p) cudaFree(sc.p);
  sc.p = nullptr; sc.cap = 0;
  CU(e, cudaMalloc(&sc.p, bytes));
  sc.cap = bytes;
  return DCB_OK;
}
}  // namespace

int dcb_stitch_fastq(dcb_engine* e, const uint8_t* bases, const uint8_t* quals, int32_t n_windows, int32_t L,
                     const int32_t* zmw_start, int32_t n_zmw, const int32_t* window_pos, const uint8_t* names,
                     const int32_t* name_off, double min_quality, int32_t min_length, uint32_t flags, uint8_t* fastq_out,
                     int64_t fastq_cap, int64_t* rec_off, int32_t* outcome, double* avg_q) {
  if (!e) return DCB_ERR_INVALID;
  if (n_windows < 0 || L <= 0 || n_zmw < 0 || fastq_cap < 0) return fail(e, DCB_ERR_INVALID, "dcb_stitch_fastq: negative size");
  if (!rec_off) return fail(e, DCB_ERR_INVALID, "dcb_stitch_fastq: null pointer");
  if (n_zmw == 0) { rec_off[0] = 0; return DCB_OK; }
  if (!bases || !quals || !zmw_start || !window_pos || !names || !name_off || !fastq_out || !outcome || !avg_q)
    return fail(e, DCB_ERR_INVALID, "dcb_stitch_fastq: null pointer");
  if (name_off[0] != 0) return fail(e, DCB_ERR_INVALID, "dcb_stitch_fastq: name_off[0] must be 0");
  for (int z = 0; z < n_zmw; ++z)
    if (name_off[z + 1] < name_off[z]) return fail(e, DCB_ERR_INVALID, "dcb_stitch_fastq: name_off must be non-decreasing");
  const size_t nbytes = (size_t)n_windows * L;
  // stage 1: concatenation + gap compaction (dcb_stitch), results stay on the device
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  int rc;
  // reuse dcb_stitch with device-side outputs into our own scratch
  if ((rc = ensure(e, e->sc_tmpb, nbytes ? nbytes : 1)) || (rc = ensure(e, e->sc_tmpq, nbytes ? nbytes : 1)) ||
      (rc = ensure(e, e->sc_dst, ((size_t)n_zmw + 1) * sizeof(int32_t))))
    return rc;
  uint8_t* d_seq = static_cast<uint8_t*>(e->sc_tmpb.p);
  uint8_t* d_qual = static_cast<uint8_t*>(e->sc_tmpq.p);
  int32_t* d_len = static_cast<int32_t*>(e->sc_dst.p);
  if (n_windows > 0) {
    rc = dcb_stitch(e, bases, quals, n_windows, L, zmw_start, n_zmw, (flags & DCB_ROWS_ON_DEVICE) | DCB_OUT_ON_DEVICE, d_seq, d_qual, d_len);
    if (rc) return rc;
  } else {
    CU(e, cudaMemsetAsync(d_len, 0, ((size_t)n_zmw + 1) * sizeof(int32_t), st));
  }
  const size_t names_bytes = (size_t)name_off[n_zmw];
  const size_t cap = (size_t)fastq_cap;
  if ((rc = ensure(e, e->sc_pos, (nbytes ? (size_t)n_windows : 1) * sizeof(int32_t))) ||
      (rc = ensure(e, e->sc_names, names_bytes ? names_bytes : 1)) ||
      (rc = ensure(e, e->sc_nameoff, ((size_t)n_zmw + 1) * sizeof(int32_t))) ||
      (rc = ensure(e, e->sc_outcome, (size_t)n_zmw * sizeof(int32_t))) || (rc = ensure(e, e->sc_avg, (size_t)n_zmw * sizeof(double))) ||
      (rc = ensure(e, e->sc_recoff, ((size_t)n_zmw + 1) * sizeof(int64_t))) || (rc = ensure(e, e->sc_fastq, cap ? cap : 1)))
    return rc;
  // dcb_stitch left zmw_start in its own scratch (d_st_start)
  if (n_windows == 0) {
    if ((size_t)n_zmw + 1 > e->st_zcap) {
      if (e->d_st_start) cudaFree(e->d_st_start);
      if (e->d_st_len) cudaFree(e->d_st_len);
      e->d_st_start = e->d_st_len = nullptr; e->st_zcap = 0;
      CU(e, cudaMalloc(reinterpret_cast<void**>(&e->d_st_start), ((size_t)n_zmw + 1) * sizeof(int32_t)));
      CU(e, cudaMalloc(reinterpret_cast<void**>(&e->d_st_len), ((size_t)n_zmw + 1) * sizeof(int32_t)));
      e->st_zcap = (size_t)n_zmw + 1;
    }
    CU(e, cudaMemcpyAsync(e->d_st_start, zmw_start, ((size_t)n_zmw + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  }
  if (n_windows > 0) CU(e, cudaMemcpyAsync(e->sc_pos.p, window_pos, (size_t)n_windows * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  if (names_bytes) CU(e, cudaMemcpyAsync(e->sc_names.p, names, names_bytes, cudaMemcpyHostToDevice, st));
  CU(e, cudaMemcpyAsync(e->sc_nameoff.p, name_off, ((size_t)n_zmw + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  int32_t* d_out = static_cast<int32_t*>(e->sc_outcome.p);
  double* d_avg = static_cast<double*>(e->sc_avg.p);
  int64_t* d_rec = static_cast<int64_t*>(e->sc_recoff.p);
  launch_read_outcome(d_qual, d_len, e->d_st_start, static_cast<const int32_t*>(e->sc_pos.p), L, n_zmw, e->d_p10, min_quality,
                      min_length, d_out, d_avg, st);
  launch_fastq(d_seq, d_qual, d_len, e->d_st_start, L, n_zmw, d_out, static_cast<const uint8_t*>(e->sc_names.p),
               static_cast<const int32_t*>(e->sc_nameoff.p), d_rec, static_cast<uint8_t*>(e->sc_fastq.p), fastq_cap, st);
  CU(e, cudaMemcpyAsync(rec_off, d_rec, ((size_t)n_zmw + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  CU(e, cudaMemcpyAsync(outcome, d_out, (size_t)n_zmw * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CU(e, cudaMemcpyAsync(avg_q, d_avg, (size_t)n_zmw * sizeof(double), cudaMemcpyDeviceToHost, st));
  CU(e, cudaStreamSynchronize(st));
  if (rec_off[n_zmw] > fastq_cap) return fail(e, DCB_ERR_INVALID, "dcb_stitch_fastq: fastq_out too small: need %lld bytes", (long long)rec_off[n_zmw]);
  if (rec_off[n_zmw] > 0) CU(e, cudaMemcpy(fastq_out, e->sc_fastq.p, (size_t)rec_off[n_zmw], cudaMemcpyDeviceToHost));
  CU(e, cudaGetLastError());
  return DCB_OK;
}

int dcb_skip_mask(dcb_engine* e, const int16_t* ccs_bq, int32_t n_windows, int32_t L, double skip_windows_above,
                  uint8_t* mask_out, double* avg_out) {
  if (!e) return DCB_ERR_INVALID;
  if (n_windows < 0 || L <= 0) return fail(e, DCB_ERR_INVALID, "dcb_skip_mask: negative size");
  if (n_windows == 0) return DCB_OK;
  if (!ccs_bq || !mask_out) return fail(e, DCB_ERR_INVALID, "dcb_skip_mask: null pointer");
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  const size_t n = (size_t)n_windows * L;
  int rc;
  if ((rc = ensure(e, e->sc_bq, n * sizeof(int16_t))) || (rc = ensure(e, e->sc_mask, (size_t)n_windows)) ||
      (rc = ensure(e, e->sc_avg, (size_t)n_windows * sizeof(double))))
    return rc;
  CU(e, cudaMemcpyAsync(e->sc_bq.p, ccs_bq, n * sizeof(int16_t), cudaMemcpyHostToDevice, st));
  launch_skip_mask(static_cast<const int16_t*>(e->sc_bq.p), n_windows, L, e->d_p10, skip_windows_above,
                   static_cast<uint8_t*>(e->sc_mask.p), static_cast<double*>(e->sc_avg.p), st);
  CU(e, cudaMemcpyAsync(mask_out, e->sc_mask.p, (size_t)n_windows, cudaMemcpyDeviceToHost, st));
  if (avg_out) CU(e, cudaMemcpyAsync(avg_out, e->sc_avg.p, (size_t)n_windows * sizeof(double), cudaMemcpyDeviceToHost, st));
  CU(e, cudaStreamSynchronize(st));
  CU(e, cudaGetLastError());
  return DCB_OK;
}

int dcb_fill_skipped(dcb_engine* e, const uint8_t* ccs_ids, const int16_t* ccs_bq, const int32_t* dst_window, int32_t k,
                     int32_t L, int32_t calibration_enabled, double calibration_threshold, double calibration_w,
                     double calibration_b, uint32_t flags, uint8_t* bases, uint8_t* quals) {
  if (!e) return DCB_ERR_INVALID;
  if (k < 0 || L <= 0) return fail(e, DCB_ERR_INVALID, "dcb_fill_skipped: negative size");
  if (k == 0) return DCB_OK;
  if (!ccs_ids || !ccs_bq || !dst_window || !bases || !quals) return fail(e, DCB_ERR_INVALID, "dcb_fill_skipped: null pointer");
  for (int j = 0; j < k; ++j)
    if (dst_window[j] < 0) return fail(e, DCB_ERR_INVALID, "dcb_fill_skipped: negative destination window");
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  const size_t n = (size_t)k * L;
  const bool out_dev = flags & DCB_OUT_ON_DEVICE;
  int rc;
  if ((rc = ensure(e, e->sc_ids, n)) || (rc = ensure(e, e->sc_bq, n * sizeof(int16_t))) ||
      (rc = ensure(e, e->sc_dst, ((size_t)k + 1) * sizeof(int32_t))) || (rc = ensure(e, e->sc_mask, sizeof(int))))
    return rc;
  if (!out_dev && ((rc = ensure(e, e->sc_tmpb, n)) || (rc = ensure(e, e->sc_tmpq, n)))) return rc;
  std::vector<int32_t> dst(dst_window, dst_window + k);
  if (!out_dev) for (int j = 0; j < k; ++j) dst[j] = j;      // dense temporary, scattered on the host below
  CU(e, cudaMemcpyAsync(e->sc_ids.p, ccs_ids, n, cudaMemcpyHostToDevice, st));
  CU(e, cudaMemcpyAsync(e->sc_bq.p, ccs_bq, n * sizeof(int16_t), cudaMemcpyHostToDevice, st));
  CU(e, cudaMemcpyAsync(e->sc_dst.p, dst.data(), (size_t)k * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  CU(e, cudaMemsetAsync(e->sc_mask.p, 0, sizeof(int), st));
  uint8_t* db = out_dev ? bases : static_cast<uint8_t*>(e->sc_tmpb.p);
  uint8_t* dq = out_dev ? quals : static_cast<uint8_t*>(e->sc_tmpq.p);
  launch_fill_skipped(static_cast<const uint8_t*>(e->sc_ids.p), static_cast<const int16_t*>(e->sc_bq.p),
                      static_cast<const int32_t*>(e->sc_dst.p), k, L, calibration_enabled, calibration_threshold,
                      calibration_w, calibration_b, e->cfg.max_base_quality, db, dq, static_cast<int*>(e->sc_mask.p), st);
  int status = 0;
  CU(e, cudaMemcpyAsync(&status, e->sc_mask.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  if (!out_dev) {
    std::vector<uint8_t> hb(n), hq(n);
    CU(e, cudaMemcpyAsync(hb.data(), db, n, cudaMemcpyDeviceToHost, st));
    CU(e, cudaMemcpyAsync(hq.data(), dq, n, cudaMemcpyDeviceToHost, st));
    CU(e, cudaStreamSynchronize(st));
    for (int j = 0; j < k; ++j) {
      memcpy(bases + (size_t)dst_window[j] * L, hb.data() + (size_t)j * L, L);
      memcpy(quals + (size_t)dst_window[j] * L, hq.data() + (size_t)j * L, L);
    }
  } else {
    CU(e, cudaStreamSynchronize(st));
  }
  CU(e, cudaGetLastError());
  if (status & 1) return fail(e, DCB_ERR_INPUT_RANGE, "dcb_fill_skipped: CCS base id outside 0..4 (clamped)");
  return DCB_OK;
}

int dcb_debug_head_epilogue(dcb_engine* e, const float* logits, int64_t n, uint8_t* bases, uint8_t* quals, float* probs) {
  if (!e || !logits || !bases || !quals) return DCB_ERR_INVALID;
  if (n < 0) return fail(e, DCB_ERR_INVALID, "dcb_debug_head_epilogue: negative token count");
  if (n == 0) return DCB_OK;
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  const int64_t chunk = std::min<int64_t>(n, 1 << 20);
  int rc;
  // in: [8] zero fc1 bias, then the chunk's logits; out: probs, then bases and quals
  if ((rc = ensure(e, e->sc_he_in, (8 + (size_t)chunk * kVocab) * sizeof(float))) ||
      (rc = ensure(e, e->sc_he_out, (size_t)chunk * (kVocab * sizeof(float) + 2))))
    return rc;
  float* d_bias = static_cast<float*>(e->sc_he_in.p);
  float* d_logits = d_bias + 8;
  float* d_probs = static_cast<float*>(e->sc_he_out.p);
  uint8_t* d_bases = reinterpret_cast<uint8_t*>(d_probs + (size_t)chunk * kVocab);
  uint8_t* d_quals = d_bases + chunk;
  CU(e, cudaMemsetAsync(d_bias, 0, 8 * sizeof(float), st));
  HeadParams hp{};
  hp.bfc = d_bias;
  set_head_quality(hp, e->cfg);
  hp.bases = d_bases; hp.quals = d_quals; hp.probs = probs ? d_probs : nullptr;
  for (int64_t t0 = 0; t0 < n; t0 += chunk) {
    const int m = (int)std::min<int64_t>(chunk, n - t0);
    CU(e, cudaMemcpyAsync(d_logits, logits + t0 * kVocab, (size_t)m * kVocab * sizeof(float), cudaMemcpyHostToDevice, st));
    launch_head_epilogue(d_logits, m, hp, st);
    CU(e, cudaMemcpyAsync(bases + t0, d_bases, (size_t)m, cudaMemcpyDeviceToHost, st));
    CU(e, cudaMemcpyAsync(quals + t0, d_quals, (size_t)m, cudaMemcpyDeviceToHost, st));
    if (probs) CU(e, cudaMemcpyAsync(probs + t0 * kVocab, d_probs, (size_t)m * kVocab * sizeof(float), cudaMemcpyDeviceToHost, st));
    CU(e, cudaStreamSynchronize(st));   // pageable host buffers: the next chunk reuses the scratch
  }
  CU(e, cudaGetLastError());
  return DCB_OK;
}

int dcb_evaluate(dcb_engine* e, const float* probs, const uint8_t* labels, const uint8_t* ccs_ids, int32_t batch,
                 int32_t L, double del_cost, double loss_reg, int32_t band_width, uint32_t flags, float* loss_out,
                 uint8_t* exact_out, int32_t* pred_counts, int32_t* ccs_counts, float* ms_out) {
  if (!e) return DCB_ERR_INVALID;
  if (band_width >= 0)
    return fail(e, DCB_ERR_INVALID, "dcb_evaluate: the banded alignment loss (band_width=%d) is not supported; "
                "pass DCB_BAND_WIDTH_NONE (params.band_width None, as the released models are trained)", band_width);
  if (batch < 0 || L <= 0 || L > 256) return fail(e, DCB_ERR_INVALID, "dcb_evaluate: need batch >= 0 and 0 < L <= 256");
  if (!(del_cost == del_cost)) return fail(e, DCB_ERR_INVALID, "dcb_evaluate: del_cost is NaN");
  if (ms_out) *ms_out = 0.f;
  if (batch == 0) return DCB_OK;
  if (!probs || !labels || !ccs_ids || !loss_out || !exact_out || !pred_counts || !ccs_counts)
    return fail(e, DCB_ERR_INVALID, "dcb_evaluate: null pointer");
  const size_t ntok = (size_t)batch * L;
  for (size_t i = 0; i < ntok; ++i)
    if (labels[i] > 4) return fail(e, DCB_ERR_INVALID, "dcb_evaluate: label id %d outside 0..4 at window %zu", labels[i], i / L);
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  const bool probs_dev = flags & DCB_ROWS_ON_DEVICE;
  const size_t out_bytes = (size_t)batch * (sizeof(float) + 10 * sizeof(int32_t) + 1);
  int rc;
  if ((rc = ensure(e, e->sc_ev_in, 2 * ntok)) || (rc = ensure(e, e->sc_ev_out, out_bytes)) ||
      (!probs_dev && (rc = ensure(e, e->sc_ev_probs, ntok * kVocab * sizeof(float)))))
    return rc;
  if (!e->ev_eval0) CU(e, cudaEventCreate(&e->ev_eval0));
  if (!e->ev_eval1) CU(e, cudaEventCreate(&e->ev_eval1));
  uint8_t* d_in = static_cast<uint8_t*>(e->sc_ev_in.p);
  const float* d_probs = probs;
  if (!probs_dev) {
    CU(e, cudaMemcpyAsync(e->sc_ev_probs.p, probs, ntok * kVocab * sizeof(float), cudaMemcpyHostToDevice, st));
    d_probs = static_cast<const float*>(e->sc_ev_probs.p);
  }
  CU(e, cudaMemcpyAsync(d_in, labels, ntok, cudaMemcpyHostToDevice, st));
  CU(e, cudaMemcpyAsync(d_in + ntok, ccs_ids, ntok, cudaMemcpyHostToDevice, st));
  float* d_loss = static_cast<float*>(e->sc_ev_out.p);
  int32_t* d_pred = reinterpret_cast<int32_t*>(d_loss + batch);
  int32_t* d_ccs = d_pred + (size_t)batch * 5;
  uint8_t* d_exact = reinterpret_cast<uint8_t*>(d_ccs + (size_t)batch * 5);
  const bool hard = !(loss_reg > 0.0);
  CU(e, cudaEventRecord(e->ev_eval0, st));
  CU(e, launch_evaluate(d_probs, d_in, d_in + ntok, batch, L, (float)del_cost, hard ? 1.f : (float)loss_reg, hard ? 1 : 0,
                        d_loss, d_exact, d_pred, d_ccs, st));
  CU(e, cudaEventRecord(e->ev_eval1, st));
  CU(e, cudaMemcpyAsync(loss_out, d_loss, (size_t)batch * sizeof(float), cudaMemcpyDeviceToHost, st));
  CU(e, cudaMemcpyAsync(pred_counts, d_pred, (size_t)batch * 5 * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CU(e, cudaMemcpyAsync(ccs_counts, d_ccs, (size_t)batch * 5 * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CU(e, cudaMemcpyAsync(exact_out, d_exact, (size_t)batch, cudaMemcpyDeviceToHost, st));
  CU(e, cudaStreamSynchronize(st));
  CU(e, cudaGetLastError());
  if (ms_out) CU(e, cudaEventElapsedTime(ms_out, e->ev_eval0, e->ev_eval1));
  return DCB_OK;
}

int dcb_distill_loss(dcb_engine* e, const float* teacher_logits, const float* student_logits, int32_t batch,
                     int32_t L, double temperature, int32_t logit_loss, uint32_t flags, float* loss_out,
                     float* ms_out) {
  if (!e) return DCB_ERR_INVALID;
  if (batch < 0 || L <= 0 || L > 256)
    return fail(e, DCB_ERR_INVALID, "dcb_distill_loss: need batch >= 0 and 0 < L <= 256 (batch=%d, L=%d)", batch, L);
  const float t32 = (float)temperature;   // the logits are divided in float32, as tf divides a float32 tensor
  if (!std::isfinite(temperature) || !(temperature > 0.0) || !std::isfinite(t32) || !(t32 > 0.f))
    return fail(e, DCB_ERR_INVALID, "dcb_distill_loss: temperature must be finite and > 0 in float32 (got %g)",
                temperature);
  if (logit_loss != DCB_LOGIT_LOSS_MSE && logit_loss != DCB_LOGIT_LOSS_KL)
    return fail(e, DCB_ERR_INVALID, "dcb_distill_loss: unknown logit loss id %d (DCB_LOGIT_LOSS_MSE = %d, "
                "DCB_LOGIT_LOSS_KL = %d)", logit_loss, DCB_LOGIT_LOSS_MSE, DCB_LOGIT_LOSS_KL);
  if (ms_out) *ms_out = 0.f;
  if (batch == 0) return DCB_OK;
  if (!teacher_logits || !student_logits || !loss_out)
    return fail(e, DCB_ERR_INVALID, "dcb_distill_loss: null pointer");
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  const size_t nlog = (size_t)batch * L * kVocab;
  int rc;
  if ((rc = ensure(e, e->sc_ds_out, (size_t)batch * sizeof(float))) ||
      (!(flags & DCB_ROWS_ON_DEVICE) && (rc = ensure(e, e->sc_ds_in, 2 * nlog * sizeof(float)))))
    return rc;
  if (!e->ev_eval0) CU(e, cudaEventCreate(&e->ev_eval0));
  if (!e->ev_eval1) CU(e, cudaEventCreate(&e->ev_eval1));
  const float* d_teacher = teacher_logits;
  const float* d_student = student_logits;
  if (!(flags & DCB_ROWS_ON_DEVICE)) {
    float* d_in = static_cast<float*>(e->sc_ds_in.p);
    CU(e, cudaMemcpyAsync(d_in, teacher_logits, nlog * sizeof(float), cudaMemcpyHostToDevice, st));
    CU(e, cudaMemcpyAsync(d_in + nlog, student_logits, nlog * sizeof(float), cudaMemcpyHostToDevice, st));
    d_teacher = d_in;
    d_student = d_in + nlog;
  }
  float* d_loss = static_cast<float*>(e->sc_ds_out.p);
  CU(e, cudaEventRecord(e->ev_eval0, st));
  CU(e, launch_distill_loss(d_teacher, d_student, batch, L, t32, logit_loss, d_loss, st));
  CU(e, cudaEventRecord(e->ev_eval1, st));
  CU(e, cudaMemcpyAsync(loss_out, d_loss, (size_t)batch * sizeof(float), cudaMemcpyDeviceToHost, st));
  CU(e, cudaStreamSynchronize(st));
  CU(e, cudaGetLastError());
  if (ms_out) CU(e, cudaEventElapsedTime(ms_out, e->ev_eval0, e->ev_eval1));
  return DCB_OK;
}

int dcb_alignment_loss_grad(dcb_engine* e, const float* probs, const uint8_t* labels, int32_t batch, int32_t L,
                            double del_cost, double loss_reg, int32_t band_width, uint32_t flags, float* loss_out,
                            float* grad_out, float* matches_out, float* ms_out) {
  if (!e) return DCB_ERR_INVALID;
  if (band_width >= 0)
    return fail(e, DCB_ERR_INVALID, "dcb_alignment_loss_grad: the banded alignment loss (band_width=%d) is not "
                "supported; pass DCB_BAND_WIDTH_NONE", band_width);
  if (batch < 0 || L <= 0 || L > 256)
    return fail(e, DCB_ERR_INVALID, "dcb_alignment_loss_grad: need batch >= 0 and 0 < L <= 256 (batch=%d, L=%d)", batch, L);
  if (!(del_cost == del_cost)) return fail(e, DCB_ERR_INVALID, "dcb_alignment_loss_grad: del_cost is NaN");
  if (ms_out) *ms_out = 0.f;
  if (batch == 0) return DCB_OK;
  if (!probs || !labels || !loss_out) return fail(e, DCB_ERR_INVALID, "dcb_alignment_loss_grad: null pointer");
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  const bool in_dev = flags & DCB_ROWS_ON_DEVICE, out_dev = flags & DCB_OUT_ON_DEVICE;
  const size_t ntok = (size_t)batch * L, np = ntok * kVocab * sizeof(float);
  const uint8_t* hl = labels;
  std::vector<uint8_t> lab_copy;
  if (in_dev) {   // the label check reads them on the host
    lab_copy.resize(ntok);
    CU(e, cudaMemcpyAsync(lab_copy.data(), labels, ntok, cudaMemcpyDeviceToHost, st));
    CU(e, cudaStreamSynchronize(st));
    hl = lab_copy.data();
  }
  for (size_t i = 0; i < ntok; ++i)
    if (hl[i] > 4)
      return fail(e, DCB_ERR_INVALID, "dcb_alignment_loss_grad: label id %d outside 0..4 at window %zu", hl[i], i / L);
  int ctas = 0;
  CU(e, loss_grad_grid(batch, &ctas));
  // host outputs go through scratch: loss [B] | grad [B, L, 5] | matches [B, L, L]
  const size_t n_grad = grad_out ? ntok * kVocab : 0, n_match = matches_out ? ntok * L : 0;
  int rc;
  if ((rc = ensure(e, e->sc_lg_dp, loss_grad_table_bytes(L, ctas))) ||
      (!in_dev && (rc = ensure(e, e->sc_lg_in, np + ntok))) ||
      (!out_dev && (rc = ensure(e, e->sc_lg_out, ((size_t)batch + n_grad + n_match) * sizeof(float)))))
    return rc;
  if (!e->ev_eval0) CU(e, cudaEventCreate(&e->ev_eval0));
  if (!e->ev_eval1) CU(e, cudaEventCreate(&e->ev_eval1));
  const float* d_probs = probs;
  const uint8_t* d_labels = labels;
  if (!in_dev) {
    float* d_in = static_cast<float*>(e->sc_lg_in.p);
    CU(e, cudaMemcpyAsync(d_in, probs, np, cudaMemcpyHostToDevice, st));
    CU(e, cudaMemcpyAsync(d_in + ntok * kVocab, labels, ntok, cudaMemcpyHostToDevice, st));
    d_probs = d_in;
    d_labels = reinterpret_cast<const uint8_t*>(d_in + ntok * kVocab);
  }
  float *d_loss = loss_out, *d_grad = grad_out, *d_match = matches_out;
  if (!out_dev) {
    d_loss = static_cast<float*>(e->sc_lg_out.p);
    d_grad = grad_out ? d_loss + batch : nullptr;
    d_match = matches_out ? d_loss + batch + n_grad : nullptr;
  }
  const bool hard = !(loss_reg > 0.0);
  CU(e, cudaEventRecord(e->ev_eval0, st));
  CU(e, launch_loss_grad(d_probs, d_labels, batch, L, (float)del_cost, hard ? 1.f : (float)loss_reg, hard ? 1 : 0,
                         static_cast<float*>(e->sc_lg_dp.p), ctas, d_loss, d_grad, d_match, st));
  CU(e, cudaEventRecord(e->ev_eval1, st));
  if (!out_dev) {
    CU(e, cudaMemcpyAsync(loss_out, d_loss, (size_t)batch * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (grad_out) CU(e, cudaMemcpyAsync(grad_out, d_grad, n_grad * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (matches_out) CU(e, cudaMemcpyAsync(matches_out, d_match, n_match * sizeof(float), cudaMemcpyDeviceToHost, st));
  }
  CU(e, cudaStreamSynchronize(st));
  CU(e, cudaGetLastError());
  if (ms_out) CU(e, cudaEventElapsedTime(ms_out, e->ev_eval0, e->ev_eval1));
  return DCB_OK;
}


int dcb_alloc_host(size_t bytes, void** out) {
  if (!out) return DCB_ERR_INVALID;
  return cudaMallocHost(out, bytes) == cudaSuccess ? DCB_OK : DCB_ERR_CUDA;
}
int dcb_free_host(void* p) { return cudaFreeHost(p) == cudaSuccess ? DCB_OK : DCB_ERR_CUDA; }

int dcb_alloc_device(dcb_engine* e, size_t bytes, void** out) {
  if (!e || !out) return DCB_ERR_INVALID;
  CU(e, cudaSetDevice(e->cfg.device));
  CU(e, cudaMalloc(out, bytes));
  return DCB_OK;
}
int dcb_free_device(dcb_engine* e, void* p) {
  if (!e) return DCB_ERR_INVALID;
  CU(e, cudaSetDevice(e->cfg.device));
  CU(e, cudaFree(p));
  return DCB_OK;
}
int dcb_memcpy_h2d(dcb_engine* e, void* dst, const void* src, size_t bytes) {
  if (!e) return DCB_ERR_INVALID;
  CU(e, cudaSetDevice(e->cfg.device));
  CU(e, cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice));
  return DCB_OK;
}
int dcb_memcpy_d2h(dcb_engine* e, void* dst, const void* src, size_t bytes) {
  if (!e) return DCB_ERR_INVALID;
  CU(e, cudaSetDevice(e->cfg.device));
  CU(e, cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost));
  return DCB_OK;
}
int dcb_synchronize(dcb_engine* e) {
  if (!e) return DCB_ERR_INVALID;
  CU(e, cudaSetDevice(e->cfg.device));
  CU(e, cudaDeviceSynchronize());
  return DCB_OK;
}

}  // extern "C"
