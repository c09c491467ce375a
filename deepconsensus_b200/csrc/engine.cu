// dcb200 engine: C-ABI implementation (include/dcb200.h) -- configuration, weight packing into
// the device operand images, workspace management and the per-chunk launch sequence.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/dcb200.h"
#include "../../include/dcb200_debug.h"
#include "kernels.h"

using namespace dcb;

namespace {

thread_local std::string g_create_error;

// Device memory of `cap` elements that the engine owns: freed by the destructor.  Every device allocation the engine
// makes for itself lives in one of these (allocated by alloc() or ensure() below).
template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) { reset(); std::swap(p, o.p); std::swap(cap, o.cap); }
    return *this;
  }
  ~DevBuf() { reset(); }
  operator T*() const { return p; }
  void reset() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  // a new block of n elements in place of the old one (contents undefined)
  cudaError_t reallocate(size_t n) {
    reset();
    const cudaError_t st = cudaMalloc(reinterpret_cast<void**>(&p), n * sizeof(T));
    if (st == cudaSuccess) cap = n;
    else p = nullptr;
    return st;
  }
};

// One embedding table of the checkpoint (networks.py:375-421) and its element offset in the table blob.  The blob's
// tables start 16-byte aligned as bf16 (the embed kernel's width-8 fast path); the float32 blob uses the same offsets.
struct EmbedTable {
  const char* layer;
  int vocab, width, off;
};

// One layer's GEMM weights on a float32-activation path, in the form that path's GEMM reads.
struct StrictMats {
  DevBuf<float> wq, wk, wv, wo, w1, w2;
};

struct LayerDev {
  DevBuf<__nv_bfloat16> wqkv;   // 6 groups x split-bf16 [72][144][8]: q_h0, q_h1, k_h0, k_h1, v_h0, v_h1
  DevBuf<__nv_bfloat16> wo;     // split-bf16 [72][288][8]
  DevBuf<__nv_bfloat16> w1;     // ff / kFFChunk groups x [36][kFFChunk][8]
  DevBuf<__nv_bfloat16> w2;     // [ff/8][288][8] (ReZero alpha folded in)
  DevBuf<float> b1;             // [ff] (both paths)
  DevBuf<float> b2;             // [288] (gain folded)
  DevBuf<float> ln_g[2], ln_b[2];   // [288] pre-norm gamma/beta of the attention / FFN sub-layer (both paths)
  struct : StrictMats {   // strict-fp32 path (strict_kernels.cu): float32 in the reference's own shapes
    DevBuf<float> b2;
    float alpha[2] = {1.f, 1.f};
  } strict;
  StrictMats tf32x3;      // tf32x3 path (tf32x3_kernels.cu): the same matrices as tf32x3_image (that precision only)
};

// The device copy of one checkpoint.  dcb_load_weights builds a complete new set before it frees the previous one.
struct Weights {
  DevBuf<EmbedCol> cols;
  DevBuf<EmbedRow> rowmeta;
  DevBuf<__nv_bfloat16> tables;
  DevBuf<__nv_bfloat16> wc;   // split-bf16 condenser [2 Epad / 8][288][8]
  DevBuf<float> pe;           // positional table [Lw][288]
  DevBuf<float> pe_img;       // same table in residual-image order (window-aligned layout only)
  std::vector<LayerDev> layers;
  DevBuf<float> fln_g, fln_b, wfc, bfc;   // final LayerNorm [288], fc1 (both paths)
  DevBuf<float> head_gw8, head_ab;        // head_kernel: gamma * Wfc (padded to 8) and the A / B sums
  struct {   // strict-fp32 path
    DevBuf<StrictEmbedRow> embed;
    DevBuf<float> tables, wc, pe;   // pe: [L][280]
  } strict;
  DevBuf<float> tf32x3_wc;          // the condenser as tf32x3_image (DCB_PRECISION_TF32X3 engines only)
};

// Kernel classes of the forward's profile, in dcb_get_profile_kernels' order; kProfNone: counted, never timed.
enum ProfKind { kProfEmbed, kProfRowGemm, kProfQkv, kProfAttention, kProfFfn, kProfHead, kProfKinds, kProfNone };

// The events around one profiled region of launches.
struct ProfRegion { cudaEvent_t start, end; ProfKind kind; };

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
    DevBuf<float> d_rows;
    DevBuf<uint8_t> d_packed;           // packed rows of a dcb_submit_packed call (allocated on first use)
    DevBuf<uint8_t> d_bases, d_quals;   // per slot: the results of batch i are copied out on `out_stream`
    DevBuf<float> d_probs, d_logits;    // while the kernels of batch i+1 already write the other slot's
    DevBuf<int> d_status;
    int* h_status = nullptr;            // pinned
    cudaEvent_t rows_ready = nullptr, ev0 = nullptr, ev1 = nullptr, done = nullptr;
    bool busy = false, used = false;
    int64_t ticket = -1;
    int launches = 0;
    std::vector<ProfRegion> prof;   // when profiling: the first prof_used are this submission's regions
    size_t prof_used = 0;
  } slots[2];
  int64_t next_ticket = 0;
  bool weights_loaded = false;
  bool debug = false;
  bool profile = false;
  float prof_ms[kProfKinds] = {};   // per ProfKind
  int prof_n[kProfKinds] = {};
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
  DevBuf<__nv_bfloat16> d_embqkv;
  DevBuf<float> d_x;
  DevBuf<__nv_bfloat16> d_xb;
  DevBuf<__nv_bfloat16> d_att;
  DevBuf<__nv_bfloat16> d_hid;   // FFN hidden activation, bf16 operand image [tile][ff/8][128][8] (debug capture only)
  DevBuf<int> d_flow;            // [chunk_tiles] the window-aligned forward's tile flags (TileFlow)
  uint32_t flow_stamp = 0;       // the last stamp a chunk gave them
  bool tile_flow = false;        // window-aligned layout: the forward's launches overlap through d_flow
  DevBuf<double> d_p10;          // 10^(-q/10), q = 0..255 (host libm pow, as NumPy)
  DevBuf<float> d_dbg;           // [stages][chunk_tiles * x_image]
  DevBuf<__nv_bfloat16> d_dbg_op;   // bf16 operand images per stage (dbg_operand_slot)
  // strict-fp32 path (strict_kernels.cu): row-major workspace, allocated on the first strict call
  struct Strict {
    DevBuf<float> emb, x, y, q, k, v, att, hid;
    int chunk_windows = 0;   // 0 until the workspace is allocated
    DevBuf<float> dbg;       // debug capture of the float32 forward (f32_images), allocated while debug is on
    int dbg_tokens = -1;     // tokens of the last captured chunk; -1: no float32 forward since capture was turned on
  } strict;
  // Host-or-device staging of the entry points besides the forward, one buffer per array, grown on demand (ensure,
  // stage_in, stage_out).  Every such call ends with a stream synchronisation, so the next one may reuse them.
  struct {   // dcb_stitch, dcb_stitch_fastq (and their _ragged forms)
    DevBuf<uint8_t> bases, quals, seq, qual, names, fastq;
    DevBuf<int32_t> start, len, pos, name_off, outcome;
    DevBuf<int64_t> rec_off, win_off;
    DevBuf<double> avg_q;
  } st;
  struct { DevBuf<int16_t> bq; DevBuf<uint8_t> mask; DevBuf<double> avg; } sk;   // dcb_skip_mask
  struct {   // dcb_fill_skipped(_ragged)
    DevBuf<uint8_t> ids, bases, quals; DevBuf<int16_t> bq; DevBuf<int32_t> dst; DevBuf<int64_t> src_off, dst_off; DevBuf<int> status;
  } fs;
  struct { DevBuf<float> probs, loss; DevBuf<uint8_t> labels, ccs, exact; DevBuf<int32_t> pred, ccs_counts; DevBuf<int> bad; } ev;   // dcb_evaluate
  struct { DevBuf<uint8_t> bq; DevBuf<unsigned long long> counts; DevBuf<int> bad_window; } evc;   // dcb_evaluate_calibration
  struct { DevBuf<float> teacher, student, loss, grad; } ds;   // dcb_distill_loss, dcb_distill_loss_grad
  struct { DevBuf<float> probs, loss, grad, matches, dp; DevBuf<uint8_t> labels; } lg;   // dcb_alignment_loss_grad
  struct { DevBuf<float> bias, logits, probs; DevBuf<uint8_t> bases, quals; } he;   // dcb_debug_head_epilogue
  // dcb_features_layout / dcb_features_pack: the uploaded records and the spaced state stay resident between the two
  struct {
    DevBuf<PrepZmw> zmw;
    DevBuf<int32_t> meta, noni, gap, zmw_windows, window_pos, window_width, num_passes, list, wl;
    DevBuf<int64_t> ccs_off;
    DevBuf<float> sn;
    DevBuf<uint32_t> cigar;
    DevBuf<uint8_t> bases, pw, ip, ccs_bases, ccs_bq, spaced, overflow, ccs_ids, packed;
    DevBuf<int4> op_scan, zmw_out;
    DevBuf<int4> win_list, window;
    DevBuf<int16_t> out_bq, ccs_bq_full;
    DevBuf<uint8_t> ccs_ids_full;
    DevBuf<int32_t> label_meta;       // dcb_features_labels
    DevBuf<uint32_t> label_cigar;
    DevBuf<uint8_t> label_bases, labels, label_status;
    DevBuf<int4> label_scan;
    DevBuf<int32_t> eval_dst;         // dcb_features_eval
    DevBuf<uint8_t> keep;
    DevBuf<int> eval_count;
    std::vector<int32_t> width;   // spaced width of every window of the resident layout
    DevBuf<int> status;
    PrepBatch batch{};
    int n_windows = -1;   // windows of the resident layout; -1: none
  } fp;
  struct {   // dcb_calib_count: one batch of reads, the regions, and the contig's bases (kept between calls)
    DevBuf<int32_t> meta;
    DevBuf<uint32_t> cigar;
    DevBuf<uint8_t> seq, qual, ref;
    DevBuf<int64_t> regions;
    DevBuf<long long> partial, partial_fail, out;
    int64_t ref_start = 0, ref_count = -1;   // ref_count -1: no bases uploaded yet
  } cb;
  struct {   // dcb_read_identity
    DevBuf<int32_t> meta, status;
    DevBuf<uint32_t> cigar;
    DevBuf<uint8_t> seq, qual, ref;
    DevBuf<long long> counts;
    DevBuf<double> avg_q;
  } ri;
  struct {   // dcb_read_errors: the batch, its truth slice and the slice's run bounds
    DevBuf<int32_t> meta, chunk_start, chunk_end, carry_start, carry_end, run_start, run_end;
    DevBuf<uint32_t> cigar;
    DevBuf<uint8_t> seq, qual, ref;
    DevBuf<long long> errors;
  } re;
  struct {   // dcb_kmer_*: the k-mer table and two pipeline slots of staged batches and per-read outputs
    DevBuf<unsigned long long> keys, stats, hist_partial, hist;
    DevBuf<unsigned int> counts;
    unsigned long long capacity = 0;
    int k = 0, partition = 0, n_partitions = 1;
    struct Slot {
      DevBuf<uint8_t> bases, qual, has_qual, keep;
      DevBuf<int64_t> offsets;
      DevBuf<int32_t> seg_read, seg_first;
      std::vector<int32_t> h_seg_read, h_seg_first;   // kept until the slot is reused: the copies read them
      DevBuf<long long> counts, partial;
      DevBuf<double> avg_q;
      DevBuf<int32_t> border;
      cudaEvent_t ev0 = nullptr, ev1 = nullptr;
      int n_reads = 0;
      int64_t n_bases = -1;   // of the batch staged last (dcb_kmer_set_count reuses it); -1: none
      bool query = false, quality = false;
    } slot[2];
    struct {   // dcb_kmer_set_* and dcb_kmer_spectrum: the evaluated reads' own k-mers, and the spectrum's bins
      DevBuf<unsigned long long> keys, stats, matrix;
      DevBuf<unsigned int> counts;
      unsigned long long capacity = 0;
      int partition = 0, n_partitions = 1;
    } set;
  } km;
  cudaEvent_t ev_eval0 = nullptr, ev_eval1 = nullptr;   // around the kernel of dcb_evaluate / _distill_loss / _loss_grad

  // Safe on a partly built engine.  The caller has made cfg.device current; the DevBuf members free themselves after
  // the streams have drained.
  ~dcb_engine() {
    for (cudaStream_t s : {copy_stream, stream, out_stream})
      if (s) cudaStreamSynchronize(s);
    std::vector<cudaEvent_t> events = {ev_eval0, ev_eval1, km.slot[0].ev0, km.slot[0].ev1, km.slot[1].ev0, km.slot[1].ev1};
    for (Slot& sl : slots) {
      events.insert(events.end(), {sl.rows_ready, sl.ev0, sl.ev1, sl.done});
      for (const ProfRegion& r : sl.prof) events.insert(events.end(), {r.start, r.end});
      if (sl.h_status) cudaFreeHost(sl.h_status);
    }
    for (cudaEvent_t ev : events)
      if (ev) cudaEventDestroy(ev);
    for (cudaStream_t s : {copy_stream, out_stream, stream})
      if (s) cudaStreamDestroy(s);
  }
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

// n zeroed elements (the operand images' padding columns rely on the zeros).  cudaMemset runs on the legacy default
// stream, which the engine's non-blocking streams do not wait for, so the fill completes before the buffer is used.
template <typename T>
int alloc(dcb_engine* e, DevBuf<T>& b, size_t n) {
  CU(e, b.reallocate(n));
  CU(e, cudaMemset(b.p, 0, n * sizeof(T)));
  CU(e, cudaStreamSynchronize(cudaStreamLegacy));
  return DCB_OK;
}

template <typename T>
int upload(dcb_engine* e, DevBuf<T>& b, const std::vector<T>& h) {
  int rc = alloc(e, b, h.size());
  if (rc) return rc;
  CU(e, cudaMemcpy(b.p, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
  return DCB_OK;
}

// At least n elements, grown on demand; contents are not preserved.  A kernel on the compute stream may still read the
// old block, so the stream drains before it is freed.
template <typename T>
int ensure(dcb_engine* e, DevBuf<T>& b, size_t n) {
  if (n <= b.cap) return DCB_OK;
  CU(e, cudaStreamSynchronize(e->stream));
  CU(e, b.reallocate(n));
  return DCB_OK;
}

// A host-or-device input of n elements: *d = src when the caller's array is on the device, else src copied into b on
// the compute stream.
template <typename T>
int stage_in(dcb_engine* e, DevBuf<T>& b, const T* src, size_t n, bool on_device, const T** d) {
  *d = src;
  if (on_device) return DCB_OK;
  int rc = ensure(e, b, n);
  if (rc) return rc;
  if (n) CU(e, cudaMemcpyAsync(b.p, src, n * sizeof(T), cudaMemcpyHostToDevice, e->stream));
  *d = b.p;
  return DCB_OK;
}

// A host-or-device output of n elements: the kernel writes `d`, and copy_out brings it to the caller's host array.
template <typename T>
struct Output {
  T* d = nullptr;
  T* host = nullptr;   // null when the kernel writes the caller's device array, or the caller wants no such output
  size_t n = 0;
};

template <typename T>
int stage_out(dcb_engine* e, DevBuf<T>& b, T* dst, size_t n, bool on_device, Output<T>* o) {
  *o = Output<T>{dst, nullptr, n};
  if (on_device || !dst) return DCB_OK;
  int rc = ensure(e, b, n);
  if (rc) return rc;
  *o = Output<T>{b.p, dst, n};
  return DCB_OK;
}

template <typename T>
int copy_out(dcb_engine* e, const Output<T>& o) {
  if (o.host && o.n) CU(e, cudaMemcpyAsync(o.host, o.d, o.n * sizeof(T), cudaMemcpyDeviceToHost, e->stream));
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

// Every path's device weights from a validated checkpoint (the tf32x3 images only for engines of that precision).
int upload_weights(dcb_engine* e, const Checkpoint& ck, Weights* w) {
  const dcb_config& c = e->cfg;
  int rc = DCB_OK;   // the first failure: later uploads are skipped
  auto up = [&](auto& b, const auto& h) { if (!rc) rc = upload(e, b, h); };
  auto copy = [&](DevBuf<float>& b, const float* src, size_t n) { up(b, std::vector<float>(src, src + n)); };

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
  up(w->tables, blob16);
  up(w->rowmeta, rowmeta);
  up(w->cols, cols);
  up(w->strict.tables, blob);
  up(w->strict.embed, e->embed);
  // ---- condenser (networks.py:426-434): B image [Epad/8][288][8]
  {
    const int E = e->E;
    auto img = pack_b_split(e->Epad, kDP, [&](int k, int nn) { return (k < E && nn < kD) ? ck.wc[(size_t)k * kD + nn] : 0.f; });
    up(w->wc, img);
    copy(w->strict.wc, ck.wc, (size_t)E * kD);
    if (c.precision == DCB_PRECISION_TF32X3) up(w->tf32x3_wc, tf32x3_image(ck.wc, E, kD));
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
    up(w->pe, pe);
    if (e->Lw == kTileM) {
      // window-aligned layout: every tile sees positions 0..127, so the table can also be laid out like the residual
      // image [72][128][4] -- a warp of the row epilogue then reads 512 contiguous bytes instead of 32 scattered rows
      std::vector<float> img((size_t)kTileM * kDP, 0.f);
      for (int l = 0; l < kTileM; ++l)
        for (int col = 0; col < kDP; ++col) img[((size_t)(col / 4) * kTileM + l) * 4 + (col & 3)] = pe[(size_t)l * kDP + col];
      up(w->pe_img, img);
    }
    std::vector<float> pe_strict((size_t)e->L * kD);   // the strict GEMM epilogue reads [L][280]
    for (int l = 0; l < e->L; ++l) std::copy_n(&pe[(size_t)l * kDP], kD, &pe_strict[(size_t)l * kD]);
    up(w->strict.pe, pe_strict);
  }
  // ---- encoder layers
  const int ff = c.filter_size;
  w->layers.resize(c.num_hidden_layers);
  for (int n_ = 0; n_ < c.num_hidden_layers; ++n_) {
    LayerDev& ld = w->layers[n_];
    const Checkpoint::Layer& l = ck.layers[n_];
    const float alpha0 = l.alpha[0], alpha1 = l.alpha[1];
    for (int s = 0; s < 2 && !c.rezero; ++s) {
      up(ld.ln_g[s], pad288(l.ln_g[s]));
      up(ld.ln_b[s], pad288(l.ln_b[s]));
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
      up(ld.wqkv, img);
    }
    {
      // out-proj: K index = head*144 + dd, N = e; ReZero alpha folded in (encoder_stack.py:88-90)
      auto img = pack_b_split(kDP, kDP, [&](int k, int nn) {
        const int head = k / kDHP, dd = k % kDHP;
        if (dd >= kDH || nn >= kD) return 0.f;
        return l.wo[((size_t)head * kDH + dd) * kD + nn] * alpha0;
      });
      up(ld.wo, img);
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
      up(ld.w1, img);
      auto img2 = pack_b(ff, kDP, [&](int k, int nn) { return nn < kD ? l.w2[(size_t)k * kD + nn] * alpha1 : 0.f; });
      up(ld.w2, img2);
    }
    copy(ld.b1, l.b1, ff);
    up(ld.b2, pad288(l.b2, alpha1));
    // the strict path: every matrix once more as float32, in the reference's own shapes
    ld.strict.alpha[0] = alpha0;
    ld.strict.alpha[1] = alpha1;
    copy(ld.strict.wq, l.wq, (size_t)kD * kD);
    copy(ld.strict.wk, l.wk, (size_t)kD * kD);
    copy(ld.strict.wv, l.wv, (size_t)kD * kD);
    copy(ld.strict.wo, l.wo, (size_t)kD * kD);
    copy(ld.strict.w1, l.w1, (size_t)kD * ff);
    copy(ld.strict.w2, l.w2, (size_t)ff * kD);
    copy(ld.strict.b2, l.b2, kD);
    if (c.precision == DCB_PRECISION_TF32X3) {
      StrictMats& m = ld.tf32x3;
      up(m.wq, tf32x3_image(l.wq, kD, kD));
      up(m.wk, tf32x3_image(l.wk, kD, kD));
      up(m.wv, tf32x3_image(l.wv, kD, kD));
      up(m.wo, tf32x3_image(l.wo, kD, kD));
      up(m.w1, tf32x3_image(l.w1, kD, ff));
      up(m.w2, tf32x3_image(l.w2, ff, kD));
    }
  }
  // ---- head
  up(w->fln_g, pad288(ck.fln_g));
  up(w->fln_b, pad288(ck.fln_b));
  copy(w->wfc, ck.wfc, kD * kVocab);
  copy(w->bfc, ck.bfc, kVocab);
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
    up(w->head_gw8, gw8);
    up(w->head_ab, ab);
  }
  if (rc) return rc;
  // the uploads have landed before any kernel on the engine's (non-blocking) streams reads them, and no kernel still
  // reads the previous set when the caller frees it
  CU(e, cudaDeviceSynchronize());
  return DCB_OK;
}

// Every launch of one submission's forward goes through run(): it counts the launches and, when profiling is on and
// `kind` is a kernel class, times them as one region of that class in the slot's events.
struct LaunchRecorder {
  dcb_engine* e;
  dcb_engine::Slot& sl;
  cudaStream_t st;
  int count = 0;
  template <typename F>
  void run(ProfKind kind, int n_launches, F&& launch) {
    count += n_launches;
    const ProfRegion* r = e->profile && kind != kProfNone ? begin(kind) : nullptr;
    launch();
    if (r) cudaEventRecord(r->end, st);
  }

  // the slot's next region, its start recorded; null (untimed; the forward still succeeds) if its events fail
  const ProfRegion* begin(ProfKind kind) {
    if (sl.prof_used == sl.prof.size()) {
      const bool clean = cudaPeekAtLastError() == cudaSuccess;
      ProfRegion r{nullptr, nullptr, kind};
      if (cudaEventCreate(&r.start) != cudaSuccess || cudaEventCreate(&r.end) != cudaSuccess) {
        if (r.start) cudaEventDestroy(r.start);
        if (clean) cudaGetLastError();   // only this failure is cleared, not an earlier launch's
        return nullptr;
      }
      sl.prof.push_back(r);
    }
    ProfRegion& r = sl.prof[sl.prof_used++];
    r.kind = kind;
    cudaEventRecord(r.start, st);
    return &r;
  }
};

// The head of the chunk from window w0 on: final LayerNorm, fc1, quality settings and the submission's outputs (device
// arrays; probs and logits nullable) from that window.  The chunk function sets the residual and the layout.
HeadParams chunk_head(const dcb_engine* e, uint8_t* bases, uint8_t* quals, float* probs, float* logits, int w0) {
  HeadParams hp{};
  hp.ln_g = e->w.fln_g; hp.ln_b = e->w.fln_b; hp.wfc = e->w.wfc; hp.bfc = e->w.bfc;
  hp.gw8 = e->w.head_gw8; hp.ab = e->w.head_ab;
  const size_t t0 = (size_t)w0 * e->L;
  hp.bases = bases + t0; hp.quals = quals + t0;
  hp.probs = probs ? probs + t0 * kVocab : nullptr;
  hp.logits = logits ? logits + t0 * kVocab : nullptr;
  set_head_quality(hp, e->cfg);
  return hp;
}

// The one thing the strict-fp32 and tf32x3 forwards do differently: the GEMM, and the form of the weights it reads.
struct StrictGemm {
  void (*launch)(const float* A, const float* B, float* C, int M, int N, int K, const StrictEpi& ep, cudaStream_t st);
  bool tf32x3;   // B is a tf32x3_image (LayerDev::tf32x3, Weights::tf32x3_wc), not a float32 [K][N] matrix
};
const StrictGemm kStrictGemm{launch_strict_gemm, false};
const StrictGemm kTf32x3Gemm{launch_tf32x3_gemm, true};

// One float32 image the debug capture of the float32 forward keeps: the stage and DCB_DEBUG_F32_* id it is read back
// by, the workspace buffer it is copied from, and its width.
struct F32Image { int stage, which; DevBuf<float> dcb_engine::Strict::*src; int width; };

// Every image the float32 capture keeps, in the order Strict::dbg stores them, each [strict chunk tokens][width]
// (include/dcb200_debug.h documents the list).
std::vector<F32Image> f32_images(const dcb_engine* e) {
  using S = dcb_engine::Strict;
  const int layers = e->cfg.num_hidden_layers, ff = e->cfg.filter_size;
  const bool ln = !e->cfg.rezero;
  std::vector<F32Image> v = {{0, DCB_DEBUG_F32_EMB, &S::emb, e->E}, {0, DCB_DEBUG_F32_X, &S::x, kD}};
  for (int n = 0; n < layers; ++n) {
    const int sa = 1 + 2 * n, sf = 2 + 2 * n;
    if (ln) v.push_back({sa, DCB_DEBUG_F32_Y, &S::y, kD});
    v.insert(v.end(), {{sa, DCB_DEBUG_F32_Q, &S::q, kD}, {sa, DCB_DEBUG_F32_K, &S::k, kD},
                       {sa, DCB_DEBUG_F32_V, &S::v, kD}, {sa, DCB_DEBUG_F32_ATT, &S::att, kD},
                       {sa, DCB_DEBUG_F32_X, &S::x, kD}});
    if (ln) v.push_back({sf, DCB_DEBUG_F32_Y, &S::y, kD});
    v.insert(v.end(), {{sf, DCB_DEBUG_F32_HID, &S::hid, ff}, {sf, DCB_DEBUG_F32_X, &S::x, kD}});
  }
  return v;
}

// Where Strict::dbg keeps image `which` of `stage`: its first column (per token of a full strict chunk) and its width.
// False for a pair that is not captured.
bool f32_image_slot(const dcb_engine* e, int stage, int which, size_t* cols, int* width) {
  *cols = 0;
  for (const F32Image& im : f32_images(e)) {
    if (im.stage == stage && im.which == which) { *width = im.width; return true; }
    *cols += im.width;
  }
  return false;
}

// One chunk of the strict-fp32 or tf32x3 forward (strict_kernels.cu, with the GEMM of `gemm`): rows [bw, R, L] ->
// outputs via hp.  Its launches are counted, not profiled.  With debug capture on, the images of f32_images are
// copied aside as the launches write them (stream-ordered copies, no launches).
void strict_forward_chunk(dcb_engine* e, LaunchRecorder& rec, const float* rows_chunk, int bw, HeadParams hp,
                          int* d_status, const StrictGemm& gemm) {
  const dcb_config& c = e->cfg;
  dcb_engine::Strict& S = e->strict;
  const Weights& W = e->w;
  const int L = e->L, M = bw * L, ff = c.filter_size;
  const cudaStream_t st = rec.st;
  // copies the images of `stage` whose id is in `whiches` (the ones the launches since the previous call wrote)
  auto snap = [&](int stage, std::initializer_list<int> whiches) {
    if (!e->debug || !S.dbg) return;
    const size_t Mc = (size_t)S.chunk_windows * L;
    size_t cols = 0;
    for (const F32Image& im : f32_images(e)) {
      if (im.stage == stage && std::find(whiches.begin(), whiches.end(), im.which) != whiches.end())
        cudaMemcpyAsync(S.dbg + cols * Mc, (S.*im.src).p, (size_t)M * im.width * sizeof(float), cudaMemcpyDeviceToDevice,
                        st);
      cols += im.width;
    }
  };
  rec.run(kProfNone, 2, [&] {
    launch_strict_embed(rows_chunk, e->R, L, e->E, bw, W.strict.embed, W.strict.tables, S.emb, d_status, st);
    StrictEpi ep;
    if (c.add_pos_encoding) { ep.pe = W.strict.pe; ep.pe_L = L; }
    gemm.launch(S.emb, gemm.tf32x3 ? W.tf32x3_wc.p : W.strict.wc.p, S.x, M, kD, e->E, ep, st);   // networks.py:509-516, :319-323
    snap(0, {DCB_DEBUG_F32_EMB, DCB_DEBUG_F32_X});
  });
  const float qscale = 1.0f / sqrtf((float)kDH);                                       // attention_layer.py:196-197
  for (int n_ = 0; n_ < c.num_hidden_layers; ++n_) {
    const LayerDev& ld = W.layers[n_];
    const StrictMats& wm = gemm.tf32x3 ? ld.tf32x3 : static_cast<const StrictMats&>(ld.strict);
    const float* yin = c.rezero ? S.x.p : S.y.p;   // each sub-layer's input: x, or LayerNorm(x) in y
    const int sa = 1 + 2 * n_, sf = 2 + 2 * n_;
    rec.run(kProfNone, c.rezero ? 7 : 9, [&] {
      if (!c.rezero) launch_strict_layernorm(S.x, S.y, M, ld.ln_g[0], ld.ln_b[0], st);
      StrictEpi eq; eq.scale = qscale;
      gemm.launch(yin, wm.wq, S.q, M, kD, kD, eq, st);
      gemm.launch(yin, wm.wk, S.k, M, kD, kD, StrictEpi(), st);
      gemm.launch(yin, wm.wv, S.v, M, kD, kD, StrictEpi(), st);
      launch_strict_attention(S.q, S.k, S.v, S.att, bw, L, c.attn_win_size, st);
      StrictEpi eo; eo.residual = S.x; eo.scale = c.rezero ? ld.strict.alpha[0] : 1.f;     // encoder_stack.py:88-92
      gemm.launch(S.att, wm.wo, S.x, M, kD, kD, eo, st);
      snap(sa, {DCB_DEBUG_F32_Y, DCB_DEBUG_F32_Q, DCB_DEBUG_F32_K, DCB_DEBUG_F32_V, DCB_DEBUG_F32_ATT, DCB_DEBUG_F32_X});
      if (!c.rezero) launch_strict_layernorm(S.x, S.y, M, ld.ln_g[1], ld.ln_b[1], st);
      StrictEpi e1; e1.bias = ld.b1; e1.relu = 1;                                      // ffn_layer.py:83-86
      gemm.launch(yin, wm.w1, S.hid, M, ff, kD, e1, st);
      StrictEpi e2; e2.bias = ld.strict.b2; e2.residual = S.x; e2.scale = c.rezero ? ld.strict.alpha[1] : 1.f;
      gemm.launch(S.hid, wm.w2, S.x, M, kD, ff, e2, st);
      snap(sf, {DCB_DEBUG_F32_Y, DCB_DEBUG_F32_HID, DCB_DEBUG_F32_X});
    });
  }
  hp.x = S.x; hp.M = M; hp.L = L; hp.Lw = L;
  rec.run(kProfNone, 1, [&] { launch_strict_head(S.x, M, hp, st); });
  if (e->debug && S.dbg) S.dbg_tokens = M;
}

// The row epilogue of the bf16 forward's residual GEMMs: x = [x_old +] product [+ bias] [+ positional encoding], and
// xb = the input of sub-layer `sub` (0 attention, 1 FFN) of layer `layer`: LayerNorm(x) for pre-LN models, x for
// ReZero, none after the last layer.
RowEpi row_epi(const dcb_engine* e, bool has_xold, const float* bias, int layer, int sub, bool pos) {
  const dcb_config& c = e->cfg;
  RowEpi epi{};
  epi.x = e->d_x;
  epi.bias = bias;
  if (pos && c.add_pos_encoding) { epi.pe = e->w.pe; epi.pe_img = e->w.pe_img; }
  if (layer < c.num_hidden_layers) {
    epi.xb = e->d_xb;
    if (!c.rezero) { epi.ln_g = e->w.layers[layer].ln_g[sub]; epi.ln_b = e->w.layers[layer].ln_b[sub]; }
  }
  epi.has_xold = has_xold;
  epi.L = e->Lw;
  return epi;
}

// One bf16 operand image the debug capture keeps: the stage and DCB_DEBUG_* id it is read back by, the workspace image
// it is copied from, and its width.
struct DbgImage { int stage, which; const DevBuf<__nv_bfloat16>* src; int width; };

// Every image the debug capture keeps, in the order d_dbg_op stores them (include/dcb200_debug.h documents the list).
// Each is chunk_tiles tiles long; at each stage the capture copies the images the launches since the previous one wrote.
std::vector<DbgImage> dbg_images(const dcb_engine* e) {
  const int layers = e->cfg.num_hidden_layers, ff = e->cfg.filter_size;
  std::vector<DbgImage> v = {{0, DCB_DEBUG_EMBED, &e->d_embqkv, e->Epad}, {0, DCB_DEBUG_XB, &e->d_xb, kDP}};
  for (int n = 0; n < layers; ++n) {
    v.insert(v.end(), {{1 + 2 * n, DCB_DEBUG_QKV, &e->d_embqkv, kQKVN}, {1 + 2 * n, DCB_DEBUG_ATT, &e->d_att, kDP},
                       {1 + 2 * n, DCB_DEBUG_XB, &e->d_xb, kDP}, {2 + 2 * n, DCB_DEBUG_HID, &e->d_hid, ff}});
    if (n + 1 < layers) v.push_back({2 + 2 * n, DCB_DEBUG_XB, &e->d_xb, kDP});
  }
  return v;
}

// Where d_dbg_op keeps image `which` of `stage`: its first column (per 128-token tile row) and its width.  False for a
// pair that is not captured.
bool dbg_operand_slot(const dcb_engine* e, int stage, int which, size_t* cols, int* width) {
  *cols = 0;
  for (const DbgImage& im : dbg_images(e)) {
    if (im.stage == stage && im.which == which) { *width = im.width; return true; }
    *cols += im.width;
  }
  return false;
}

// The last chunk's valid tokens of a captured image [tile][iw / K][128][K] (device) as token-major out [tokens][ow],
// ow <= iw.
template <int K, typename T>
int read_capture(dcb_engine* e, const T* image, int iw, int ow, T* out, int64_t out_elems) {
  const int Mlay = e->last_chunk_tokens;               // tokens in the layout
  const int M = Mlay / e->Lw * e->L;                   // valid tokens
  if (out_elems < (int64_t)M * ow) return fail(e, DCB_ERR_INVALID, "output too small: need %lld", (long long)M * ow);
  CU(e, cudaSetDevice(e->cfg.device));
  std::vector<T> img((size_t)(Mlay + kTileM - 1) / kTileM * kTileM * iw);
  CU(e, cudaMemcpy(img.data(), image, img.size() * sizeof(T), cudaMemcpyDeviceToHost));
  for (int t = 0; t < M; ++t) {
    const int tl = t / e->L * e->Lw + t % e->L;        // position of valid token t in the layout
    const int tile = tl / kTileM, r = tl % kTileM;
    for (int col = 0; col < ow; ++col)
      out[(size_t)t * ow + col] = img[(((size_t)tile * (iw / K) + col / K) * kTileM + r) * K + col % K];
  }
  return DCB_OK;
}

// One chunk of the bf16 forward (kernels.cu): windows from float32 rows [bw, R, L] or packed rows (the other null) ->
// outputs via hp.  With debug capture on, each stage's residual and operand images are copied aside.
void bf16_forward_chunk(dcb_engine* e, LaunchRecorder& rec, const float* rows_chunk, const uint8_t* packed_chunk,
                        int bw, HeadParams hp, int* d_status) {
  const dcb_config& c = e->cfg;
  const Weights& W = e->w;
  const int L = e->L, Lw = e->Lw, M = bw * Lw;   // M: tokens in the (possibly window-aligned) layout
  const int T = (M + kTileM - 1) / kTileM;
  const cudaStream_t st = rec.st;
  // Window-aligned layout: every launch reads only what the launches before it wrote at the same tile, so each one
  // after the embedding may start a tile once the launch before it has stamped that tile (TileFlow; kernels.cu's
  // launch() explains why the overlapping launches cannot deadlock).  A chunk's stamps follow the previous chunk's, so
  // no launch mistakes a flag an earlier chunk left for its own; when the stamps would wrap, the flags start over
  // from zero.  The embedding is a plain launch: the chunk before has completed when it starts.
  const bool flow = e->tile_flow;
  const uint32_t nstamps = 3 + 3 * (uint32_t)c.num_hidden_layers;
  if (flow && e->flow_stamp > UINT32_MAX - nstamps) {
    cudaMemsetAsync(e->d_flow, 0, e->chunk_tiles * sizeof(int), st);
    e->flow_stamp = 0;
  }
  // the flow of the chunk's next launch (both halves of a two-launch kernel share one): it waits for the stamp of the
  // launch before and leaves the next one
  auto next_flow = [&](bool advance = true) {
    TileFlow f{};
    if (flow) {
      f.flags = e->d_flow;
      f.status = d_status;
      f.wait = (int)e->flow_stamp;
      f.done = (int)(e->flow_stamp + 1);
      if (advance) ++e->flow_stamp;
    }
    return f;
  };
  int stage = 0;
  auto snap = [&]() {
    if (e->debug) {   // stream-ordered copies only
      const size_t ximg = x_image_elems(), cw = (size_t)e->chunk_tiles * kTileM;
      cudaMemcpyAsync(e->d_dbg + (size_t)stage * e->chunk_tiles * ximg, e->d_x, T * ximg * sizeof(float), cudaMemcpyDeviceToDevice, st);
      size_t cols = 0;
      for (const DbgImage& im : dbg_images(e)) {
        if (im.stage == stage)
          cudaMemcpyAsync(e->d_dbg_op + cols * cw, im.src->p, (size_t)T * kTileM * im.width * sizeof(__nv_bfloat16),
                          cudaMemcpyDeviceToDevice, st);
        cols += im.width;
      }
    }
    ++stage;
  };
  rec.run(kProfEmbed, 1, [&] {
    launch_embed(rows_chunk, packed_chunk, e->pl, e->R, L, Lw, M, T, e->echunks, W.cols, W.rowmeta, W.tables,
                 e->table_elems, e->d_embqkv, d_status, next_flow(), st);
  });
  rec.run(kProfRowGemm, 1, [&] {   // condenser + positional encoding; xb = layer 0's attention input
    launch_gemm_row(e->d_embqkv, W.wc, e->Epad / 16, 2 * (e->Epad / 16), T, row_epi(e, false, nullptr, 0, 0, true),
                    next_flow(), st);
  });
  snap();
  for (int n_ = 0; n_ < c.num_hidden_layers; ++n_) {
    const LayerDev& ld = W.layers[n_];
    if (Lw == kTileM) {
      // one window per tile: q/k/v stay on the SM, two launches over half of the tiles each (the debug capture's
      // q/k/v image is stored only when it is kept)
      rec.run(kProfAttention, 2, [&] {
        __nv_bfloat16* qkv = e->debug ? e->d_embqkv.p : nullptr;
        for (int half = 0; half < 2; ++half)
          launch_qkv_attention(half, e->d_xb, ld.wqkv, L, c.attn_win_size, T, qkv, e->d_att, next_flow(half == 1), st);
      });
    } else {
      rec.run(kProfQkv, 1, [&] { launch_gemm_qkv(e->d_xb, ld.wqkv, T, e->d_embqkv, st); });
      rec.run(kProfAttention, 1, [&] { launch_attention(e->d_embqkv, e->d_att, L, Lw, c.attn_win_size, bw, st); });
    }
    rec.run(kProfRowGemm, 1, [&] {   // attention out-projection + residual; xb = the FFN sub-layer's input
      launch_gemm_row(e->d_att, ld.wo, kDP / 16, 2 * (kDP / 16), T, row_epi(e, true, nullptr, n_, 1, false), next_flow(),
                      st);
    });
    snap();
    rec.run(kProfFfn, 2, [&] {   // relu(xb W1 + b1) W2 + b2 + residual, half of the tiles per launch; xb = next layer's
      const RowEpi epi = row_epi(e, true, ld.b2, n_ + 1, 0, false);
      __nv_bfloat16* hid = e->debug ? e->d_hid.p : nullptr;
      for (int half = 0; half < 2; ++half)
        launch_ffn(half, e->d_xb, ld.w1, ld.b1, ld.w2, c.filter_size, T, hid, epi, next_flow(half == 1), st);
    });
    if (e->profile) e->prof_ffn_tokens += (long long)bw * L;   // valid tokens (layout padding is not algorithmic work)
    snap();
  }
  hp.x = e->d_x; hp.M = M; hp.L = L; hp.Lw = Lw;
  rec.run(kProfHead, 1, [&] { launch_head(hp, T, next_flow(), st); });
  e->last_chunk_tokens = M;
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
  if (cfg->precision != DCB_PRECISION_BF16 && cfg->precision != DCB_PRECISION_FP32 && cfg->precision != DCB_PRECISION_TF32X3)
    return fail(nullptr, DCB_ERR_INVALID, "precision must be DCB_PRECISION_BF16, DCB_PRECISION_FP32 or DCB_PRECISION_TF32X3");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail(nullptr, DCB_ERR_CUDA, "no CUDA device available (the dcb200 engine has no CPU fallback)");
  if (cfg->device < 0 || cfg->device >= ndev) return fail(nullptr, DCB_ERR_INVALID, "bad device ordinal %d", cfg->device);
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, cfg->device) != cudaSuccess || prop.major != 9)
    return fail(nullptr, DCB_ERR_CUDA, "device %d is not an sm_90 GPU (compute capability %d.%d)", cfg->device,
                prop.major, prop.minor);

  std::unique_ptr<dcb_engine> eng(new dcb_engine());
  dcb_engine* e = eng.get();
  e->cfg = *cfg;
  e->num_sms = prop.multiProcessorCount;
  e->L = cfg->max_length;
  e->Lw = e->L;
  bool align = true, tile_flow = true;
#ifdef DCB_DEV_SWITCHES
  // Developer build only (libdcb200_dev.so, csrc/build.sh): environment switches that select the alternative token
  // layout (DCB_ALIGN=0) and serialize every launch of the window-aligned forward (DCB_TILE_FLOW=0).  The product
  // library ignores the environment.
  if (const char* env = getenv("DCB_ALIGN")) align = atoi(env) != 0;
  if (const char* env = getenv("DCB_TILE_FLOW")) tile_flow = atoi(env) != 0;
#endif
  // window-aligned tiling: one window per 128-token tile when it fits (the positional table is then read in residual-
  // image order); otherwise windows are packed back to back
  if (align && e->L <= kTileM) e->Lw = kTileM;
  e->tile_flow = tile_flow && e->Lw == kTileM;
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
  const int ct = cfg->chunk_tiles > 0 ? cfg->chunk_tiles : 8 * e->num_sms;   // measured: larger chunks win (kernels are not DRAM-bound)
  const int max_tiles = (int)(((int64_t)cfg->max_batch * e->Lw + kTileM - 1) / kTileM);
  e->chunk_windows = std::max(1, std::min(cfg->max_batch, ct * kTileM / e->Lw));
  e->chunk_tiles = std::min(max_tiles, (e->chunk_windows * e->Lw + kTileM - 1) / kTileM);

  // on failure the engine's destructor releases what was built, and its message becomes the create error
  const int rc = [&]() -> int {
    CU(e, cudaSetDevice(cfg->device));
    CU(e, cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
    CU(e, cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking));
    CU(e, cudaStreamCreateWithFlags(&e->out_stream, cudaStreamNonBlocking));
    for (auto& sl : e->slots) {
      CU(e, cudaEventCreateWithFlags(&sl.rows_ready, cudaEventDisableTiming));
      CU(e, cudaEventCreate(&sl.ev0));
      CU(e, cudaEventCreate(&sl.ev1));
      CU(e, cudaEventCreateWithFlags(&sl.done, cudaEventDisableTiming));
      CU(e, cudaMallocHost(reinterpret_cast<void**>(&sl.h_status), sizeof(int)));
    }
    CU(e, cudaEventCreate(&e->ev_eval0));
    CU(e, cudaEventCreate(&e->ev_eval1));
    CU(e, kernels_init());
    CU(e, tf32x3_init());
    std::vector<double> p10(256);
    for (int q = 0; q < 256; ++q) p10[q] = pow(10.0, (double)q / -10.0);    // utils.py:103: 10 ** (q / -10.0)
    int rc = upload(e, e->d_p10, p10);
    const size_t T = e->chunk_tiles, mtok = (size_t)cfg->max_batch * e->L;
    for (auto& sl : e->slots) {
      if (!rc) rc = alloc(e, sl.d_rows, (size_t)cfg->max_batch * e->R * e->L);
      if (!rc) rc = alloc(e, sl.d_status, 1);
      if (!rc) rc = alloc(e, sl.d_bases, mtok);
      if (!rc) rc = alloc(e, sl.d_quals, mtok);
    }
    if (!rc) rc = alloc(e, e->d_embqkv, T * kTileM * (size_t)std::max(e->Epad, kQKVN));
    if (!rc) rc = alloc(e, e->d_x, T * x_image_elems());
    if (!rc) rc = alloc(e, e->d_xb, T * act_image_elems(kDP));
    if (!rc) rc = alloc(e, e->d_att, T * act_image_elems(kDP));
    if (!rc && e->tile_flow) rc = alloc(e, e->d_flow, T);
    return rc;
  }();
  if (rc) {
    g_create_error = e->err;
    return rc;
  }
  *out = eng.release();
  return DCB_OK;
}

void dcb_destroy(dcb_engine* e) {
  if (!e) return;
  cudaSetDevice(e->cfg.device);
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
  if ((rc = upload_weights(e, ck, &w))) return rc;
  e->w = std::move(w);
  e->weights_loaded = true;
  return DCB_OK;
}

int dcb_set_debug(dcb_engine* e, int32_t enabled) {
  if (!e) return DCB_ERR_INVALID;
  e->debug = enabled != 0;
  if (!e->debug && e->strict.dbg) {   // the float32 capture exists only while debug is on (it can be large)
    CU(e, cudaSetDevice(e->cfg.device));
    e->strict.dbg.reset();
    e->strict.dbg_tokens = -1;
  }
  if (e->debug && !e->d_dbg) {
    CU(e, cudaSetDevice(e->cfg.device));
    const size_t stages = 1 + 2 * (size_t)e->cfg.num_hidden_layers;
    size_t cols = 0;
    for (const DbgImage& im : dbg_images(e)) cols += im.width;
    int rc = alloc(e, e->d_dbg, stages * e->chunk_tiles * x_image_elems());
    if (!rc) rc = alloc(e, e->d_dbg_op, cols * e->chunk_tiles * kTileM);
    if (!rc) rc = alloc(e, e->d_hid, e->chunk_tiles * act_image_elems(e->cfg.filter_size));
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
  sl.ticket = e->next_ticket;
  if (batch == 0) { sl.busy = true; sl.used = false; *ticket_out = e->next_ticket++; return DCB_OK; }
  if ((!rows && !packed) || !bases_out || !quals_out) return fail(e, DCB_ERR_INVALID, "null rows / output buffer");
  CU(e, cudaSetDevice(e->cfg.device));
  const dcb_config& c = e->cfg;
  if (packed && (c.pw_max > 255 || c.ip_max > 255 || c.strand_max > 3 || c.ccs_bq_max > 256))
    return fail(e, DCB_ERR_INVALID, "packed rows need PW_MAX, IP_MAX <= 255, STRAND_MAX <= 3 and CCS_BQ_MAX <= 256");
  const int L = e->L, R = e->R;
  const size_t mtok = (size_t)c.max_batch * L;
  if (probs_out && !sl.d_probs) { int rc = alloc(e, sl.d_probs, mtok * kVocab); if (rc) return rc; }
  if (logits_out && !sl.d_logits) { int rc = alloc(e, sl.d_logits, mtok * kVocab); if (rc) return rc; }
  const bool rows_dev = flags & DCB_ROWS_ON_DEVICE;
  const bool out_dev = flags & DCB_OUT_ON_DEVICE;
  if ((flags & DCB_STRICT_FP32) && (flags & DCB_FAST_BF16)) return fail(e, DCB_ERR_INVALID, "DCB_STRICT_FP32 and DCB_FAST_BF16 are exclusive");
  const bool strict = (flags & DCB_STRICT_FP32) || (c.precision == DCB_PRECISION_FP32 && !(flags & DCB_FAST_BF16));
  const bool tf32x3 = c.precision == DCB_PRECISION_TF32X3 && !(flags & (DCB_STRICT_FP32 | DCB_FAST_BF16));
  const bool f32 = strict || tf32x3;   // the strict path's forward: float32 rows and activations
  if (rows_dev && ((reinterpret_cast<uintptr_t>(rows) | reinterpret_cast<uintptr_t>(packed)) & 15))
    return fail(e, DCB_ERR_INVALID, "device-resident rows must be 16-byte aligned");
  if (f32 && !e->strict.chunk_windows) {
    // workspace of the strict path, on first use: ~16 k tokens per chunk
    dcb_engine::Strict& S = e->strict;
    const int cw = std::max(1, std::min(c.max_batch, 16384 / L));
    const size_t Mc = (size_t)cw * L;
    int rc = alloc(e, S.emb, Mc * e->E);
    for (DevBuf<float>* b : {&S.x, &S.y, &S.q, &S.k, &S.v, &S.att})
      if (!rc) rc = alloc(e, *b, Mc * kD);
    if (!rc) rc = alloc(e, S.hid, Mc * c.filter_size);
    if (rc) return rc;
    S.chunk_windows = cw;
  }
  if (f32 && e->debug && !e->strict.dbg) {
    // the float32 capture, on the first float32 forward with debug on: every image of f32_images for a full chunk
    size_t cols = 0;
    for (const F32Image& im : f32_images(e)) cols += im.width;
    int rc = alloc(e, e->strict.dbg, cols * e->strict.chunk_windows * L);
    if (rc) return rc;
  }
  cudaStream_t st = e->stream;
  if (packed && !rows_dev && !sl.d_packed) {
    int rc = alloc(e, sl.d_packed, (size_t)c.max_batch * e->pl.stride);
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
  LaunchRecorder rec{e, sl, st};
  const uint8_t* packed_base = packed ? (rows_dev ? packed : sl.d_packed) : nullptr;
  // the default path's embedding kernel reads packed rows directly; the strict path gets the float32 rows they stand for
  if (packed_base && f32) rec.run(kProfNone, 1, [&] { launch_unpack_rows(packed_base, e->pl, batch, sl.d_rows, st); });
  const float* rows_base = packed ? sl.d_rows : (rows_dev ? rows : sl.d_rows);
  CU(e, cudaMemsetAsync(sl.d_status, 0, sizeof(int), st));
  CU(e, cudaEventRecord(sl.ev0, st));
  uint8_t* bases = out_dev ? bases_out : sl.d_bases.p;
  uint8_t* quals = out_dev ? quals_out : sl.d_quals.p;
  float* probs = probs_out ? (out_dev ? probs_out : sl.d_probs.p) : nullptr;
  float* logits = logits_out ? (out_dev ? logits_out : sl.d_logits.p) : nullptr;
  const int chunk_windows = f32 ? e->strict.chunk_windows : e->chunk_windows;
  for (int w0 = 0; w0 < batch; w0 += chunk_windows) {
    const int bw = std::min(chunk_windows, batch - w0);
    const HeadParams hp = chunk_head(e, bases, quals, probs, logits, w0);
    const float* rows_chunk = rows_base + (size_t)w0 * R * L;
    if (f32) strict_forward_chunk(e, rec, rows_chunk, bw, hp, sl.d_status, strict ? kStrictGemm : kTf32x3Gemm);
    else if (packed_base) bf16_forward_chunk(e, rec, nullptr, packed_base + (size_t)w0 * e->pl.stride, bw, hp, sl.d_status);
    else bf16_forward_chunk(e, rec, rows_chunk, nullptr, bw, hp, sl.d_status);
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
  sl.launches = rec.count;
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
  // the format keeps pw / ip and the ccs_bq id (at most CCS_BQ_MAX - 1) in one byte each and strand in 2 bits
  if (c.pw_max > 255 || c.ip_max > 255 || c.strand_max > 3 || c.ccs_bq_max > 256)
    return fail(e, DCB_ERR_INVALID, "packed rows need PW_MAX, IP_MAX <= 255, STRAND_MAX <= 3 and CCS_BQ_MAX <= 256");
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
  for (size_t i = 0; i < sl.prof_used; ++i) {
    const ProfRegion& r = sl.prof[i];
    float ms = 0.f;
    CU(e, cudaEventElapsedTime(&ms, r.start, r.end));
    e->prof_ms[r.kind] += ms;
    ++e->prof_n[r.kind];
  }
  sl.prof_used = 0;
  if (status & kStatusTileWait)
    return fail(e, DCB_ERR_CUDA, "a launch of the forward waited over a second for a tile of the launch before it; "
                                 "the outputs are not valid");
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
  e->prof_ffn_tokens = 0;
  for (auto& sl : e->slots) sl.prof_used = 0;
  for (int i = 0; i < kProfKinds; ++i) { e->prof_ms[i] = 0.f; e->prof_n[i] = 0; }
  return DCB_OK;
}

int dcb_get_profile(dcb_engine* e, float* ffn_ms_total, int32_t* ffn_launches, int64_t* ffn_tokens) {
  if (!e || !ffn_ms_total || !ffn_launches || !ffn_tokens) return DCB_ERR_INVALID;
  *ffn_ms_total = e->prof_ms[kProfFfn];
  *ffn_launches = e->prof_n[kProfFfn];
  *ffn_tokens = e->prof_ffn_tokens;
  return DCB_OK;
}

int dcb_get_profile_kernels(dcb_engine* e, float* ms6, int32_t* n6) {
  if (!e || !ms6 || !n6) return DCB_ERR_INVALID;
  for (int i = 0; i < kProfKinds; ++i) { ms6[i] = e->prof_ms[i]; n6[i] = e->prof_n[i]; }
  return DCB_OK;
}

int dcb_debug_residual(dcb_engine* e, int32_t stage, float* out, int64_t out_elems) {
  if (!e || !out) return DCB_ERR_INVALID;
  if (!e->debug || !e->d_dbg) return fail(e, DCB_ERR_STATE, "debug capture not enabled");
  const int stages = 1 + 2 * e->cfg.num_hidden_layers;
  if (stage < 0 || stage >= stages) return fail(e, DCB_ERR_INVALID, "stage %d outside [0,%d)", stage, stages);
  return read_capture<4>(e, e->d_dbg + (size_t)stage * e->chunk_tiles * x_image_elems(), kDP, kD, out, out_elems);
}

int dcb_debug_operand(dcb_engine* e, int32_t stage, int32_t which, uint16_t* out, int64_t out_elems) {
  if (!e || !out) return DCB_ERR_INVALID;
  if (!e->debug || !e->d_dbg_op) return fail(e, DCB_ERR_STATE, "debug capture not enabled");
  size_t cols = 0;
  int w = 0;
  if (!dbg_operand_slot(e, stage, which, &cols, &w))
    return fail(e, DCB_ERR_INVALID, "operand %d is not captured at stage %d", which, stage);
  const __nv_bfloat16* img = e->d_dbg_op + cols * e->chunk_tiles * kTileM;
  return read_capture<8>(e, reinterpret_cast<const uint16_t*>(img), w, w, out, out_elems);
}

int dcb_debug_f32(dcb_engine* e, int32_t stage, int32_t which, float* out, int64_t out_elems) {
  if (!e || !out) return DCB_ERR_INVALID;
  const dcb_engine::Strict& S = e->strict;
  if (!e->debug) return fail(e, DCB_ERR_STATE, "debug capture not enabled");
  if (!S.dbg || S.dbg_tokens < 0) return fail(e, DCB_ERR_STATE, "no float32 forward since debug capture was enabled");
  size_t cols = 0;
  int w = 0;
  if (!f32_image_slot(e, stage, which, &cols, &w))
    return fail(e, DCB_ERR_INVALID, "float32 image %d is not captured at stage %d", which, stage);
  const size_t n = (size_t)S.dbg_tokens * w;
  if (out_elems < (int64_t)n) return fail(e, DCB_ERR_INVALID, "output too small: need %lld", (long long)n);
  CU(e, cudaSetDevice(e->cfg.device));
  CU(e, cudaStreamSynchronize(e->stream));
  CU(e, cudaMemcpy(out, S.dbg + cols * S.chunk_windows * e->L, n * sizeof(float), cudaMemcpyDeviceToHost));
  return DCB_OK;
}

// read z is the windows [zmw_start[z], zmw_start[z + 1]) of n_windows
static int check_zmw_start(dcb_engine* e, const int32_t* zmw_start, int n_zmw, int n_windows) {
  if (zmw_start[0] < 0 || zmw_start[n_zmw] > n_windows) return fail(e, DCB_ERR_INVALID, "dcb_stitch: zmw_start outside [0, n_windows]");
  for (int z = 0; z < n_zmw; ++z)
    if (zmw_start[z + 1] < zmw_start[z]) return fail(e, DCB_ERR_INVALID, "dcb_stitch: zmw_start must be non-decreasing");
  return DCB_OK;
}

// window offsets [n + 1] of a ragged call: 0 first, non-decreasing
static int check_offsets(dcb_engine* e, const char* fn, const int64_t* off, int n) {
  if (!off) return fail(e, DCB_ERR_INVALID, "%s: null window offsets", fn);
  if (off[0] != 0) return fail(e, DCB_ERR_INVALID, "%s: window offsets must start at 0", fn);
  for (int w = 0; w < n; ++w)
    if (off[w + 1] < off[w]) return fail(e, DCB_ERR_INVALID, "%s: window offsets must be non-decreasing", fn);
  return DCB_OK;
}

// win_off (host, nullable): window w starts at win_off[w]; NULL: every window is L wide
static int stitch_impl(dcb_engine* e, const uint8_t* bases, const uint8_t* quals, const int64_t* win_off, int32_t n_windows,
                       int32_t L, const int32_t* zmw_start, int32_t n_zmw, uint32_t flags, uint8_t* seq_out, uint8_t* qual_out,
                       int32_t* len_out) {
  if (n_zmw == 0 || n_windows == 0) return DCB_OK;
  if (!bases || !quals || !zmw_start || !seq_out || !qual_out || !len_out) return fail(e, DCB_ERR_INVALID, "dcb_stitch: null pointer");
  int rc = check_zmw_start(e, zmw_start, n_zmw, n_windows);
  if (rc) return rc;
  CU(e, cudaSetDevice(e->cfg.device));
  const size_t nbytes = (size_t)window_offset(win_off, n_windows, L);
  const bool in_dev = flags & DCB_ROWS_ON_DEVICE, out_dev = flags & DCB_OUT_ON_DEVICE;
  const uint8_t *db, *dq;
  const int32_t* d_start;
  const int64_t* d_off = nullptr;
  Output<uint8_t> seq, qual;
  Output<int32_t> len;
  if ((rc = stage_in(e, e->st.bases, bases, nbytes, in_dev, &db)) || (rc = stage_in(e, e->st.quals, quals, nbytes, in_dev, &dq)) ||
      (rc = stage_in(e, e->st.start, zmw_start, (size_t)n_zmw + 1, false, &d_start)) ||
      (win_off && (rc = stage_in(e, e->st.win_off, win_off, (size_t)n_windows + 1, false, &d_off))) ||
      (rc = stage_out(e, e->st.seq, seq_out, nbytes, out_dev, &seq)) ||
      (rc = stage_out(e, e->st.qual, qual_out, nbytes, out_dev, &qual)) ||
      (rc = stage_out(e, e->st.len, len_out, (size_t)n_zmw, out_dev, &len)))
    return rc;
  launch_stitch(db, dq, L, d_off, d_start, n_zmw, seq.d, qual.d, len.d, e->stream);
  if ((rc = copy_out(e, seq)) || (rc = copy_out(e, qual)) || (rc = copy_out(e, len))) return rc;
  CU(e, cudaStreamSynchronize(e->stream));
  CU(e, cudaGetLastError());
  return DCB_OK;
}

int dcb_stitch(dcb_engine* e, const uint8_t* bases, const uint8_t* quals, int32_t n_windows, int32_t L,
               const int32_t* zmw_start, int32_t n_zmw, uint32_t flags,
               uint8_t* seq_out, uint8_t* qual_out, int32_t* len_out) {
  if (!e) return DCB_ERR_INVALID;
  if (n_windows < 0 || L <= 0 || n_zmw < 0) return fail(e, DCB_ERR_INVALID, "dcb_stitch: negative size");
  return stitch_impl(e, bases, quals, nullptr, n_windows, L, zmw_start, n_zmw, flags, seq_out, qual_out, len_out);
}

int dcb_stitch_ragged(dcb_engine* e, const uint8_t* bases, const uint8_t* quals, const int64_t* win_off, int32_t n_windows,
                      const int32_t* zmw_start, int32_t n_zmw, uint32_t flags, uint8_t* seq_out, uint8_t* qual_out,
                      int32_t* len_out) {
  if (!e) return DCB_ERR_INVALID;
  if (n_windows < 0 || n_zmw < 0) return fail(e, DCB_ERR_INVALID, "dcb_stitch_ragged: negative size");
  int rc = check_offsets(e, "dcb_stitch_ragged", win_off, n_windows);
  if (rc) return rc;
  return stitch_impl(e, bases, quals, win_off, n_windows, 1, zmw_start, n_zmw, flags, seq_out, qual_out, len_out);
}

static int stitch_fastq_impl(dcb_engine* e, const uint8_t* bases, const uint8_t* quals, const int64_t* win_off,
                             int32_t n_windows, int32_t L, const int32_t* zmw_start, int32_t n_zmw, const int32_t* window_pos,
                             const uint8_t* names, const int32_t* name_off, double min_quality, int32_t min_length,
                             uint32_t flags, uint8_t* fastq_out, int64_t fastq_cap, int64_t* rec_off, int32_t* outcome,
                             double* avg_q) {
  if (!rec_off) return fail(e, DCB_ERR_INVALID, "dcb_stitch_fastq: null pointer");
  if (n_zmw == 0) { rec_off[0] = 0; return DCB_OK; }
  if (!bases || !quals || !zmw_start || !window_pos || !names || !name_off || !fastq_out || !outcome || !avg_q)
    return fail(e, DCB_ERR_INVALID, "dcb_stitch_fastq: null pointer");
  if (name_off[0] != 0) return fail(e, DCB_ERR_INVALID, "dcb_stitch_fastq: name_off[0] must be 0");
  for (int z = 0; z < n_zmw; ++z)
    if (name_off[z + 1] < name_off[z]) return fail(e, DCB_ERR_INVALID, "dcb_stitch_fastq: name_off must be non-decreasing");
  int rc = check_zmw_start(e, zmw_start, n_zmw, n_windows);
  if (rc) return rc;
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  const size_t nbytes = (size_t)window_offset(win_off, n_windows, L), nz = n_zmw;
  const bool in_dev = flags & DCB_ROWS_ON_DEVICE;
  const uint8_t *db, *dq, *d_names;
  const int32_t *d_start, *d_pos, *d_name_off;
  const int64_t* d_off = nullptr;
  Output<int64_t> rec;
  Output<int32_t> out;
  Output<double> avg;
  if ((rc = stage_in(e, e->st.bases, bases, nbytes, in_dev, &db)) || (rc = stage_in(e, e->st.quals, quals, nbytes, in_dev, &dq)) ||
      (rc = stage_in(e, e->st.start, zmw_start, nz + 1, false, &d_start)) ||
      (win_off && (rc = stage_in(e, e->st.win_off, win_off, (size_t)n_windows + 1, false, &d_off))) ||
      (rc = stage_in(e, e->st.pos, window_pos, (size_t)n_windows, false, &d_pos)) ||
      (rc = stage_in(e, e->st.names, names, (size_t)name_off[n_zmw], false, &d_names)) ||
      (rc = stage_in(e, e->st.name_off, name_off, nz + 1, false, &d_name_off)) ||
      (rc = ensure(e, e->st.seq, nbytes)) || (rc = ensure(e, e->st.qual, nbytes)) || (rc = ensure(e, e->st.len, nz)) ||
      (rc = ensure(e, e->st.fastq, (size_t)fastq_cap)) || (rc = stage_out(e, e->st.rec_off, rec_off, nz + 1, false, &rec)) ||
      (rc = stage_out(e, e->st.outcome, outcome, nz, false, &out)) || (rc = stage_out(e, e->st.avg_q, avg_q, nz, false, &avg)))
    return rc;
  // concatenation + gap compaction (with no windows, every read is empty), then the filters and the records
  launch_stitch(db, dq, L, d_off, d_start, n_zmw, e->st.seq, e->st.qual, e->st.len, st);
  launch_read_outcome(e->st.qual, e->st.len, d_off, d_start, d_pos, L, n_zmw, e->d_p10, min_quality, min_length, out.d, avg.d, st);
  launch_fastq(e->st.seq, e->st.qual, e->st.len, d_off, d_start, L, n_zmw, out.d, d_names, d_name_off, rec.d, e->st.fastq,
               fastq_cap, st);
  if ((rc = copy_out(e, rec)) || (rc = copy_out(e, out)) || (rc = copy_out(e, avg))) return rc;
  CU(e, cudaStreamSynchronize(st));
  if (rec_off[n_zmw] > fastq_cap) return fail(e, DCB_ERR_INVALID, "dcb_stitch_fastq: fastq_out too small: need %lld bytes", (long long)rec_off[n_zmw]);
  if (rec_off[n_zmw] > 0) CU(e, cudaMemcpy(fastq_out, e->st.fastq, (size_t)rec_off[n_zmw], cudaMemcpyDeviceToHost));
  CU(e, cudaGetLastError());
  return DCB_OK;
}

int dcb_stitch_fastq(dcb_engine* e, const uint8_t* bases, const uint8_t* quals, int32_t n_windows, int32_t L,
                     const int32_t* zmw_start, int32_t n_zmw, const int32_t* window_pos, const uint8_t* names,
                     const int32_t* name_off, double min_quality, int32_t min_length, uint32_t flags, uint8_t* fastq_out,
                     int64_t fastq_cap, int64_t* rec_off, int32_t* outcome, double* avg_q) {
  if (!e) return DCB_ERR_INVALID;
  if (n_windows < 0 || L <= 0 || n_zmw < 0 || fastq_cap < 0) return fail(e, DCB_ERR_INVALID, "dcb_stitch_fastq: negative size");
  return stitch_fastq_impl(e, bases, quals, nullptr, n_windows, L, zmw_start, n_zmw, window_pos, names, name_off, min_quality,
                           min_length, flags, fastq_out, fastq_cap, rec_off, outcome, avg_q);
}

int dcb_stitch_fastq_ragged(dcb_engine* e, const uint8_t* bases, const uint8_t* quals, const int64_t* win_off,
                            int32_t n_windows, int32_t L, const int32_t* zmw_start, int32_t n_zmw, const int32_t* window_pos,
                            const uint8_t* names, const int32_t* name_off, double min_quality, int32_t min_length,
                            uint32_t flags, uint8_t* fastq_out, int64_t fastq_cap, int64_t* rec_off, int32_t* outcome,
                            double* avg_q) {
  if (!e) return DCB_ERR_INVALID;
  if (n_windows < 0 || L <= 0 || n_zmw < 0 || fastq_cap < 0) return fail(e, DCB_ERR_INVALID, "dcb_stitch_fastq_ragged: negative size");
  int rc = check_offsets(e, "dcb_stitch_fastq_ragged", win_off, n_windows);
  if (rc) return rc;
  return stitch_fastq_impl(e, bases, quals, win_off, n_windows, L, zmw_start, n_zmw, window_pos, names, name_off, min_quality,
                           min_length, flags, fastq_out, fastq_cap, rec_off, outcome, avg_q);
}

int dcb_skip_mask(dcb_engine* e, const int16_t* ccs_bq, int32_t n_windows, int32_t L, double skip_windows_above,
                  uint8_t* mask_out, double* avg_out) {
  if (!e) return DCB_ERR_INVALID;
  if (n_windows < 0 || L <= 0) return fail(e, DCB_ERR_INVALID, "dcb_skip_mask: negative size");
  if (n_windows == 0) return DCB_OK;
  if (!ccs_bq || !mask_out) return fail(e, DCB_ERR_INVALID, "dcb_skip_mask: null pointer");
  CU(e, cudaSetDevice(e->cfg.device));
  const int16_t* d_bq;
  Output<uint8_t> mask;
  Output<double> avg;
  int rc;
  if ((rc = stage_in(e, e->sk.bq, ccs_bq, (size_t)n_windows * L, false, &d_bq)) ||
      (rc = stage_out(e, e->sk.mask, mask_out, (size_t)n_windows, false, &mask)) ||
      (rc = stage_out(e, e->sk.avg, avg_out, (size_t)n_windows, false, &avg)))
    return rc;
  launch_skip_mask(d_bq, n_windows, L, e->d_p10, skip_windows_above, mask.d, avg.d, e->stream);
  if ((rc = copy_out(e, mask)) || (rc = copy_out(e, avg))) return rc;
  CU(e, cudaStreamSynchronize(e->stream));
  CU(e, cudaGetLastError());
  return DCB_OK;
}

// src_off (host, nullable): skipped window j is src_off[j] .. src_off[j + 1] of ccs_ids / ccs_bq, else j * L ..;
// dst_off (host, nullable, [n_dst + 1]): output window d starts at dst_off[d], else d * L
static int fill_skipped_impl(dcb_engine* e, const uint8_t* ccs_ids, const int16_t* ccs_bq, const int64_t* src_off,
                             const int32_t* dst_window, int32_t k, const int64_t* dst_off, int32_t n_dst, int32_t L,
                             int32_t calibration_enabled, double calibration_threshold, double calibration_w,
                             double calibration_b, uint32_t flags, uint8_t* bases, uint8_t* quals) {
  if (k == 0) return DCB_OK;
  if (!ccs_ids || !ccs_bq || !dst_window || !bases || !quals) return fail(e, DCB_ERR_INVALID, "dcb_fill_skipped: null pointer");
  for (int j = 0; j < k; ++j) {
    if (dst_window[j] < 0) return fail(e, DCB_ERR_INVALID, "dcb_fill_skipped: negative destination window");
    if (dst_off && dst_window[j] >= n_dst) return fail(e, DCB_ERR_INVALID, "dcb_fill_skipped: destination window outside [0, n_dst)");
    if (dst_off && dst_off[dst_window[j] + 1] - dst_off[dst_window[j]] != src_off[j + 1] - src_off[j])
      return fail(e, DCB_ERR_INVALID, "dcb_fill_skipped: skipped window %d and its destination differ in width", j);
  }
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  const size_t n = (size_t)window_offset(src_off, k, L);
  const bool out_dev = flags & DCB_OUT_ON_DEVICE;
  // host outputs: the kernel writes the windows back to back as they come in (destination j, offsets src_off), and
  // they are scattered into the caller's rows on the host below
  std::vector<int32_t> dst(dst_window, dst_window + k);
  std::vector<uint8_t> hb(out_dev ? 0 : n), hq(out_dev ? 0 : n);
  if (!out_dev) for (int j = 0; j < k; ++j) dst[j] = j;
  const int64_t* kernel_dst_off = out_dev ? dst_off : src_off;
  const uint8_t* d_ids;
  const int16_t* d_bq;
  const int32_t* d_dst;
  const int64_t *d_src_off = nullptr, *d_dst_off = nullptr;
  Output<uint8_t> ob, oq;
  Output<int> ostatus;
  int status = 0;
  int rc;
  if ((rc = stage_in(e, e->fs.ids, ccs_ids, n, false, &d_ids)) || (rc = stage_in(e, e->fs.bq, ccs_bq, n, false, &d_bq)) ||
      (rc = stage_in(e, e->fs.dst, dst.data(), (size_t)k, false, &d_dst)) ||
      (src_off && (rc = stage_in(e, e->fs.src_off, src_off, (size_t)k + 1, false, &d_src_off))) ||
      (kernel_dst_off && (rc = stage_in(e, e->fs.dst_off, kernel_dst_off, out_dev ? (size_t)n_dst + 1 : (size_t)k + 1, false,
                                        &d_dst_off))) ||
      (rc = stage_out(e, e->fs.status, &status, 1, false, &ostatus)) ||
      (rc = stage_out(e, e->fs.bases, out_dev ? bases : hb.data(), n, out_dev, &ob)) ||
      (rc = stage_out(e, e->fs.quals, out_dev ? quals : hq.data(), n, out_dev, &oq)))
    return rc;
  CU(e, cudaMemsetAsync(ostatus.d, 0, sizeof(int), st));
  launch_fill_skipped(d_ids, d_bq, d_src_off, d_dst, d_dst_off, k, L, (int64_t)n, calibration_enabled, calibration_threshold, calibration_w,
                      calibration_b, e->cfg.max_base_quality, ob.d, oq.d, ostatus.d, st);
  if ((rc = copy_out(e, ostatus)) || (rc = copy_out(e, ob)) || (rc = copy_out(e, oq))) return rc;
  CU(e, cudaStreamSynchronize(st));
  for (int j = 0; j < k && !out_dev; ++j) {
    const size_t s0 = (size_t)window_offset(src_off, j, L), w = (size_t)window_offset(src_off, j + 1, L) - s0;
    const size_t o = (size_t)window_offset(dst_off, dst_window[j], L);
    memcpy(bases + o, hb.data() + s0, w);
    memcpy(quals + o, hq.data() + s0, w);
  }
  CU(e, cudaGetLastError());
  if (status & 1) return fail(e, DCB_ERR_INPUT_RANGE, "dcb_fill_skipped: CCS base id outside 0..4 (clamped)");
  return DCB_OK;
}

int dcb_fill_skipped(dcb_engine* e, const uint8_t* ccs_ids, const int16_t* ccs_bq, const int32_t* dst_window, int32_t k,
                     int32_t L, int32_t calibration_enabled, double calibration_threshold, double calibration_w,
                     double calibration_b, uint32_t flags, uint8_t* bases, uint8_t* quals) {
  if (!e) return DCB_ERR_INVALID;
  if (k < 0 || L <= 0) return fail(e, DCB_ERR_INVALID, "dcb_fill_skipped: negative size");
  return fill_skipped_impl(e, ccs_ids, ccs_bq, nullptr, dst_window, k, nullptr, 0, L, calibration_enabled,
                           calibration_threshold, calibration_w, calibration_b, flags, bases, quals);
}

int dcb_fill_skipped_ragged(dcb_engine* e, const uint8_t* ccs_ids, const int16_t* ccs_bq, const int64_t* src_off,
                            const int32_t* dst_window, int32_t k, const int64_t* dst_off, int32_t n_dst,
                            int32_t calibration_enabled, double calibration_threshold, double calibration_w,
                            double calibration_b, uint32_t flags, uint8_t* bases, uint8_t* quals) {
  if (!e) return DCB_ERR_INVALID;
  if (k < 0 || n_dst < 0) return fail(e, DCB_ERR_INVALID, "dcb_fill_skipped_ragged: negative size");
  int rc;
  if ((rc = check_offsets(e, "dcb_fill_skipped_ragged", src_off, k)) || (rc = check_offsets(e, "dcb_fill_skipped_ragged", dst_off, n_dst)))
    return rc;
  return fill_skipped_impl(e, ccs_ids, ccs_bq, src_off, dst_window, k, dst_off, n_dst, 1, calibration_enabled,
                           calibration_threshold, calibration_w, calibration_b, flags, bases, quals);
}

int dcb_debug_head_epilogue(dcb_engine* e, const float* logits, int64_t n, uint8_t* bases, uint8_t* quals, float* probs) {
  if (!e || !logits || !bases || !quals) return DCB_ERR_INVALID;
  if (n < 0) return fail(e, DCB_ERR_INVALID, "dcb_debug_head_epilogue: negative token count");
  if (n == 0) return DCB_OK;
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  const int64_t chunk = std::min<int64_t>(n, 1 << 20);
  int rc = ensure(e, e->he.bias, 8);   // fc1 bias: zero
  if (rc) return rc;
  CU(e, cudaMemsetAsync(e->he.bias, 0, 8 * sizeof(float), st));
  HeadParams hp{};
  hp.bfc = e->he.bias;
  set_head_quality(hp, e->cfg);
  for (int64_t t0 = 0; t0 < n; t0 += chunk) {   // the first chunk is the largest: the buffers grow once
    const size_t m = (size_t)std::min<int64_t>(chunk, n - t0);
    const float* d_logits;
    Output<uint8_t> ob, oq;
    Output<float> op;
    if ((rc = stage_in(e, e->he.logits, logits + t0 * kVocab, m * kVocab, false, &d_logits)) ||
        (rc = stage_out(e, e->he.bases, bases + t0, m, false, &ob)) || (rc = stage_out(e, e->he.quals, quals + t0, m, false, &oq)) ||
        (rc = stage_out(e, e->he.probs, probs ? probs + t0 * kVocab : nullptr, m * kVocab, false, &op)))
      return rc;
    hp.bases = ob.d; hp.quals = oq.d; hp.probs = op.d;
    launch_head_epilogue(d_logits, (int)m, hp, st);
    if ((rc = copy_out(e, ob)) || (rc = copy_out(e, oq)) || (rc = copy_out(e, op))) return rc;
    CU(e, cudaStreamSynchronize(st));   // pageable host buffers: the next chunk reuses the staging
  }
  CU(e, cudaGetLastError());
  return DCB_OK;
}

// The argument checks of dcb_evaluate and dcb_alignment_loss_grad (`fn` names the call in the message).
static int check_alignment_args(dcb_engine* e, const char* fn, int32_t batch, int32_t L, double del_cost, int32_t band_width) {
  if (band_width >= 0)
    return fail(e, DCB_ERR_INVALID, "%s: the banded alignment loss (band_width=%d) is not supported; pass "
                "DCB_BAND_WIDTH_NONE (params.band_width None, as the released models are trained)", fn, band_width);
  if (batch < 0 || L <= 0 || L > 256)
    return fail(e, DCB_ERR_INVALID, "%s: need batch >= 0 and 0 < L <= 256 (batch=%d, L=%d)", fn, batch, L);
  if (!(del_cost == del_cost)) return fail(e, DCB_ERR_INVALID, "%s: del_cost is NaN", fn);
  return DCB_OK;
}

// Every label must be a base id 0..4.  Device labels are read back to the host first.
static int check_labels(dcb_engine* e, const char* fn, const uint8_t* labels, int32_t batch, int32_t L, bool on_device) {
  const size_t ntok = (size_t)batch * L;
  std::vector<uint8_t> copy;
  if (on_device) {
    copy.resize(ntok);
    CU(e, cudaMemcpyAsync(copy.data(), labels, ntok, cudaMemcpyDeviceToHost, e->stream));
    CU(e, cudaStreamSynchronize(e->stream));
    labels = copy.data();
  }
  for (size_t i = 0; i < ntok; ++i)
    if (labels[i] > 4) return fail(e, DCB_ERR_INVALID, "%s: label id %d outside 0..4 at window %zu", fn, labels[i], i / L);
  return DCB_OK;
}

int dcb_evaluate(dcb_engine* e, const float* probs, const uint8_t* labels, const uint8_t* ccs_ids, int32_t batch,
                 int32_t L, double del_cost, double loss_reg, int32_t band_width, uint32_t flags, float* loss_out,
                 uint8_t* exact_out, int32_t* pred_counts, int32_t* ccs_counts, float* ms_out) {
  if (!e) return DCB_ERR_INVALID;
  int rc = check_alignment_args(e, "dcb_evaluate", batch, L, del_cost, band_width);
  if (rc) return rc;
  if (ms_out) *ms_out = 0.f;
  if (batch == 0) return DCB_OK;
  if (!probs || !labels || !ccs_ids || !loss_out || !exact_out || !pred_counts || !ccs_counts)
    return fail(e, DCB_ERR_INVALID, "dcb_evaluate: null pointer");
  const size_t ntok = (size_t)batch * L;
  const bool lab_dev = flags & DCB_LABELS_ON_DEVICE;
  if (!lab_dev && (rc = check_labels(e, "dcb_evaluate", labels, batch, L, false))) return rc;
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  const float* d_probs;
  const uint8_t *d_labels, *d_ccs;
  Output<float> loss;
  Output<int32_t> pred, ccs;
  Output<uint8_t> exact;
  if ((rc = stage_in(e, e->ev.probs, probs, ntok * kVocab, flags & DCB_ROWS_ON_DEVICE, &d_probs)) ||
      (rc = stage_in(e, e->ev.labels, labels, ntok, lab_dev, &d_labels)) || (rc = stage_in(e, e->ev.ccs, ccs_ids, ntok, lab_dev, &d_ccs)) ||
      (lab_dev && ((rc = ensure(e, e->ev.labels, ntok)) || (rc = ensure(e, e->ev.bad, 1)))) ||
      (rc = stage_out(e, e->ev.loss, loss_out, (size_t)batch, false, &loss)) ||
      (rc = stage_out(e, e->ev.pred, pred_counts, (size_t)batch * 5, false, &pred)) ||
      (rc = stage_out(e, e->ev.ccs_counts, ccs_counts, (size_t)batch * 5, false, &ccs)) ||
      (rc = stage_out(e, e->ev.exact, exact_out, (size_t)batch, false, &exact)))
    return rc;
  int bad = 0;
  if (lab_dev) {
    // device labels are checked on the device: the kernels read a copy in which an id above 4 is 0, and the flag it
    // raises comes back with the results
    CU(e, cudaMemsetAsync(e->ev.bad.p, 0, sizeof(int), st));
    launch_copy_label_ids(labels, e->ev.labels.p, ntok, e->ev.bad.p, st);
    d_labels = e->ev.labels.p;
  }
  const bool hard = !(loss_reg > 0.0);
  CU(e, cudaEventRecord(e->ev_eval0, st));
  CU(e, launch_evaluate(d_probs, d_labels, d_ccs, batch, L, (float)del_cost, hard ? 1.f : (float)loss_reg, hard ? 1 : 0,
                        loss.d, exact.d, pred.d, ccs.d, st));
  CU(e, cudaEventRecord(e->ev_eval1, st));
  if ((rc = copy_out(e, loss)) || (rc = copy_out(e, pred)) || (rc = copy_out(e, ccs)) || (rc = copy_out(e, exact))) return rc;
  if (lab_dev) CU(e, cudaMemcpyAsync(&bad, e->ev.bad.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  CU(e, cudaStreamSynchronize(st));
  CU(e, cudaGetLastError());
  if (bad) return fail(e, DCB_ERR_INVALID, "dcb_evaluate: a device label id lies outside 0..4");
  if (ms_out) CU(e, cudaEventElapsedTime(ms_out, e->ev_eval0, e->ev_eval1));
  return DCB_OK;
}

int dcb_evaluate_calibration(dcb_engine* e, const float* probs, const uint8_t* labels, const uint8_t* ccs_ids,
                             const uint8_t* ccs_bq, int32_t batch, int32_t L, uint32_t flags, int64_t* counts_out,
                             int64_t* deletions_out, int32_t* pred_counts, int32_t* ccs_counts, float* ms_out) {
  if (!e) return DCB_ERR_INVALID;
  int rc = check_alignment_args(e, "dcb_evaluate_calibration", batch, L, 0.0, DCB_BAND_WIDTH_NONE);
  if (rc) return rc;
  if (ms_out) *ms_out = 0.f;
  if (!counts_out || !deletions_out) return fail(e, DCB_ERR_INVALID, "dcb_evaluate_calibration: null pointer");
  std::fill(counts_out, counts_out + 2 * DCB_CALIB_BINS * 2, (int64_t)0);
  deletions_out[0] = deletions_out[1] = 0;
  if (batch == 0) return DCB_OK;
  if (!probs || !labels || !ccs_ids || !ccs_bq || !pred_counts || !ccs_counts)
    return fail(e, DCB_ERR_INVALID, "dcb_evaluate_calibration: null pointer");
  const size_t ntok = (size_t)batch * L;
  const bool lab_dev = flags & DCB_LABELS_ON_DEVICE;
  if (!lab_dev && (rc = check_labels(e, "dcb_evaluate_calibration", labels, batch, L, false))) return rc;
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  const float* d_probs;
  const uint8_t *d_labels, *d_ccs, *d_bq;
  Output<int32_t> pred, ccs;
  constexpr size_t kCounts = 2 * DCB_CALIB_BINS * 2;   // then the two deletion totals
  if ((rc = stage_in(e, e->ev.probs, probs, ntok * kVocab, flags & DCB_ROWS_ON_DEVICE, &d_probs)) ||
      (rc = stage_in(e, e->ev.labels, labels, ntok, lab_dev, &d_labels)) || (rc = stage_in(e, e->ev.ccs, ccs_ids, ntok, lab_dev, &d_ccs)) ||
      (rc = stage_in(e, e->evc.bq, ccs_bq, ntok, lab_dev, &d_bq)) ||
      (lab_dev && ((rc = ensure(e, e->ev.labels, ntok)) || (rc = ensure(e, e->ev.bad, 1)))) ||
      (rc = ensure(e, e->ev.exact, (size_t)batch)) || (rc = ensure(e, e->evc.counts, kCounts + 2)) ||
      (rc = ensure(e, e->evc.bad_window, 1)) ||
      (rc = stage_out(e, e->ev.pred, pred_counts, (size_t)batch * 5, false, &pred)) ||
      (rc = stage_out(e, e->ev.ccs_counts, ccs_counts, (size_t)batch * 5, false, &ccs)))
    return rc;
  int bad = 0, bad_window = INT_MAX;
  if (lab_dev) {   // as dcb_evaluate: device labels are checked on the device
    CU(e, cudaMemsetAsync(e->ev.bad.p, 0, sizeof(int), st));
    launch_copy_label_ids(labels, e->ev.labels.p, ntok, e->ev.bad.p, st);
    d_labels = e->ev.labels.p;
  }
  CU(e, cudaMemsetAsync(e->evc.counts.p, 0, (kCounts + 2) * sizeof(unsigned long long), st));
  CU(e, cudaMemcpyAsync(e->evc.bad_window.p, &bad_window, sizeof(int), cudaMemcpyHostToDevice, st));
  static_assert(DCB_CALIB_BINS == kCalibBins, "one bin per quality 0..99");
  const EvalCalibOut calib{d_bq, e->evc.counts.p, e->evc.counts.p + kCounts, e->evc.bad_window.p};
  CU(e, cudaEventRecord(e->ev_eval0, st));
  CU(e, launch_evaluate_calibration(d_probs, d_labels, d_ccs, batch, L, e->ev.exact.p, pred.d, ccs.d, calib, st));
  CU(e, cudaEventRecord(e->ev_eval1, st));
  if ((rc = copy_out(e, pred)) || (rc = copy_out(e, ccs))) return rc;
  static_assert(sizeof(unsigned long long) == sizeof(int64_t), "int64 counts");
  CU(e, cudaMemcpyAsync(counts_out, e->evc.counts.p, kCounts * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  CU(e, cudaMemcpyAsync(deletions_out, e->evc.counts.p + kCounts, 2 * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  CU(e, cudaMemcpyAsync(&bad_window, e->evc.bad_window.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  if (lab_dev) CU(e, cudaMemcpyAsync(&bad, e->ev.bad.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  CU(e, cudaStreamSynchronize(st));
  CU(e, cudaGetLastError());
  if (bad) return fail(e, DCB_ERR_INVALID, "dcb_evaluate_calibration: a device label id lies outside 0..4");
  if (bad_window != INT_MAX)
    return fail(e, DCB_ERR_INVALID, "dcb_evaluate_calibration: window %d of the batch has a CCS base quality outside "
                "0..%d", bad_window, DCB_CALIB_BINS - 1);
  if (ms_out) CU(e, cudaEventElapsedTime(ms_out, e->ev_eval0, e->ev_eval1));
  return DCB_OK;
}

// The argument checks of dcb_distill_loss and dcb_distill_loss_grad (`fn` names the call in the message).
static int check_distill_args(dcb_engine* e, const char* fn, int32_t batch, int32_t L, double temperature, int32_t logit_loss) {
  if (batch < 0 || L <= 0 || L > 256)
    return fail(e, DCB_ERR_INVALID, "%s: need batch >= 0 and 0 < L <= 256 (batch=%d, L=%d)", fn, batch, L);
  const float t32 = (float)temperature;   // the logits are divided in float32, as tf divides a float32 tensor
  if (!std::isfinite(temperature) || !(temperature > 0.0) || !std::isfinite(t32) || !(t32 > 0.f))
    return fail(e, DCB_ERR_INVALID, "%s: temperature must be finite and > 0 in float32 (got %g)", fn, temperature);
  if (logit_loss != DCB_LOGIT_LOSS_MSE && logit_loss != DCB_LOGIT_LOSS_KL)
    return fail(e, DCB_ERR_INVALID, "%s: unknown logit loss id %d (DCB_LOGIT_LOSS_MSE = %d, DCB_LOGIT_LOSS_KL = %d)",
                fn, logit_loss, DCB_LOGIT_LOSS_MSE, DCB_LOGIT_LOSS_KL);
  return DCB_OK;
}

// dcb_distill_loss and dcb_distill_loss_grad: the loss, and its gradient when grad_out is not null (`fn` names the call
// in messages).
static int distill_impl(dcb_engine* e, const char* fn, const float* teacher_logits, const float* student_logits,
                        int32_t batch, int32_t L, double temperature, int32_t logit_loss, uint32_t flags, float* loss_out,
                        float* grad_out, float* ms_out) {
  if (!e) return DCB_ERR_INVALID;
  int rc = check_distill_args(e, fn, batch, L, temperature, logit_loss);
  if (rc) return rc;
  if (ms_out) *ms_out = 0.f;
  if (batch == 0) return DCB_OK;
  if (!teacher_logits || !student_logits || !loss_out) return fail(e, DCB_ERR_INVALID, "%s: null pointer", fn);
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  const size_t nlog = (size_t)batch * L * kVocab;
  const bool in_dev = flags & DCB_ROWS_ON_DEVICE, out_dev = flags & DCB_OUT_ON_DEVICE;
  const float *d_teacher, *d_student;
  Output<float> loss, grad;
  if ((rc = stage_in(e, e->ds.teacher, teacher_logits, nlog, in_dev, &d_teacher)) ||
      (rc = stage_in(e, e->ds.student, student_logits, nlog, in_dev, &d_student)) ||
      (rc = stage_out(e, e->ds.loss, loss_out, (size_t)batch, out_dev, &loss)) ||
      (rc = stage_out(e, e->ds.grad, grad_out, nlog, out_dev, &grad)))
    return rc;
  CU(e, cudaEventRecord(e->ev_eval0, st));
  CU(e, launch_distill_loss_grad(d_teacher, d_student, batch, L, (float)temperature, logit_loss, loss.d, grad.d, st));
  CU(e, cudaEventRecord(e->ev_eval1, st));
  if ((rc = copy_out(e, loss)) || (rc = copy_out(e, grad))) return rc;
  CU(e, cudaStreamSynchronize(st));
  CU(e, cudaGetLastError());
  if (ms_out) CU(e, cudaEventElapsedTime(ms_out, e->ev_eval0, e->ev_eval1));
  return DCB_OK;
}

int dcb_distill_loss(dcb_engine* e, const float* teacher_logits, const float* student_logits, int32_t batch,
                     int32_t L, double temperature, int32_t logit_loss, uint32_t flags, float* loss_out,
                     float* ms_out) {
  // loss_out is always a host array: DCB_OUT_ON_DEVICE does not apply here
  return distill_impl(e, "dcb_distill_loss", teacher_logits, student_logits, batch, L, temperature, logit_loss,
                      flags & ~DCB_OUT_ON_DEVICE, loss_out, nullptr, ms_out);
}

int dcb_distill_loss_grad(dcb_engine* e, const float* teacher_logits, const float* student_logits, int32_t batch,
                          int32_t L, double temperature, int32_t logit_loss, uint32_t flags, float* loss_out,
                          float* grad_out, float* ms_out) {
  return distill_impl(e, "dcb_distill_loss_grad", teacher_logits, student_logits, batch, L, temperature, logit_loss,
                      flags, loss_out, grad_out, ms_out);
}

int dcb_alignment_loss_grad(dcb_engine* e, const float* probs, const uint8_t* labels, int32_t batch, int32_t L,
                            double del_cost, double loss_reg, int32_t band_width, uint32_t flags, float* loss_out,
                            float* grad_out, float* matches_out, float* ms_out) {
  if (!e) return DCB_ERR_INVALID;
  int rc = check_alignment_args(e, "dcb_alignment_loss_grad", batch, L, del_cost, band_width);
  if (rc) return rc;
  if (ms_out) *ms_out = 0.f;
  if (batch == 0) return DCB_OK;
  if (!probs || !labels || !loss_out) return fail(e, DCB_ERR_INVALID, "dcb_alignment_loss_grad: null pointer");
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  const bool in_dev = flags & DCB_ROWS_ON_DEVICE, out_dev = flags & DCB_OUT_ON_DEVICE;
  const size_t ntok = (size_t)batch * L;
  if ((rc = check_labels(e, "dcb_alignment_loss_grad", labels, batch, L, in_dev))) return rc;
  int ctas = 0;
  CU(e, loss_grad_grid(batch, &ctas));
  const float* d_probs;
  const uint8_t* d_labels;
  Output<float> loss, grad, match;
  if ((rc = ensure(e, e->lg.dp, loss_grad_table_bytes(L, ctas) / sizeof(float))) ||
      (rc = stage_in(e, e->lg.probs, probs, ntok * kVocab, in_dev, &d_probs)) ||
      (rc = stage_in(e, e->lg.labels, labels, ntok, in_dev, &d_labels)) ||
      (rc = stage_out(e, e->lg.loss, loss_out, (size_t)batch, out_dev, &loss)) ||
      (rc = stage_out(e, e->lg.grad, grad_out, ntok * kVocab, out_dev, &grad)) ||
      (rc = stage_out(e, e->lg.matches, matches_out, ntok * L, out_dev, &match)))
    return rc;
  const bool hard = !(loss_reg > 0.0);
  CU(e, cudaEventRecord(e->ev_eval0, st));
  CU(e, launch_loss_grad(d_probs, d_labels, batch, L, (float)del_cost, hard ? 1.f : (float)loss_reg, hard ? 1 : 0,
                         e->lg.dp, ctas, loss.d, grad.d, match.d, st));
  CU(e, cudaEventRecord(e->ev_eval1, st));
  if ((rc = copy_out(e, loss)) || (rc = copy_out(e, grad)) || (rc = copy_out(e, match))) return rc;
  CU(e, cudaStreamSynchronize(st));
  CU(e, cudaGetLastError());
  if (ms_out) CU(e, cudaEventElapsedTime(ms_out, e->ev_eval0, e->ev_eval1));
  return DCB_OK;
}

// Spaced state one dcb_features_layout call may hold (bytes); a larger batch of ZMWs is split by the caller.
static constexpr int64_t kPrepScratchMax = 1ll << 31;

// wl_off / wl (host, nullable): CCS smart windows, ZMW z cut at wl[wl_off[z] .. wl_off[z + 1])
static int features_layout_impl(dcb_engine* e, const dcb_records* rec, const int32_t* wl_off, const int32_t* wl, int32_t ins_trim,
                                int32_t max_windows, int32_t* zmw_windows, int32_t* window_pos, uint8_t* overflow,
                                int32_t* window_width, int16_t* ccs_bq, int32_t* num_passes, uint8_t* ccs_ids,
                                int32_t* n_windows_out, float* ms_out) {
  auto& fp = e->fp;
  fp.n_windows = -1;
  if (!rec || !n_windows_out || rec->n_zmw < 0 || max_windows < 0) return fail(e, DCB_ERR_INVALID, "dcb_features_layout: bad argument");
  *n_windows_out = 0;
  if (ms_out) *ms_out = 0.f;
  const int nz = rec->n_zmw;
  if (nz == 0) { fp.n_windows = 0; return DCB_OK; }
  if (!rec->zmw_read_off || !rec->zmw_ccs_off || !rec->zmw_ccs_bq_any || !rec->read_meta || !rec->read_sn || !zmw_windows ||
      (max_windows && (!window_pos || !overflow || !ccs_bq || !num_passes || !ccs_ids)))
    return fail(e, DCB_ERR_INVALID, "dcb_features_layout: null pointer");
  if (e->pl.stride > 48 * 1024) return fail(e, DCB_ERR_INVALID, "dcb_features_layout: packed rows above 48 KB per window are not supported");
  // Size everything from the records' own numbers; the kernel checks what it derives from the cigars against these
  // bounds, so inconsistent records end in an error, never in a write outside the scratch.
  const int L = e->L, P = e->cfg.max_passes;
  const int n_reads = rec->zmw_read_off[nz], n_ccs = rec->zmw_ccs_off[nz];
  if (rec->zmw_read_off[0] != 0 || rec->zmw_ccs_off[0] != 0 || n_reads < 0 || n_ccs < 0 || rec->n_cigar < 0 || rec->n_query < 0)
    return fail(e, DCB_ERR_INVALID, "dcb_features_layout: bad offsets");
  if (wl_off && (wl_off[0] != 0 || !wl)) return fail(e, DCB_ERR_INVALID, "dcb_features_layout_smart: bad window length offsets");
  std::vector<PrepZmw> zmw(nz);
  int64_t gap_total = 0, plane_total = 0, win_total = 0;
  for (int z = 0; z < nz; ++z) {
    PrepZmw& zm = zmw[z];
    zm.read0 = rec->zmw_read_off[z];
    zm.n_reads = rec->zmw_read_off[z + 1] - zm.read0;
    zm.ccs_off = rec->zmw_ccs_off[z];
    zm.ccs_len = rec->zmw_ccs_off[z + 1] - zm.ccs_off;
    if (zm.read0 < 0 || zm.n_reads < 1 || zm.ccs_off < 0 || zm.ccs_len < 0 || zm.ccs_len > (1 << 24))
      return fail(e, DCB_ERR_INVALID, "dcb_features_layout: ZMW %d needs at least one subread and non-decreasing offsets", z);
    zm.keep = std::min(P, zm.n_reads);
    zm.bq_any = rec->zmw_ccs_bq_any[z] != 0;
    int64_t mb = zm.ccs_len, ins = 0;
    for (int r = zm.read0; r < zm.read0 + zm.n_reads; ++r) {
      const int32_t* m = rec->read_meta + (size_t)r * DCB_READ_META;
      if (m[0] < 0 || m[1] < 0 || (int64_t)m[0] + m[1] > rec->n_cigar || m[2] < 0 || m[3] < 0 || (int64_t)m[2] + m[3] > rec->n_query ||
          m[4] < 0 || m[4] > (1 << 24) || m[6] < 0 || m[7] < m[6] || m[7] > (1 << 24) || m[8] < 0 || m[8] > (1 << 24))
        return fail(e, DCB_ERR_INVALID, "dcb_features_layout: read %d of ZMW %d has offsets or lengths out of range", r - zm.read0, z);
      mb = std::max<int64_t>(mb, (int64_t)m[4] + (m[7] - m[6]));
      ins += m[8];
    }
    const int64_t wb = (mb + ins + 15) / 16 * 16 + 16;
    const int64_t bytes = wb * (3 * zm.keep + 3);
    if (plane_total + bytes > kPrepScratchMax)
      return fail(e, DCB_ERR_INVALID, "dcb_features_layout: the spaced reads of this batch need more than %lld bytes of scratch "
                  "(ZMW %d alone: %lld); pass fewer ZMWs per call", (long long)kPrepScratchMax, z, (long long)bytes);
    zm.mb = (int32_t)mb; zm.wb = (int32_t)wb;
    zm.gap_off = gap_total; gap_total += mb + 2;
    zm.plane_off = plane_total; plane_total += bytes;
    zm.win_off = (int32_t)win_total; zm.win_cap = (int32_t)std::min<int64_t>((wb + L - 1) / L, std::max(zm.ccs_len, 1));
    if (wl_off) {   // the reference fails on these (pre_lib.py:625-650): an AssertionError or an IndexError
      zm.wl_off = wl_off[z]; zm.wl_n = wl_off[z + 1] - wl_off[z];
      if (zm.wl_n < 0) return fail(e, DCB_ERR_INVALID, "dcb_features_layout_smart: window length offsets of ZMW %d decrease", z);
      int64_t sum = 0, nonzero = 0;
      for (int j = 0; j < zm.wl_n; ++j) {
        if (wl[zm.wl_off + j] < 0) return fail(e, DCB_ERR_INVALID, "dcb_features_layout_smart: negative window length in ZMW %d", z);
        sum += wl[zm.wl_off + j];
        nonzero += wl[zm.wl_off + j] > 0;
      }
      if (sum != zm.ccs_len)
        return fail(e, DCB_ERR_INVALID, "dcb_features_layout_smart: the window lengths of ZMW %d cover %lld CCS bases, its CCS read has %d",
                    z, (long long)sum, zm.ccs_len);
      zm.win_cap = (int32_t)nonzero;
    }
    win_total += zm.win_cap;
  }
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  PrepBatch& b = fp.batch;
  b = PrepBatch{};
  b.n_zmw = nz; b.ins_trim = ins_trim; b.pl = e->pl;
  int rc;
  if ((rc = stage_in(e, fp.zmw, (const PrepZmw*)zmw.data(), (size_t)nz, false, &b.zmw)) ||
      (rc = stage_in(e, fp.meta, rec->read_meta, (size_t)n_reads * DCB_READ_META, false, &b.read_meta)) ||
      (rc = stage_in(e, fp.sn, rec->read_sn, (size_t)n_reads * 4, false, &b.read_sn)) ||
      (rc = stage_in(e, fp.cigar, rec->cigar, (size_t)rec->n_cigar, false, &b.cigar)) ||
      (rc = stage_in(e, fp.bases, rec->bases, (size_t)rec->n_query, false, &b.bases)) ||
      (rc = stage_in(e, fp.pw, rec->pw, (size_t)rec->n_query, false, &b.pw)) ||
      (rc = stage_in(e, fp.ip, rec->ip, (size_t)rec->n_query, false, &b.ip)) ||
      (rc = stage_in(e, fp.ccs_bases, rec->ccs_bases, (size_t)n_ccs, false, &b.ccs_bases)) ||
      (rc = stage_in(e, fp.ccs_bq, rec->ccs_bq, (size_t)n_ccs, false, &b.ccs_bq)) ||
      (wl_off && (rc = stage_in(e, fp.wl, wl, (size_t)wl_off[nz], false, &b.wl))) ||
      (rc = ensure(e, fp.window_width, (size_t)win_total)) ||
      (rc = ensure(e, fp.op_scan, (size_t)rec->n_cigar + 1)) || (rc = ensure(e, fp.noni, (size_t)n_reads)) ||
      (rc = ensure(e, fp.gap, (size_t)gap_total)) || (rc = ensure(e, fp.spaced, (size_t)plane_total)) ||
      (rc = ensure(e, fp.win_list, (size_t)win_total)) || (rc = ensure(e, fp.zmw_out, (size_t)nz)) ||
      (rc = ensure(e, fp.status, 1)) || (rc = ensure(e, fp.zmw_windows, (size_t)nz)) ||
      (rc = ensure(e, fp.window, (size_t)win_total)) || (rc = ensure(e, fp.window_pos, (size_t)win_total)) ||
      (rc = ensure(e, fp.overflow, (size_t)win_total)) || (rc = ensure(e, fp.num_passes, (size_t)win_total)) ||
      (rc = ensure(e, fp.ccs_ids, (size_t)win_total * L)) || (rc = ensure(e, fp.out_bq, (size_t)win_total * L)))
    return rc;
  b.op_scan = fp.op_scan; b.read_noni_qs = fp.noni; b.gap = fp.gap; b.spaced = fp.spaced; b.win_list = fp.win_list;
  b.zmw_out = fp.zmw_out; b.status = fp.status;
  CU(e, cudaMemsetAsync(fp.status.p, 0, sizeof(int), st));
  CU(e, cudaMemsetAsync(fp.gap.p, 0, (size_t)gap_total * sizeof(int32_t), st));
  for (const PrepZmw& zm : zmw) {   // gaps: base 0, kinetics 0, CCS id 0, CCS quality -1
    CU(e, cudaMemsetAsync(fp.spaced.p + zm.plane_off, 0, (size_t)zm.wb * (3 * zm.keep + 1), st));
    CU(e, cudaMemsetAsync(fp.spaced.p + zm.plane_off + (size_t)zm.wb * (3 * zm.keep + 1), 0xff, (size_t)zm.wb * 2, st));
  }
  const PrepWindows out{fp.zmw_windows, fp.window, fp.window_pos, fp.overflow, fp.window_width, fp.num_passes, fp.ccs_ids, fp.out_bq};
  CU(e, cudaEventRecord(e->ev_eval0, st));
  launch_prep_layout(b, out, st);
  CU(e, cudaEventRecord(e->ev_eval1, st));
  int status = 0;
  CU(e, cudaMemcpyAsync(&status, fp.status.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  CU(e, cudaMemcpyAsync(zmw_windows, fp.zmw_windows.p, (size_t)nz * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CU(e, cudaStreamSynchronize(st));
  CU(e, cudaGetLastError());
  if (ms_out) CU(e, cudaEventElapsedTime(ms_out, e->ev_eval0, e->ev_eval1));
  if (status & 4) return fail(e, DCB_ERR_INVALID, "dcb_features_layout_smart: overflow window in a CCS read without base "
                               "qualities (not supported)");
  if (status) return fail(e, DCB_ERR_INVALID, "dcb_features_layout: a record's cigar disagrees with the columns, query bases or "
                          "insertion count its read_meta states");
  int64_t n = 0;
  for (int z = 0; z < nz; ++z) n += zmw_windows[z];
  *n_windows_out = (int32_t)n;
  if (n > max_windows) return fail(e, DCB_ERR_INVALID, "dcb_features_layout: %lld windows, max_windows is %d", (long long)n, max_windows);
  if (n) {
    CU(e, cudaMemcpyAsync(window_pos, fp.window_pos.p, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    CU(e, cudaMemcpyAsync(overflow, fp.overflow.p, (size_t)n, cudaMemcpyDeviceToHost, st));
    CU(e, cudaMemcpyAsync(num_passes, fp.num_passes.p, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    CU(e, cudaMemcpyAsync(ccs_ids, fp.ccs_ids.p, (size_t)n * L, cudaMemcpyDeviceToHost, st));
    CU(e, cudaMemcpyAsync(ccs_bq, fp.out_bq.p, (size_t)n * L * sizeof(int16_t), cudaMemcpyDeviceToHost, st));
    fp.width.resize(n);
    CU(e, cudaMemcpyAsync(fp.width.data(), fp.window_width.p, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    CU(e, cudaStreamSynchronize(st));
    if (window_width) memcpy(window_width, fp.width.data(), (size_t)n * sizeof(int32_t));
  }
  fp.n_windows = (int)n;
  return DCB_OK;
}

int dcb_features_layout(dcb_engine* e, const dcb_records* rec, int32_t ins_trim, int32_t max_windows, int32_t* zmw_windows,
                        int32_t* window_pos, uint8_t* overflow, int16_t* ccs_bq, int32_t* num_passes, uint8_t* ccs_ids,
                        int32_t* n_windows_out, float* ms_out) {
  if (!e) return DCB_ERR_INVALID;
  return features_layout_impl(e, rec, nullptr, nullptr, ins_trim, max_windows, zmw_windows, window_pos, overflow, nullptr, ccs_bq,
                              num_passes, ccs_ids, n_windows_out, ms_out);
}

int dcb_features_layout_smart(dcb_engine* e, const dcb_records* rec, const int32_t* wl_off, const int32_t* wl, int32_t ins_trim,
                              int32_t max_windows, int32_t* zmw_windows, int32_t* window_pos, uint8_t* overflow,
                              int32_t* window_width, int16_t* ccs_bq, int32_t* num_passes, uint8_t* ccs_ids,
                              int32_t* n_windows_out, float* ms_out) {
  if (!e) return DCB_ERR_INVALID;
  e->fp.n_windows = -1;
  if (!wl_off) return fail(e, DCB_ERR_INVALID, "dcb_features_layout_smart: null window lengths");
  if (max_windows && !window_width) return fail(e, DCB_ERR_INVALID, "dcb_features_layout_smart: null pointer");
  return features_layout_impl(e, rec, wl_off, wl, ins_trim, max_windows, zmw_windows, window_pos, overflow, window_width, ccs_bq,
                              num_passes, ccs_ids, n_windows_out, ms_out);
}

int dcb_features_pack(dcb_engine* e, const int32_t* windows, int32_t n, uint32_t flags, uint8_t* packed_out, float* ms_out) {
  if (!e) return DCB_ERR_INVALID;
  auto& fp = e->fp;
  if (ms_out) *ms_out = 0.f;
  if (n < 0) return fail(e, DCB_ERR_INVALID, "dcb_features_pack: negative size");
  if (fp.n_windows < 0) return fail(e, DCB_ERR_STATE, "dcb_features_pack before a successful dcb_features_layout");
  if (n == 0) return DCB_OK;
  if (!windows || !packed_out) return fail(e, DCB_ERR_INVALID, "dcb_features_pack: null pointer");
  const bool out_dev = flags & DCB_OUT_ON_DEVICE;
  if (out_dev && (reinterpret_cast<uintptr_t>(packed_out) & 15)) return fail(e, DCB_ERR_INVALID, "dcb_features_pack: device output must be 16-byte aligned");
  for (int i = 0; i < n; ++i)
    if (windows[i] < 0 || windows[i] >= fp.n_windows)
      return fail(e, DCB_ERR_INVALID, "dcb_features_pack: window %d outside the layout's %d windows", windows[i], fp.n_windows);
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  const int32_t* d_list;
  Output<uint8_t> packed;
  int rc;
  if ((rc = stage_in(e, fp.list, windows, (size_t)n, false, &d_list)) ||
      (rc = stage_out(e, fp.packed, packed_out, (size_t)n * e->pl.stride, out_dev, &packed)))
    return rc;
  CU(e, cudaEventRecord(e->ev_eval0, st));
  launch_prep_pack(fp.batch, fp.window, d_list, n, fp.n_windows, packed.d, st);
  CU(e, cudaEventRecord(e->ev_eval1, st));
  if ((rc = copy_out(e, packed))) return rc;
  CU(e, cudaStreamSynchronize(st));
  CU(e, cudaGetLastError());
  if (ms_out) CU(e, cudaEventElapsedTime(ms_out, e->ev_eval0, e->ev_eval1));
  return DCB_OK;
}

int dcb_features_ccs(dcb_engine* e, const int32_t* windows, int32_t n, const int64_t* off, uint8_t* ccs_ids, int16_t* ccs_bq,
                     float* ms_out) {
  if (!e) return DCB_ERR_INVALID;
  auto& fp = e->fp;
  if (ms_out) *ms_out = 0.f;
  if (n < 0) return fail(e, DCB_ERR_INVALID, "dcb_features_ccs: negative size");
  if (fp.n_windows < 0) return fail(e, DCB_ERR_STATE, "dcb_features_ccs before a successful dcb_features_layout");
  if (n == 0) return DCB_OK;
  if (!windows || !off || !ccs_ids || !ccs_bq) return fail(e, DCB_ERR_INVALID, "dcb_features_ccs: null pointer");
  if (off[0] != 0) return fail(e, DCB_ERR_INVALID, "dcb_features_ccs: off[0] must be 0");
  for (int i = 0; i < n; ++i) {
    if (windows[i] < 0 || windows[i] >= fp.n_windows)
      return fail(e, DCB_ERR_INVALID, "dcb_features_ccs: window %d outside the layout's %d windows", windows[i], fp.n_windows);
    if (off[i + 1] - off[i] != fp.width[windows[i]])
      return fail(e, DCB_ERR_INVALID, "dcb_features_ccs: entry %d: window %d is %d columns wide", i, windows[i], fp.width[windows[i]]);
  }
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  const size_t total = (size_t)off[n];
  const int32_t* d_list;
  const int64_t* d_off;
  Output<uint8_t> ids;
  Output<int16_t> bq;
  int rc;
  if ((rc = stage_in(e, fp.list, windows, (size_t)n, false, &d_list)) || (rc = stage_in(e, fp.ccs_off, off, (size_t)n + 1, false, &d_off)) ||
      (rc = stage_out(e, fp.ccs_ids_full, ccs_ids, total, false, &ids)) || (rc = stage_out(e, fp.ccs_bq_full, ccs_bq, total, false, &bq)))
    return rc;
  CU(e, cudaEventRecord(e->ev_eval0, st));
  launch_features_ccs(fp.batch, fp.window, d_list, n, d_off, ids.d, bq.d, st);
  CU(e, cudaEventRecord(e->ev_eval1, st));
  if ((rc = copy_out(e, ids)) || (rc = copy_out(e, bq))) return rc;
  CU(e, cudaStreamSynchronize(st));
  CU(e, cudaGetLastError());
  if (ms_out) CU(e, cudaEventElapsedTime(ms_out, e->ev_eval0, e->ev_eval1));
  return DCB_OK;
}

// The label batch of dcb_features_labels / dcb_features_eval: every offset and every operation is checked here, so the
// kernels index only inside the arrays they are given; the cigar ranges must follow one another (ZMW z's scan scratch
// is [offset + z, offset + z + count]), disjoint ranges keeping the CTAs' scratch apart.  `fn` names the call.
static int check_label_batch(dcb_engine* e, const char* fn, const dcb_labels* lab, int nz) {
  if (!lab->label_meta || (lab->n_cigar && !lab->cigar) || (lab->n_bases && !lab->bases) || lab->n_cigar < 0 || lab->n_bases < 0)
    return fail(e, DCB_ERR_INVALID, "%s: null pointer or negative size", fn);
  int64_t cig_end = 0;
  for (int z = 0; z < nz; ++z) {
    const int32_t* m = lab->label_meta + (size_t)z * DCB_LABEL_META;
    if (m[0] < cig_end || m[1] < 0 || (int64_t)m[0] + m[1] > lab->n_cigar || m[2] < 0 || m[3] < 0 ||
        (int64_t)m[2] + m[3] > lab->n_bases || m[4] < 0 || m[4] > (1 << 24) || m[5] < 0 || m[5] > (1 << 24))
      return fail(e, DCB_ERR_INVALID, "%s: label of ZMW %d has offsets or lengths out of range, or a cigar "
                  "range that overlaps or precedes the previous label's", fn, z);
    cig_end = (int64_t)m[0] + m[1];
    int64_t noni = m[4], ins = 0, nq = 0;
    for (int o = m[0]; o < m[0] + m[1]; ++o) {
      const uint32_t c = lab->cigar[o], op = c & 15, len = c >> 4;
      if (op != 0 && op != 1 && op != 2 && op != 7 && op != 8)
        return fail(e, DCB_ERR_INVALID, "%s: label of ZMW %d has cigar operation %u (only M, I, D, =, X)", fn, z, op);
      (op == 1 ? ins : noni) += len;
      if (op != 2) nq += len;
    }
    if (nq != m[3] || noni > (1 << 24) || ins > (1 << 24))
      return fail(e, DCB_ERR_INVALID, "%s: the cigar of ZMW %d's label covers %lld bases, it has %d", fn, z, (long long)nq, m[3]);
    for (int q = m[2]; q < m[2] + m[3]; ++q)
      if (lab->bases[q] < 1 || lab->bases[q] > 4)
        return fail(e, DCB_ERR_INVALID, "%s: label of ZMW %d has base id %d (only 1..4)", fn, z, lab->bases[q]);
  }
  return DCB_OK;
}

// Uploads a checked label batch and points lb at it (scan scratch included).
static int stage_labels(dcb_engine* e, const dcb_labels* lab, int nz, LabelBatch* lb) {
  auto& fp = e->fp;
  int rc;
  if ((rc = stage_in(e, fp.label_meta, lab->label_meta, (size_t)nz * DCB_LABEL_META, false, &lb->meta)) ||
      (rc = stage_in(e, fp.label_cigar, lab->cigar, (size_t)lab->n_cigar, false, &lb->cigar)) ||
      (rc = stage_in(e, fp.label_bases, lab->bases, (size_t)lab->n_bases, false, &lb->bases)) ||
      (rc = ensure(e, fp.label_scan, (size_t)lab->n_cigar + nz)))
    return rc;
  lb->scan = fp.label_scan;
  return DCB_OK;
}

int dcb_features_labels(dcb_engine* e, const dcb_labels* lab, const int32_t* windows, int32_t n, uint8_t* labels_out,
                        uint8_t* status_out, int32_t* ccs_width_out, float* ms_out) {
  if (!e) return DCB_ERR_INVALID;
  auto& fp = e->fp;
  if (ms_out) *ms_out = 0.f;
  if (n < 0 || !lab) return fail(e, DCB_ERR_INVALID, "dcb_features_labels: bad argument");
  if (fp.n_windows < 0) return fail(e, DCB_ERR_STATE, "dcb_features_labels before a successful dcb_features_layout");
  const int nz = fp.batch.n_zmw;
  if (lab->n_zmw != nz) return fail(e, DCB_ERR_INVALID, "dcb_features_labels: %d labels for a layout of %d ZMWs", lab->n_zmw, nz);
  if (ccs_width_out && nz) {
    std::vector<int4> zo(nz);
    CU(e, cudaMemcpyAsync(zo.data(), fp.zmw_out.p, (size_t)nz * sizeof(int4), cudaMemcpyDeviceToHost, e->stream));
    CU(e, cudaStreamSynchronize(e->stream));
    for (int z = 0; z < nz; ++z) ccs_width_out[z] = zo[z].y;
  }
  if (n == 0) return DCB_OK;
  if (!windows || !labels_out || !status_out || !lab->label_meta || (lab->n_cigar && !lab->cigar) || (lab->n_bases && !lab->bases) ||
      lab->n_cigar < 0 || lab->n_bases < 0)
    return fail(e, DCB_ERR_INVALID, "dcb_features_labels: null pointer or negative size");
  for (int i = 0; i < n; ++i)
    if (windows[i] < 0 || windows[i] >= fp.n_windows)
      return fail(e, DCB_ERR_INVALID, "dcb_features_labels: window %d outside the layout's %d windows", windows[i], fp.n_windows);
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  const int L = e->L;
  const int32_t* d_list;
  LabelBatch lb{};
  Output<uint8_t> rows, status;
  int rc;
  if ((rc = check_label_batch(e, "dcb_features_labels", lab, nz)) || (rc = stage_labels(e, lab, nz, &lb))) return rc;
  if ((rc = stage_in(e, fp.list, windows, (size_t)n, false, &d_list)) ||
      (rc = stage_out(e, fp.labels, labels_out, (size_t)n * L, false, &rows)) ||
      (rc = stage_out(e, fp.label_status, status_out, (size_t)n, false, &status)))
    return rc;
  CU(e, cudaEventRecord(e->ev_eval0, st));
  launch_labels(fp.batch, lb, fp.window, d_list, n, rows.d, status.d, st);
  CU(e, cudaEventRecord(e->ev_eval1, st));
  if ((rc = copy_out(e, rows)) || (rc = copy_out(e, status))) return rc;
  CU(e, cudaStreamSynchronize(st));
  CU(e, cudaGetLastError());
  if (ms_out) CU(e, cudaEventElapsedTime(ms_out, e->ev_eval0, e->ev_eval1));
  return DCB_OK;
}

int dcb_features_eval(dcb_engine* e, const dcb_labels* lab, const uint8_t* keep_zmw, int32_t n_keep, int32_t capacity,
                      uint8_t* packed_out, uint8_t* labels_out, uint8_t* ccs_out, uint8_t* status_out, int32_t* ccs_width_out,
                      int32_t* windows_out, int32_t* k_out, float* ms_out) {
  if (!e) return DCB_ERR_INVALID;
  auto& fp = e->fp;
  if (ms_out) *ms_out = 0.f;
  if (!lab || !k_out || capacity < 0) return fail(e, DCB_ERR_INVALID, "dcb_features_eval: bad argument");
  *k_out = 0;
  if (fp.n_windows < 0) return fail(e, DCB_ERR_STATE, "dcb_features_eval before a successful dcb_features_layout");
  const int nz = fp.batch.n_zmw, n = fp.n_windows;
  if (lab->n_zmw != nz) return fail(e, DCB_ERR_INVALID, "dcb_features_eval: %d labels for a layout of %d ZMWs", lab->n_zmw, nz);
  if (n_keep != nz || (nz && !keep_zmw))
    return fail(e, DCB_ERR_INVALID, "dcb_features_eval: a keep mask of %d entries for a layout of %d ZMWs", n_keep, nz);
  if (capacity && (!packed_out || !labels_out || !ccs_out)) return fail(e, DCB_ERR_INVALID, "dcb_features_eval: null pointer");
  if (reinterpret_cast<uintptr_t>(packed_out) & 15) return fail(e, DCB_ERR_INVALID, "dcb_features_eval: packed_out must be 16-byte aligned");
  int rc;
  if ((rc = check_label_batch(e, "dcb_features_eval", lab, nz))) return rc;
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  if (ccs_width_out && nz) {
    std::vector<int4> zo(nz);
    CU(e, cudaMemcpyAsync(zo.data(), fp.zmw_out.p, (size_t)nz * sizeof(int4), cudaMemcpyDeviceToHost, st));
    CU(e, cudaStreamSynchronize(st));
    for (int z = 0; z < nz; ++z) ccs_width_out[z] = zo[z].y;
  }
  if (n == 0) return DCB_OK;
  const int L = e->L;
  LabelBatch lb{};
  const uint8_t* d_keep;
  if ((rc = stage_labels(e, lab, nz, &lb)) || (rc = stage_in(e, fp.keep, keep_zmw, (size_t)nz, false, &d_keep)) ||
      (rc = ensure(e, fp.labels, (size_t)n * L)) || (rc = ensure(e, fp.label_status, (size_t)n)) ||
      (rc = ensure(e, fp.eval_dst, (size_t)n)) || (rc = ensure(e, fp.list, (size_t)n)) || (rc = ensure(e, fp.eval_count, 1)))
    return rc;
  CU(e, cudaEventRecord(e->ev_eval0, st));
  launch_features_eval(fp.batch, lb, fp.window, n, fp.ccs_ids, d_keep, capacity, fp.labels, fp.label_status, fp.eval_dst, fp.list,
                       fp.eval_count, packed_out, labels_out, ccs_out, st);
  CU(e, cudaEventRecord(e->ev_eval1, st));
  int k = 0;
  CU(e, cudaMemcpyAsync(&k, fp.eval_count.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  if (status_out) CU(e, cudaMemcpyAsync(status_out, fp.label_status.p, (size_t)n, cudaMemcpyDeviceToHost, st));
  CU(e, cudaStreamSynchronize(st));
  CU(e, cudaGetLastError());
  *k_out = k;
  if (k > capacity) return fail(e, DCB_ERR_INVALID, "dcb_features_eval: %d windows are kept, the capacity is %d", k, capacity);
  if (windows_out && k) {
    CU(e, cudaMemcpyAsync(windows_out, fp.list.p, (size_t)k * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    CU(e, cudaStreamSynchronize(st));
  }
  if (ms_out) CU(e, cudaEventElapsedTime(ms_out, e->ev_eval0, e->ev_eval1));
  return DCB_OK;
}

// Read r of a batch from dcb_calib_get_batch as the kernels that walk it may trust it: offsets inside the arrays, its
// cigar's query length equal to its base count, and endpos equal to bam_endpos (pos plus the reference length, or
// pos + 1).
static int check_aligned_read(dcb_engine* e, const char* who, int32_t r, const int32_t* read_meta, const uint32_t* cigar,
                              int64_t n_cigar, int64_t n_bases) {
  const int32_t* m = read_meta + (size_t)r * DCB_CALIB_META;
  if (m[0] < 0 || m[2] < 0 || m[3] < 0 || m[4] < 0 || m[5] < 0 || (int64_t)m[2] + m[3] > n_cigar ||
      (int64_t)m[4] + m[5] > n_bases)
    return fail(e, DCB_ERR_INVALID, "%s: read %d: offsets outside the batch", who, r);
  int64_t q = 0, rl = 0;
  for (int32_t k = 0; k < m[3]; ++k) {
    const uint32_t v = cigar[m[2] + k];
    const int op = v & 15;
    if (op == 0 || op == 1 || op == 4 || op == 7 || op == 8) q += v >> 4;
    if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) rl += v >> 4;
  }
  if (q != m[5]) return fail(e, DCB_ERR_INVALID, "%s: read %d: its cigar covers %lld bases, it has %d", who, r, (long long)q, m[5]);
  if ((int64_t)m[1] != m[0] + (rl ? rl : 1)) return fail(e, DCB_ERR_INVALID, "%s: read %d: endpos is not bam_endpos", who, r);
  return DCB_OK;
}

// The batch as dcb_calib_count's kernels may trust it: every read as check_aligned_read has it, and few enough bases
// per read for the kernel's 32-bit histogram.
static int check_calib_batch(dcb_engine* e, const dcb_calib_input* in) {
  if (in->n_reads < 0 || in->n_regions < 0 || in->n_cigar < 0 || in->n_bases < 0 || in->interval_length <= 0 ||
      in->ref_count < 0 || in->contig_length < 0 || in->n_bases > INT32_MAX || in->n_cigar > INT32_MAX)
    return fail(e, DCB_ERR_INVALID, "dcb_calib_count: bad sizes");
  if ((in->n_reads && (!in->read_meta || (in->n_cigar && !in->cigar) || (in->n_bases && (!in->seq || !in->qual)))) ||
      (in->n_regions && !in->regions))
    return fail(e, DCB_ERR_INVALID, "dcb_calib_count: null array");
  for (int32_t k = 0; k < in->n_regions; ++k)
    if (in->regions[2 * k] < 0 || in->regions[2 * k] > in->regions[2 * k + 1] || in->regions[2 * k + 1] > INT32_MAX)
      return fail(e, DCB_ERR_INVALID, "dcb_calib_count: region %d is not 0 <= start <= stop < 2^31", k);
  for (int32_t r = 0; r < in->n_reads; ++r) {
    int rc = check_aligned_read(e, "dcb_calib_count", r, in->read_meta, in->cigar, in->n_cigar, in->n_bases);
    if (rc) return rc;
    const int32_t nb = in->read_meta[(size_t)r * DCB_CALIB_META + 5];
    if ((int64_t)nb * 2 * in->n_regions >= (1ll << 32))   // the kernel's per-read 32-bit histogram
      return fail(e, DCB_ERR_INVALID, "dcb_calib_count: read %d: %d bases over %d regions could overflow a count", r, nb, in->n_regions);
  }
  return DCB_OK;
}

int dcb_calib_count(dcb_engine* e, const dcb_calib_input* in, int64_t* counts, int64_t* failure, float* ms_out) {
  if (!e) return DCB_ERR_INVALID;
  if (ms_out) *ms_out = 0.f;
  if (!in || !counts || !failure) return fail(e, DCB_ERR_INVALID, "dcb_calib_count: null argument");
  memset(counts, 0, 2 * kCalibBins * sizeof(int64_t));
  failure[0] = -1; failure[1] = failure[2] = 0;
  int rc;
  if ((rc = check_calib_batch(e, in))) return rc;
  auto& cb = e->cb;
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  if (in->ref_bases) {
    if ((rc = ensure(e, cb.ref, (size_t)std::max<int64_t>(in->ref_count, 1)))) return rc;
    cb.ref_count = -1;
    if (in->ref_count) CU(e, cudaMemcpyAsync(cb.ref.p, in->ref_bases, (size_t)in->ref_count, cudaMemcpyHostToDevice, st));
    cb.ref_start = in->ref_start;
    cb.ref_count = in->ref_count;
  } else if (cb.ref_count < 0 || cb.ref_start != in->ref_start || cb.ref_count != in->ref_count) {
    return fail(e, DCB_ERR_STATE, "dcb_calib_count: no reference bases for [%lld, +%lld) were given", (long long)in->ref_start,
                (long long)in->ref_count);
  }
  const int grid = std::min(in->n_reads, 1024);
  const int32_t* d_meta;
  const uint32_t* d_cigar;
  const uint8_t *d_seq, *d_qual;
  const int64_t* d_regions;
  if ((rc = stage_in(e, cb.meta, in->read_meta, (size_t)in->n_reads * DCB_CALIB_META, false, &d_meta)) ||
      (rc = stage_in(e, cb.cigar, in->cigar, (size_t)in->n_cigar, false, &d_cigar)) ||
      (rc = stage_in(e, cb.seq, in->seq, (size_t)in->n_bases, false, &d_seq)) ||
      (rc = stage_in(e, cb.qual, in->qual, (size_t)in->n_bases, false, &d_qual)) ||
      (rc = stage_in(e, cb.regions, in->regions, (size_t)in->n_regions * 2, false, &d_regions)) ||
      (rc = ensure(e, cb.partial, (size_t)std::max(grid, 1) * 2 * kCalibBins)) ||
      (rc = ensure(e, cb.partial_fail, (size_t)std::max(grid, 1) * 2)) || (rc = ensure(e, cb.out, 2 * kCalibBins + 3)))
    return rc;
  CalibBatch c{d_meta, d_cigar, d_seq, d_qual, in->n_reads, in->n_regions, d_regions, in->interval_length, cb.ref.p,
               in->ref_start, in->ref_count, in->contig_length, in->calibration_enabled ? 1 : 0, in->threshold, in->w, in->b};
  CU(e, cudaEventRecord(e->ev_eval0, st));
  launch_calib_count(c, grid, cb.partial.p, cb.partial_fail.p, cb.out.p, st);
  CU(e, cudaEventRecord(e->ev_eval1, st));
  long long out[2 * kCalibBins + 3];
  CU(e, cudaMemcpyAsync(out, cb.out.p, sizeof out, cudaMemcpyDeviceToHost, st));
  CU(e, cudaStreamSynchronize(st));
  CU(e, cudaGetLastError());
  for (int k = 0; k < 2 * kCalibBins; ++k) counts[k] = out[k];
  for (int k = 0; k < 3; ++k) failure[k] = out[2 * kCalibBins + k];
  if (ms_out) CU(e, cudaEventElapsedTime(ms_out, e->ev_eval0, e->ev_eval1));
  return DCB_OK;
}

static_assert(kIdentityCounts == DCB_IDENTITY_COUNTS && kIdentityOk == DCB_IDENTITY_OK &&
              kIdentityPastContig == DCB_IDENTITY_PAST_CONTIG && kIdentitySkipOp == DCB_IDENTITY_SKIP_OP &&
              kIdentityBorderline == DCB_IDENTITY_BORDERLINE && kIdentityBadInput == DCB_IDENTITY_BAD_INPUT,
              "the kernel writes the ABI's status codes");

// A dcb_identity_input as the identity and errors kernels may trust it: sizes, arrays, and every read as
// check_aligned_read has it.
static int check_identity_input(dcb_engine* e, const char* who, const dcb_identity_input* in) {
  if (in->n_reads < 0 || in->n_cigar < 0 || in->n_bases < 0 || in->ref_count < 0 || in->contig_length < 0 ||
      in->n_bases > INT32_MAX || in->n_cigar > INT32_MAX)
    return fail(e, DCB_ERR_INVALID, "%s: bad sizes", who);
  if ((in->n_reads && (!in->read_meta || (in->n_cigar && !in->cigar) || (in->n_bases && (!in->seq || !in->qual)))) ||
      (in->ref_count && !in->ref_bases))
    return fail(e, DCB_ERR_INVALID, "%s: null array", who);
  int rc;
  for (int32_t r = 0; r < in->n_reads; ++r)
    if ((rc = check_aligned_read(e, who, r, in->read_meta, in->cigar, in->n_cigar, in->n_bases))) return rc;
  return DCB_OK;
}

int dcb_read_identity(dcb_engine* e, const dcb_identity_input* in, int64_t* counts, double* avg_q, int32_t* status,
                      float* ms_out) {
  if (!e) return DCB_ERR_INVALID;
  if (ms_out) *ms_out = 0.f;
  if (!in || !counts || !avg_q || !status) return fail(e, DCB_ERR_INVALID, "dcb_read_identity: null argument");
  int rc;
  if ((rc = check_identity_input(e, "dcb_read_identity", in))) return rc;
  auto& ri = e->ri;
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  const int32_t* d_meta;
  const uint32_t* d_cigar;
  const uint8_t *d_seq, *d_qual, *d_ref;
  Output<long long> o_counts;
  Output<double> o_avg;
  Output<int32_t> o_status;
  const size_t n = (size_t)in->n_reads;
  if ((rc = stage_in(e, ri.meta, in->read_meta, n * DCB_CALIB_META, false, &d_meta)) ||
      (rc = stage_in(e, ri.cigar, in->cigar, (size_t)in->n_cigar, false, &d_cigar)) ||
      (rc = stage_in(e, ri.seq, in->seq, (size_t)in->n_bases, false, &d_seq)) ||
      (rc = stage_in(e, ri.qual, in->qual, (size_t)in->n_bases, false, &d_qual)) ||
      (rc = stage_in(e, ri.ref, in->ref_bases, (size_t)in->ref_count, false, &d_ref)) ||
      (rc = stage_out(e, ri.counts, reinterpret_cast<long long*>(counts), n * kIdentityCounts, false, &o_counts)) ||
      (rc = stage_out(e, ri.avg_q, avg_q, n, false, &o_avg)) || (rc = stage_out(e, ri.status, status, n, false, &o_status)))
    return rc;
  IdentityBatch c{d_meta, d_cigar, d_seq, d_qual, in->n_reads, d_ref, in->ref_start, in->ref_count, in->contig_length,
                  e->d_p10.p};
  CU(e, cudaEventRecord(e->ev_eval0, st));
  launch_read_identity(c, o_counts.d, o_avg.d, o_status.d, st);
  CU(e, cudaEventRecord(e->ev_eval1, st));
  if ((rc = copy_out(e, o_counts)) || (rc = copy_out(e, o_avg)) || (rc = copy_out(e, o_status))) return rc;
  CU(e, cudaStreamSynchronize(st));
  CU(e, cudaGetLastError());
  if (ms_out) CU(e, cudaEventElapsedTime(ms_out, e->ev_eval0, e->ev_eval1));
  return DCB_OK;
}

static_assert(kErrorBins == DCB_ERRORS_BINS && kErrorSub == DCB_ERRORS_SUB && kErrorInsEvents == DCB_ERRORS_INS_EVENTS &&
              kErrorInsBases == DCB_ERRORS_INS_BASES && kErrorDelEvents == DCB_ERRORS_DEL_EVENTS &&
              kErrorDelBases == DCB_ERRORS_DEL_BASES && kErrorRuns == DCB_ERRORS_RUNS &&
              kErrorMatrix == DCB_ERRORS_MATRIX && kErrorCols == DCB_ERRORS_COLS && kErrorMatrix + 25 == kErrorCols,
              "the kernel writes the ABI's error columns");

int dcb_read_errors(dcb_engine* e, const dcb_identity_input* in, int64_t* errors, float* ms_out) {
  if (!e) return DCB_ERR_INVALID;
  if (ms_out) *ms_out = 0.f;
  if (!in || !errors) return fail(e, DCB_ERR_INVALID, "dcb_read_errors: null argument");
  int rc;
  if ((rc = check_identity_input(e, "dcb_read_errors", in))) return rc;
  if (in->ref_start < 0 || in->ref_count > INT32_MAX || in->ref_start + in->ref_count > in->contig_length)
    return fail(e, DCB_ERR_INVALID, "dcb_read_errors: the slice [%lld, +%lld) is not inside the contig (length %lld)",
                (long long)in->ref_start, (long long)in->ref_count, (long long)in->contig_length);
  for (int32_t r = 0; r < in->n_reads; ++r) {   // the truth positions the kernel may read, whole runs aside
    const int32_t* m = in->read_meta + (size_t)r * DCB_CALIB_META;
    const int64_t lo = std::max<int64_t>(m[0] - 1, 0), hi = std::min<int64_t>((int64_t)m[1] + 1, in->contig_length);
    if (lo < hi && (lo < in->ref_start || hi > in->ref_start + in->ref_count))
      return fail(e, DCB_ERR_INVALID, "dcb_read_errors: read %d: the slice [%lld, +%lld) does not hold [%lld, %lld)", r,
                  (long long)in->ref_start, (long long)in->ref_count, (long long)lo, (long long)hi);
  }
  auto& re = e->re;
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  const int32_t* d_meta;
  const uint32_t* d_cigar;
  const uint8_t *d_seq, *d_qual, *d_ref;
  Output<long long> o_errors;
  const size_t n = (size_t)in->n_reads, n_ref = (size_t)in->ref_count;
  const size_t n_chunks = (size_t)std::max(run_bounds_chunks((int)in->ref_count), 1);
  if ((rc = stage_in(e, re.meta, in->read_meta, n * DCB_CALIB_META, false, &d_meta)) ||
      (rc = stage_in(e, re.cigar, in->cigar, (size_t)in->n_cigar, false, &d_cigar)) ||
      (rc = stage_in(e, re.seq, in->seq, (size_t)in->n_bases, false, &d_seq)) ||
      (rc = stage_in(e, re.qual, in->qual, (size_t)in->n_bases, false, &d_qual)) ||
      (rc = stage_in(e, re.ref, in->ref_bases, n_ref, false, &d_ref)) ||
      (rc = ensure(e, re.run_start, std::max<size_t>(n_ref, 1))) || (rc = ensure(e, re.run_end, std::max<size_t>(n_ref, 1))) ||
      (rc = ensure(e, re.chunk_start, n_chunks)) || (rc = ensure(e, re.chunk_end, n_chunks)) ||
      (rc = ensure(e, re.carry_start, n_chunks)) || (rc = ensure(e, re.carry_end, n_chunks)) ||
      (rc = stage_out(e, re.errors, reinterpret_cast<long long*>(errors), n * kErrorCols, false, &o_errors)))
    return rc;
  IdentityBatch c{d_meta, d_cigar, d_seq, d_qual, in->n_reads, d_ref, in->ref_start, in->ref_count, in->contig_length,
                  e->d_p10.p};
  CU(e, cudaEventRecord(e->ev_eval0, st));
  launch_run_bounds(d_ref, (int)in->ref_count, re.chunk_start.p, re.chunk_end.p, re.carry_start.p, re.carry_end.p,
                    re.run_start.p, re.run_end.p, st);
  launch_read_errors(c, re.run_start.p, re.run_end.p, o_errors.d, st);
  CU(e, cudaEventRecord(e->ev_eval1, st));
  if ((rc = copy_out(e, o_errors))) return rc;
  CU(e, cudaStreamSynchronize(st));
  CU(e, cudaGetLastError());
  if (ms_out) CU(e, cudaEventElapsedTime(ms_out, e->ev_eval0, e->ev_eval1));
  return DCB_OK;
}

static_assert(kKmerHist == DCB_KMER_HIST && kKmerStatSlots + 1 == DCB_KMER_STATS, "the ABI's k-mer table sizes");
static_assert(kSpecBins == DCB_KMER_SPECTRUM_BINS && DCB_KMER_SPECTRUM_STATS == 5, "the ABI's spectrum sizes");

namespace {

// The slots of a k-mer table in table_bytes (<= 0: half the device's free memory): the largest power of two, at
// least 64 and at most 2^32, of 12-byte slots that fits.
int kmer_capacity(dcb_engine* e, const char* who, int64_t table_bytes, unsigned long long* out) {
  if (table_bytes <= 0) {
    size_t free_b = 0, total_b = 0;
    CU(e, cudaMemGetInfo(&free_b, &total_b));
    table_bytes = (int64_t)(free_b / 2);
  }
  constexpr int64_t kSlotBytes = sizeof(unsigned long long) + sizeof(unsigned int);
  unsigned long long cap = 64;
  while (cap < (1ull << 32) && (int64_t)(2 * cap) * kSlotBytes <= table_bytes) cap *= 2;
  if ((int64_t)cap * kSlotBytes > table_bytes)
    return fail(e, DCB_ERR_INVALID, "%s: %lld bytes hold fewer than 64 slots", who, (long long)table_bytes);
  *out = cap;
  return DCB_OK;
}

}  // namespace

int dcb_kmer_table_init(dcb_engine* e, int64_t table_bytes, int32_t k, int64_t* capacity) {
  if (!e) return DCB_ERR_INVALID;
  if (k < 1 || k > 31) return fail(e, DCB_ERR_INVALID, "dcb_kmer_table_init: k must be between 1 and 31, got %d", k);
  auto& km = e->km;
  CU(e, cudaSetDevice(e->cfg.device));
  CU(e, cudaStreamSynchronize(e->stream));
  km.keys.reset(); km.counts.reset(); km.capacity = 0;
  unsigned long long cap;
  int rc = kmer_capacity(e, "dcb_kmer_table_init", table_bytes, &cap);
  if (rc) return rc;
  for (auto& sl : km.slot)
    for (cudaEvent_t* ev : {&sl.ev0, &sl.ev1})
      if (!*ev) CU(e, cudaEventCreate(ev));
  if ((rc = ensure(e, km.keys, cap)) || (rc = ensure(e, km.counts, cap)) || (rc = ensure(e, km.stats, kKmerStatSlots)) ||
      (rc = ensure(e, km.hist, kKmerHist + 1)) ||
      (rc = ensure(e, km.hist_partial, (size_t)kmer_hist_grid(cap) * (kKmerHist + 1))))
    return rc;
  km.capacity = cap;
  km.k = k;
  if (capacity) *capacity = (int64_t)cap;
  return dcb_kmer_table_clear(e, 0, 1);
}

int dcb_kmer_table_clear(dcb_engine* e, int32_t partition, int32_t n_partitions) {
  if (!e) return DCB_ERR_INVALID;
  auto& km = e->km;
  if (!km.capacity) return fail(e, DCB_ERR_STATE, "dcb_kmer_table_clear: no table (dcb_kmer_table_init)");
  if (n_partitions < 1 || partition < 0 || partition >= n_partitions)
    return fail(e, DCB_ERR_INVALID, "dcb_kmer_table_clear: partition %d of %d", partition, n_partitions);
  CU(e, cudaSetDevice(e->cfg.device));
  CU(e, cudaMemsetAsync(km.keys.p, 0xff, km.capacity * sizeof(unsigned long long), e->stream));   // every key empty
  CU(e, cudaMemsetAsync(km.counts.p, 0, km.capacity * sizeof(unsigned int), e->stream));
  CU(e, cudaMemsetAsync(km.stats.p, 0, kKmerStatSlots * sizeof(unsigned long long), e->stream));
  CU(e, cudaStreamSynchronize(e->stream));
  km.partition = partition;
  km.n_partitions = n_partitions;
  return DCB_OK;
}

namespace {

// Stages one batch into pipeline slot `slot`: the bases and offsets, and with `quality` the qualities and flags.
int kmer_stage(dcb_engine* e, const char* who, const dcb_kmer_batch* b, int32_t slot, bool quality, KmerBatch* kb) {
  auto& km = e->km;
  if (!km.capacity) return fail(e, DCB_ERR_STATE, "%s: no table (dcb_kmer_table_init)", who);
  if (!b || slot < 0 || slot > 1) return fail(e, DCB_ERR_INVALID, "%s: null batch or slot %d", who, slot);
  if (b->n_reads < 0 || b->n_bases < 0) return fail(e, DCB_ERR_INVALID, "%s: bad sizes", who);
  if (b->n_reads && (!b->offsets || (b->n_bases && !b->bases) || (quality && (!b->has_qual || (b->n_bases && !b->qual)))))
    return fail(e, DCB_ERR_INVALID, "%s: null array", who);
  if (b->n_reads) {
    if (b->offsets[0] != 0 || b->offsets[b->n_reads] != b->n_bases)
      return fail(e, DCB_ERR_INVALID, "%s: offsets must run from 0 to n_bases", who);
    for (int32_t r = 0; r < b->n_reads; ++r)
      if (b->offsets[r + 1] < b->offsets[r]) return fail(e, DCB_ERR_INVALID, "%s: offsets decrease at read %d", who, r);
  }
  auto& sl = km.slot[slot];
  CU(e, cudaSetDevice(e->cfg.device));
  const uint8_t *d_bases, *d_qual = nullptr, *d_has = nullptr;
  const int64_t* d_off;
  int rc;
  if ((rc = stage_in(e, sl.bases, b->bases, (size_t)b->n_bases, false, &d_bases)) ||
      (rc = stage_in(e, sl.offsets, b->offsets, (size_t)b->n_reads + 1, false, &d_off)) ||
      (quality && ((rc = stage_in(e, sl.qual, b->qual, (size_t)b->n_bases, false, &d_qual)) ||
                   (rc = stage_in(e, sl.has_qual, b->has_qual, (size_t)b->n_reads, false, &d_has)))))
    return rc;
  *kb = KmerBatch{d_bases, d_qual, d_off, d_has, b->n_reads, b->n_bases};
  sl.n_reads = b->n_reads;
  sl.n_bases = b->n_bases;
  return DCB_OK;
}

KmerTable kmer_table(dcb_engine* e) {
  auto& km = e->km;
  return KmerTable{km.keys.p, km.counts.p, km.stats.p, km.capacity, km.k, km.partition, km.n_partitions};
}

KmerTable kmer_set_table(dcb_engine* e) {
  auto& s = e->km.set;
  return KmerTable{s.keys.p, s.counts.p, s.stats.p, s.capacity, e->km.k, s.partition, s.n_partitions};
}

}  // namespace

int dcb_kmer_count(dcb_engine* e, const dcb_kmer_batch* b, int32_t slot) {
  if (!e) return DCB_ERR_INVALID;
  KmerBatch kb;
  int rc = kmer_stage(e, "dcb_kmer_count", b, slot, false, &kb);
  if (rc) return rc;
  auto& sl = e->km.slot[slot];
  sl.query = false;
  CU(e, cudaEventRecord(sl.ev0, e->stream));
  launch_kmer_count(kmer_table(e), kb, e->stream);
  CU(e, cudaGetLastError());
  CU(e, cudaEventRecord(sl.ev1, e->stream));
  return DCB_OK;
}

int dcb_kmer_query(dcb_engine* e, const dcb_kmer_batch* b, int32_t min_count, int32_t with_quality, int32_t slot) {
  if (!e) return DCB_ERR_INVALID;
  if (min_count < 1) return fail(e, DCB_ERR_INVALID, "dcb_kmer_query: min_count must be at least 1, got %d", min_count);
  KmerBatch kb;
  int rc = kmer_stage(e, "dcb_kmer_query", b, slot, with_quality != 0, &kb);
  if (rc) return rc;
  auto& sl = e->km.slot[slot];
  const size_t n = (size_t)std::max(b->n_reads, 1);
  // one CTA per kKmerSegment k-mer end positions of a read, at least one per read
  sl.h_seg_first.assign(1, 0);
  sl.h_seg_read.clear();
  for (int32_t r = 0; r < b->n_reads; ++r) {
    const int64_t segs = std::max<int64_t>(1, (b->offsets[r + 1] - b->offsets[r] + kKmerSegment - 1) / kKmerSegment);
    if ((int64_t)sl.h_seg_read.size() + segs > INT32_MAX)
      return fail(e, DCB_ERR_INVALID, "dcb_kmer_query: the batch needs more than 2^31 segments");
    sl.h_seg_read.insert(sl.h_seg_read.end(), (size_t)segs, r);
    sl.h_seg_first.push_back((int32_t)sl.h_seg_read.size());
  }
  const size_t n_seg = sl.h_seg_read.size();
  const int32_t *d_seg_read, *d_seg_first;
  if ((rc = ensure(e, sl.counts, 2 * n)) || (rc = ensure(e, sl.avg_q, n)) || (rc = ensure(e, sl.border, n)) ||
      (rc = ensure(e, sl.partial, 2 * std::max<size_t>(n_seg, 1))) ||
      (rc = stage_in(e, sl.seg_read, sl.h_seg_read.data(), n_seg, false, &d_seg_read)) ||
      (rc = stage_in(e, sl.seg_first, sl.h_seg_first.data(), sl.h_seg_first.size(), false, &d_seg_first)))
    return rc;
  sl.query = true;
  sl.quality = with_quality != 0;
  CU(e, cudaEventRecord(sl.ev0, e->stream));
  launch_kmer_query(kmer_table(e), kb, KmerSegments{d_seg_read, d_seg_first, (int)n_seg}, (unsigned int)min_count,
                    with_quality ? e->d_p10.p : nullptr, sl.partial.p, sl.counts.p, sl.avg_q.p, sl.border.p, e->stream);
  CU(e, cudaGetLastError());
  CU(e, cudaEventRecord(sl.ev1, e->stream));
  return DCB_OK;
}

int dcb_kmer_wait(dcb_engine* e, int32_t slot, int64_t* counts, double* avg_q, int32_t* borderline, float* ms_out) {
  if (!e) return DCB_ERR_INVALID;
  if (ms_out) *ms_out = 0.f;
  if (slot < 0 || slot > 1 || !e->km.slot[slot].ev1) return fail(e, DCB_ERR_INVALID, "dcb_kmer_wait: bad slot %d", slot);
  auto& sl = e->km.slot[slot];
  CU(e, cudaSetDevice(e->cfg.device));
  // The copies run on the output stream behind this slot's kernel only, so the other slot's kernel keeps running.
  cudaStream_t os = e->out_stream;
  CU(e, cudaStreamWaitEvent(os, sl.ev1, 0));
  const size_t n = (size_t)sl.n_reads;
  if (sl.query && n) {
    if (counts) CU(e, cudaMemcpyAsync(counts, sl.counts.p, 2 * n * sizeof(long long), cudaMemcpyDeviceToHost, os));
    if (sl.quality && avg_q) CU(e, cudaMemcpyAsync(avg_q, sl.avg_q.p, n * sizeof(double), cudaMemcpyDeviceToHost, os));
    if (sl.quality && borderline)
      CU(e, cudaMemcpyAsync(borderline, sl.border.p, n * sizeof(int32_t), cudaMemcpyDeviceToHost, os));
  }
  CU(e, cudaStreamSynchronize(os));
  CU(e, cudaGetLastError());
  if (ms_out) CU(e, cudaEventElapsedTime(ms_out, sl.ev0, sl.ev1));
  return DCB_OK;
}

int dcb_kmer_table_stats(dcb_engine* e, int64_t* stats, int64_t* histogram) {
  if (!e) return DCB_ERR_INVALID;
  auto& km = e->km;
  if (!km.capacity) return fail(e, DCB_ERR_STATE, "dcb_kmer_table_stats: no table (dcb_kmer_table_init)");
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  unsigned long long s[kKmerStatSlots], h[kKmerHist + 1];
  if (histogram) launch_kmer_histogram(kmer_table(e), km.hist_partial.p, kmer_hist_grid(km.capacity), km.hist.p, st);
  CU(e, cudaGetLastError());
  CU(e, cudaMemcpyAsync(s, km.stats.p, sizeof s, cudaMemcpyDeviceToHost, st));
  if (histogram) CU(e, cudaMemcpyAsync(h, km.hist.p, sizeof h, cudaMemcpyDeviceToHost, st));
  CU(e, cudaStreamSynchronize(st));
  if (stats) {
    stats[0] = (int64_t)km.capacity;
    for (int i = 0; i < kKmerStatSlots; ++i) stats[i + 1] = (int64_t)s[i];
  }
  if (histogram)
    for (int c = 0; c <= kKmerHist; ++c) histogram[c] = (int64_t)h[c];
  return DCB_OK;
}

int dcb_kmer_set_init(dcb_engine* e, int64_t table_bytes, int64_t* capacity) {
  if (!e) return DCB_ERR_INVALID;
  auto& km = e->km;
  auto& s = km.set;
  if (!km.capacity) return fail(e, DCB_ERR_STATE, "dcb_kmer_set_init: no table (dcb_kmer_table_init)");
  CU(e, cudaSetDevice(e->cfg.device));
  CU(e, cudaStreamSynchronize(e->stream));
  s.keys.reset(); s.counts.reset(); s.capacity = 0;
  unsigned long long cap;
  int rc = kmer_capacity(e, "dcb_kmer_set_init", table_bytes, &cap);
  if (rc) return rc;
  if ((rc = ensure(e, s.keys, cap)) || (rc = ensure(e, s.counts, cap)) || (rc = ensure(e, s.stats, kKmerStatSlots)) ||
      (rc = ensure(e, s.matrix, (size_t)kSpecBins * kSpecBins)))
    return rc;
  s.capacity = cap;
  if (capacity) *capacity = (int64_t)cap;
  return dcb_kmer_set_clear(e, 0, 1);
}

int dcb_kmer_set_clear(dcb_engine* e, int32_t partition, int32_t n_partitions) {
  if (!e) return DCB_ERR_INVALID;
  auto& s = e->km.set;
  if (!s.capacity) return fail(e, DCB_ERR_STATE, "dcb_kmer_set_clear: no set table (dcb_kmer_set_init)");
  if (n_partitions < 1 || partition < 0 || partition >= n_partitions)
    return fail(e, DCB_ERR_INVALID, "dcb_kmer_set_clear: partition %d of %d", partition, n_partitions);
  CU(e, cudaSetDevice(e->cfg.device));
  CU(e, cudaMemsetAsync(s.keys.p, 0xff, s.capacity * sizeof(unsigned long long), e->stream));   // every key empty
  CU(e, cudaMemsetAsync(s.counts.p, 0, s.capacity * sizeof(unsigned int), e->stream));
  CU(e, cudaMemsetAsync(s.stats.p, 0, kKmerStatSlots * sizeof(unsigned long long), e->stream));
  CU(e, cudaStreamSynchronize(e->stream));
  s.partition = partition;
  s.n_partitions = n_partitions;
  return DCB_OK;
}

int dcb_kmer_set_count(dcb_engine* e, const dcb_kmer_batch* b, const uint8_t* keep, int32_t slot) {
  if (!e) return DCB_ERR_INVALID;
  auto& km = e->km;
  if (!km.set.capacity) return fail(e, DCB_ERR_STATE, "dcb_kmer_set_count: no set table (dcb_kmer_set_init)");
  if (!b || slot < 0 || slot > 1) return fail(e, DCB_ERR_INVALID, "dcb_kmer_set_count: null batch or slot %d", slot);
  if (b->n_reads < 0 || b->n_bases < 0) return fail(e, DCB_ERR_INVALID, "dcb_kmer_set_count: bad sizes");
  if (b->n_reads && !keep) return fail(e, DCB_ERR_INVALID, "dcb_kmer_set_count: null array");
  auto& sl = km.slot[slot];
  // the batch the last dcb_kmer_query or dcb_kmer_count staged on this slot: its bases and offsets are on the device
  if (sl.n_bases < 0 || sl.n_reads != b->n_reads || sl.n_bases != b->n_bases)
    return fail(e, DCB_ERR_INVALID,
                "dcb_kmer_set_count: slot %d holds %d reads and %lld bases, not this batch's %d and %lld (stage it "
                "with dcb_kmer_query first)", slot, sl.n_reads, (long long)sl.n_bases, b->n_reads, (long long)b->n_bases);
  CU(e, cudaSetDevice(e->cfg.device));
  const uint8_t* d_keep;
  int rc = stage_in(e, sl.keep, keep, (size_t)b->n_reads, false, &d_keep);
  if (rc) return rc;
  const KmerBatch kb{sl.bases.p, nullptr, sl.offsets.p, nullptr, b->n_reads, b->n_bases};
  sl.query = false;
  CU(e, cudaEventRecord(sl.ev0, e->stream));
  launch_kmer_set_count(kmer_set_table(e), kb, d_keep, e->stream);
  CU(e, cudaGetLastError());
  CU(e, cudaEventRecord(sl.ev1, e->stream));
  return DCB_OK;
}

int dcb_kmer_spectrum(dcb_engine* e, int64_t* matrix, int64_t* stats) {
  if (!e) return DCB_ERR_INVALID;
  auto& km = e->km;
  auto& s = km.set;
  if (!km.capacity) return fail(e, DCB_ERR_STATE, "dcb_kmer_spectrum: no table (dcb_kmer_table_init)");
  if (!s.capacity) return fail(e, DCB_ERR_STATE, "dcb_kmer_spectrum: no set table (dcb_kmer_set_init)");
  if (!matrix) return fail(e, DCB_ERR_INVALID, "dcb_kmer_spectrum: null array");
  if (s.partition != km.partition || s.n_partitions != km.n_partitions)
    return fail(e, DCB_ERR_STATE, "dcb_kmer_spectrum: the set table holds partition %d of %d, the table %d of %d",
                s.partition, s.n_partitions, km.partition, km.n_partitions);
  CU(e, cudaSetDevice(e->cfg.device));
  cudaStream_t st = e->stream;
  constexpr size_t kCells = (size_t)kSpecBins * kSpecBins;
  CU(e, cudaMemsetAsync(s.matrix.p, 0, kCells * sizeof(unsigned long long), st));
  launch_kmer_spectrum(kmer_table(e), kmer_set_table(e), s.matrix.p, st);
  CU(e, cudaGetLastError());
  std::vector<unsigned long long> m(kCells);
  unsigned long long v[kKmerStatSlots];
  CU(e, cudaMemcpyAsync(m.data(), s.matrix.p, kCells * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  CU(e, cudaMemcpyAsync(v, s.stats.p, sizeof v, cudaMemcpyDeviceToHost, st));
  CU(e, cudaStreamSynchronize(st));
  CU(e, cudaGetLastError());
  for (size_t i = 0; i < kCells; ++i) matrix[i] = (int64_t)m[i];
  if (stats) {
    stats[0] = (int64_t)s.capacity;
    for (int i = 0; i < DCB_KMER_SPECTRUM_STATS - 1; ++i) stats[i + 1] = (int64_t)v[i];
  }
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
