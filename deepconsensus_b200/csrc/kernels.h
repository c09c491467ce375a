// Launchers of the dcb200 device kernels (definitions in kernels.cu).
#pragma once
#include <cuda_runtime.h>

#include <vector>

#include "common.h"

namespace dcb {

cudaError_t kernels_init();

size_t embed_smem_bytes(int R, int echunks, int table_elems);
// `flow` (common.h, TileFlow): the launch's place in the window-aligned forward's tile flow; null flags elsewhere (a
// plain, serialized launch).
// `packed` != null: the rows are read from packed input rows (include/dcb200.h) instead of `rows`.
void launch_embed(const float* rows, const uint8_t* packed, const PackedLayout& pl, int R, int L, int Lw, int M, int ntiles, int echunks,
                  const EmbedCol* cols, const EmbedRow* rowmeta, const __nv_bfloat16* tables,
                  int table_elems, __nv_bfloat16* emb, int* status, const TileFlow& flow, cudaStream_t st);
// D = A * B^T with the 288-wide row epilogue (condenser + pos-enc, attention out-proj).
// b_ksteps == 2 * a_ksteps: b_img holds split-bf16 weights [W_hi; W_lo] along K (kernels.cu, gemm_kernel).
void launch_gemm_row(const __nv_bfloat16* a_img, const __nv_bfloat16* b_img, int a_ksteps, int b_ksteps, int ntiles,
                     const RowEpi& epi, const TileFlow& flow, cudaStream_t st);
// fused q/k/v projection: A [tile][36][128][8] -> qkv image [tile][108][128][8]; b_img: kQKVN / kQKVGroup groups of
// split-bf16 weights [72][kQKVGroup][8] (hi chunks, then lo chunks)
void launch_gemm_qkv(const __nv_bfloat16* a_img, const __nv_bfloat16* b_img, int ntiles,
                     __nv_bfloat16* qkv_img, cudaStream_t st);
// One half of the FFN relu(xb W1 + b1) W2 + b2 with the row epilogue `epi` (kernels.cu, ffn_gemm_kernel): half 0
// runs tiles [0, ceil(ntiles / 2)), half 1 the rest, each over the whole filter.  w1_img: ff / kFFChunk groups of
// [36][kFFChunk][8]; w2_img: [ff/8][288][8].  hid_img, when not null, receives the bf16 hidden activation as an
// operand image [tile][ff/8][128][8].
void launch_ffn(int half, const __nv_bfloat16* xb_img, const __nv_bfloat16* w1_img, const float* b1,
                const __nv_bfloat16* w2_img, int ff, int ntiles, __nv_bfloat16* hid_img, const RowEpi& epi,
                const TileFlow& flow, cudaStream_t st);
void launch_unpack_rows(const uint8_t* packed, const PackedLayout& pl, int nwindows, float* rows, cudaStream_t st);
void launch_attention(const __nv_bfloat16* qkv, __nv_bfloat16* att, int L, int Lw, int win, int nwindows,
                      cudaStream_t st);
// The window-aligned layout only (Lw == kTileM, L <= 128): one half of the q/k/v projection and banded attention with
// q/k/v kept on the SM (kernels.cu, qkv_attention_kernel): half 0 runs tiles [0, ceil(ntiles / 2)), half 1 the rest.
// xb_img: A [tile][36][128][8]; wqkv: launch_gemm_qkv's weight image; att: [tile][36][128][8], rows < L written.
// qkv_img, when not null, also receives the q/k/v image launch_gemm_qkv writes (debug capture).
void launch_qkv_attention(int half, const __nv_bfloat16* xb_img, const __nv_bfloat16* wqkv, int L, int win,
                          int ntiles, __nv_bfloat16* qkv_img, __nv_bfloat16* att, const TileFlow& flow,
                          cudaStream_t st);
void launch_head(const HeadParams& p, int ntiles, const TileFlow& flow, cudaStream_t st);
// Windows of the post-model stage are contiguous in their byte arrays: window w starts at win_off[w] (int64
// [n_windows + 1], windows of any width) or, with win_off NULL, at w * L.
__host__ __device__ inline int64_t window_offset(const int64_t* win_off, int w, int L) {
  return win_off ? win_off[w] : (int64_t)w * L;
}
// per-read window concatenation + gap compaction; read z = windows [zmw_start[z], zmw_start[z+1]) (device pointers)
void launch_stitch(const uint8_t* bases, const uint8_t* quals, int L, const int64_t* win_off, const int32_t* zmw_start,
                   int n_zmw, uint8_t* seq_out, uint8_t* qual_out, int32_t* len_out, cudaStream_t st);


// ---- post-model stage on the device (post_kernels.cu); outcome codes: DCB_READ_* of include/dcb200.h
// The missing-window check counts windows: window i of a read is missing when it starts beyond i * L, whatever the
// widths of the windows before it (stitch_utils.py:60-78).
void launch_read_outcome(const uint8_t* qual, const int32_t* len, const int64_t* win_off, const int32_t* zmw_start,
                         const int32_t* window_pos, int L, int n_zmw, const double* p10, double min_quality, int min_length,
                         int32_t* outcome, double* avg_q, cudaStream_t st);
void launch_fastq(const uint8_t* seq, const uint8_t* qual, const int32_t* len, const int64_t* win_off, const int32_t* zmw_start,
                  int L, int n_zmw, const int32_t* outcome, const uint8_t* names, const int32_t* name_off, int64_t* rec_off,
                  uint8_t* fastq, int64_t cap, cudaStream_t st);
void launch_skip_mask(const int16_t* ccs_bq, int n_windows, int L, const double* p10, double thr, uint8_t* mask,
                      double* avg_out, cudaStream_t st);
// window j of the k skipped windows: src_off[j] .. src_off[j + 1] of ccs_ids / ccs_bq (j * L .. (j + 1) * L with src_off
// NULL; total = the characters of all k), written at window_offset(dst_off, dst[j], L) of bases / quals
void launch_fill_skipped(const uint8_t* ccs_ids, const int16_t* ccs_bq, const int64_t* src_off, const int32_t* dst,
                         const int64_t* dst_off, int k, int L, int64_t total, int calib_enabled, double thr, double cw,
                         double cb, int max_q, uint8_t* bases, uint8_t* quals, int* status, cudaStream_t st);
// head_finish on final logits [n][5] (device pointer) into p.bases / p.quals / p.probs (dcb_debug_head_epilogue)
void launch_head_epilogue(const float* logits, int n, const HeadParams& p, cudaStream_t st);

// ---- feature construction from raw records (prep_kernels.cu); the record arrays are those of dcb_records
// (include/dcb200.h), all pointers device pointers
constexpr int kReadMeta = 10;   // DCB_READ_META
struct PrepZmw {
  int32_t read0, n_reads;     // its subreads in read_meta / read_sn
  int32_t keep;               // min(max_passes, n_reads): the subreads that feed rows (all of them take part in spacing)
  int32_t ccs_off, ccs_len, bq_any;
  int32_t mb;                 // bound on any read's non-insertion columns: `gap` holds mb + 2 entries
  int32_t wb;                 // bound on the spaced width, a multiple of 16
  int32_t win_off, win_cap;   // its slice of win_list
  int32_t wl_off, wl_n;       // CCS smart windows: its window lengths wl[wl_off .. wl_off + wl_n)
  int64_t gap_off;            // element offset into gap
  int64_t plane_off;          // byte offset into spaced: u8 [keep][3][wb] base / pw / ip, u8 [wb] CCS ids, i16 [wb] CCS bq
};
struct PrepBatch {
  int n_zmw, ins_trim;
  PackedLayout pl;
  const PrepZmw* zmw;
  const int32_t* read_meta;
  const float* read_sn;
  const uint32_t* cigar;
  const uint8_t *bases, *pw, *ip, *ccs_bases, *ccs_bq;
  const int32_t* wl;          // CCS smart windows (the `wl` tags, sum = CCS length per ZMW); NULL: fixed-width windows
  // scratch, kept from the layout to the pack calls
  int4* op_scan;              // per cigar operation: columns, non-insertion columns, query bases before it, insertion run in front
  int32_t* read_noni_qs;      // per read: non-insertion columns cut away in front of the clip
  int32_t* gap;               // zeroed before the layout: the gap widths G, then their exclusive scan E
  uint8_t* spaced;            // planes zeroed, CCS bq filled with -1 before the layout
  int4* win_list;             // per ZMW: (start column, window_pos, spaced width) of the windows that hold a CCS position
  int4* zmw_out;              // per ZMW: spaced width, ccs_width, windows, largest non-insertion count
  int* status;                // bit 0: records exceed the bounds they were sized by; bit 1: window index out of range;
                              // bit 2: an overflow window in a CCS read without base qualities
};
struct PrepWindows {          // dense over the batch, ZMW by ZMW
  int32_t* zmw_windows;       // [n_zmw]
  int4* window;               // (ZMW, start column, spaced width)
  int32_t* window_pos;
  uint8_t* overflow;
  int32_t* window_width;
  int32_t* num_passes;
  uint8_t* ccs_ids;           // [n][L]
  int16_t* ccs_bq;            // [n][L]
};
void launch_prep_layout(const PrepBatch& b, const PrepWindows& out, cudaStream_t st);
// packed rows of windows list[0..n_list) (indices into the layout's n_windows windows), in that order
void launch_prep_pack(const PrepBatch& b, const int4* window, const int32_t* list, int n_list, int n_windows, uint8_t* packed,
                      cudaStream_t st);
// training labels of windows list[0..n_list) of the resident layout (dcb_features_labels): meta [n_zmw][kLabelMeta] =
// cigar offset, cigar count, base offset, base count, pos (the indent), ccs0 (CCS index of the first cigar column);
// the cigar holds M / I / D / = / X only, bases are ids 1..4.  scan: n_cigar + n_zmw entries of scratch.
constexpr int kLabelMeta = 6;   // DCB_LABEL_META
struct LabelBatch {
  const int32_t* meta;
  const uint32_t* cigar;
  const uint8_t* bases;
  int4* scan;
};
void launch_labels(const PrepBatch& b, const LabelBatch& lb, const int4* window, const int32_t* list, int n_list,
                   uint8_t* labels_out, uint8_t* status_out, cudaStream_t st);
// evaluation inputs of the resident layout (dcb_features_eval): the label rows and statuses of all n_windows windows
// (label_rows [n][L], status [n]), then the windows with status != 2 whose ZMW has keep_zmw set, compacted in window
// order (dst [n]: place or -1; list [n]: window of each place; *count), and for places below cap their packed row,
// label row and CCS row (ccs_rows: the layout's [n][L]) in packed / labels_out / ccs_out
void launch_features_eval(const PrepBatch& b, const LabelBatch& lb, const int4* window, int n_windows, const uint8_t* ccs_rows,
                          const uint8_t* keep_zmw, int cap, uint8_t* label_rows, uint8_t* status, int32_t* dst, int32_t* list,
                          int* count, uint8_t* packed, uint8_t* labels_out, uint8_t* ccs_out, cudaStream_t st);
// ---- base-quality calibration counts (calib_kernels.cu, dcb_calib_count).  All pointers are device pointers; the
// batch is validated on the host (offsets in bounds, each cigar's query length equal to its base count, endpos equal
// to bam_endpos).  out: int64 [2 * kCalibBins + 3] = counts [bin][match, mismatch], then the lowest failing read
// (-1: none), its reference position and its kind.  partial / partial_fail: grid * 2 * kCalibBins and grid * 2 entries.
constexpr int kCalibMeta = 6;   // DCB_CALIB_META
constexpr int kCalibBins = 100;
constexpr int kCalibPastContig = 1, kCalibBadQuality = 2, kCalibBadInput = 3;   // DCB_CALIB_*
struct CalibBatch {
  const int32_t* read_meta;
  const uint32_t* cigar;
  const uint8_t* seq;
  const uint8_t* qual;
  int n_reads, n_regions;
  const int64_t* regions;
  int64_t interval_length;
  const uint8_t* ref;
  int64_t ref_start, ref_count, contig_length;
  int calibration_enabled;
  double threshold, w, b;
};
void launch_calib_count(const CalibBatch& c, int grid, long long* partial, long long* partial_fail, long long* out,
                        cudaStream_t st);
// ---- read identity (calib_kernels.cu, dcb_read_identity), one CTA per read of a batch validated as for the
// calibration counts.  counts: int64 [n_reads][kIdentityCounts] = matches, mismatches, insertions, deletions,
// soft-clipped bases; avg_q [n_reads]; status [n_reads] = kIdentity*.
constexpr int kIdentityCounts = 5;
constexpr int kIdentityOk = 0, kIdentityPastContig = 1, kIdentitySkipOp = 2, kIdentityBorderline = 3,
              kIdentityBadInput = 4;   // DCB_IDENTITY_*
struct IdentityBatch {
  const int32_t* read_meta;   // [n_reads][kCalibMeta]
  const uint32_t* cigar;
  const uint8_t* seq;
  const uint8_t* qual;
  int n_reads;
  const uint8_t* ref;         // the contig's bases [ref_start, ref_start + ref_count)
  int64_t ref_start, ref_count, contig_length;
  const double* p10;          // 10^(-q/10), q = 0..255
};
void launch_read_identity(const IdentityBatch& c, long long* counts, double* avg_q, int32_t* status, cudaStream_t st);
// ---- read errors (calib_kernels.cu, dcb_read_errors).  launch_run_bounds: every position p of the truth slice ref [n]
// gets its maximal ACGT run [run_start[p], run_end[p]) (slice-relative, the slice's edges cutting runs; [p, p) for a
// non-ACGT byte), by segmented scans in three launches; chunk_* and carry_* hold run_bounds_chunks(n) entries each.
// launch_read_errors: one CTA per read of a batch validated as for read identity, whose slice c.ref the run bounds
// describe; errors: int64 [n_reads][kErrorCols], the DCB_ERRORS_* layout.
constexpr int kErrorBins = 21;   // DCB_ERRORS_*
constexpr int kErrorSub = 0, kErrorInsEvents = 21, kErrorInsBases = 42, kErrorDelEvents = 63, kErrorDelBases = 84,
              kErrorRuns = 105, kErrorMatrix = 126, kErrorCols = 151;
int run_bounds_chunks(int n);
void launch_run_bounds(const uint8_t* ref, int n, int* chunk_start, int* chunk_end, int* carry_start, int* carry_end,
                       int* run_start, int* run_end, cudaStream_t st);
void launch_read_errors(const IdentityBatch& c, const int* run_start, const int* run_end, long long* errors,
                        cudaStream_t st);
// ---- k-mer table (kmer_kernels.cu, dcb_kmer_*).  keys: capacity uint64 (kKmerEmpty = free), counts: capacity uint32,
// capacity a power of two.  stats: uint64 [kKmerStatSlots] = claimed keys, overflow flag, k-mers counted, their probe
// steps, k-mers queried, their probe steps.  Device pointers.
constexpr unsigned long long kKmerEmpty = ~0ull;
constexpr int kKmerStatSlots = 6;
constexpr int kKmerHist = 256;   // DCB_KMER_HIST
struct KmerTable {
  unsigned long long* keys;
  unsigned int* counts;
  unsigned long long* stats;
  unsigned long long capacity;
  int k, partition, n_partitions;
};
struct KmerBatch {
  const uint8_t* bases;
  const uint8_t* qual;
  const int64_t* offsets;      // [n_reads + 1]
  const uint8_t* has_qual;
  int n_reads;
  int64_t n_bases;
};
void launch_kmer_count(const KmerTable& t, const KmerBatch& b, cudaStream_t st);
// The query's CTAs: read r is segments first[r] .. first[r + 1] - 1 (at least one), each of kKmerSegment k-mer end
// positions but the last; read[s] is segment s's read.
constexpr int kKmerSegment = 16384;
struct KmerSegments {
  const int32_t* read;    // [n_segments]
  const int32_t* first;   // [n_reads + 1]
  int n_segments;
};
// per read: counts [2r] = k-mer positions of the partition, [2r + 1] = those with a count below min_count; with p10
// (not null), avg_q [r] and borderline [r] as dcb_read_identity's avg_phred.  partial: 2 x n_segments entries.
void launch_kmer_query(const KmerTable& t, const KmerBatch& b, const KmerSegments& sg, unsigned int min_count,
                       const double* p10, long long* partial, long long* counts, double* avg_q, int32_t* borderline,
                       cudaStream_t st);
// hist [kKmerHist + 1]: [c] = keys with count c (c = 1..255), [kKmerHist] = keys with count >= 256; partial holds
// grid x (kKmerHist + 1) entries, grid from kmer_hist_grid
int kmer_hist_grid(unsigned long long capacity);
void launch_kmer_histogram(const KmerTable& t, unsigned long long* partial, int grid, unsigned long long* hist,
                           cudaStream_t st);
// The set table (`kmer_qv --spectrum`): the same layout, slot and partition rule, and stats slots 0..3.
// launch_kmer_set_count counts the k-mers of the reads with keep[r] != 0 (device [n_reads]) into it.
void launch_kmer_set_count(const KmerTable& set, const KmerBatch& b, const uint8_t* keep, cudaStream_t st);
// matrix [kSpecBins][kSpecBins] (zeroed by the caller) += distinct keys of the partition by (short count, set count),
// each capped at kKmerHist.  Both tables hold the same partition.
constexpr int kSpecBins = kKmerHist + 1;   // DCB_KMER_SPECTRUM_BINS
void launch_kmer_spectrum(const KmerTable& shrt, const KmerTable& set, unsigned long long* matrix, cudaStream_t st);
// the CCS ids / qualities of windows list[0..n_list) at full width, window j at off[j] of ccs_ids / ccs_bq
void launch_features_ccs(const PrepBatch& b, const int4* window, const int32_t* list, int n_list, const int64_t* off,
                         uint8_t* ccs_ids, int16_t* ccs_bq, cudaStream_t st);

// ---- evaluation on labelled windows (eval_kernels.cu): alignment loss, exact-match flag, alignment counts [B][5] of
// the prediction and of the CCS row.  hard_min != 0: loss_reg None.  All pointers are device pointers.
cudaError_t launch_evaluate(const float* probs, const uint8_t* labels, const uint8_t* ccs_ids, int B, int L,
                            float del_cost, float loss_reg, int hard_min, float* loss, uint8_t* exact,
                            int32_t* pred_counts, int32_t* ccs_counts, cudaStream_t st);
// Base-quality calibration counts of align_identity_kernel<true>: qualities 0..kCalibBins-1 (the bins of
// dcb_calib_count), column 0 match, 1 mismatch.
constexpr int kCalibMaxQ = 93;   // the head's cap (max_base_quality) on the prediction's quality
struct EvalCalibOut {
  const uint8_t* ccs_bq;         // [B, L] raw CCS base quality of every position
  unsigned long long* counts;    // int64 [2][kCalibBins][2] (prediction, CCS), zeroed by the caller; added to
  unsigned long long* deletions; // int64 [2], zeroed by the caller; added to
  int* bad_window;               // INT_MAX from the caller; the lowest window with a quality above kCalibBins - 1
};
// Byte offset of the shared histogram in align_identity_kernel<true>'s dynamic shared memory.
__host__ __device__ constexpr size_t eval_calib_hist_offset(int L) {
  return ((size_t)9 * (L + 1) * sizeof(float) + 6 * (size_t)L + (size_t)(L + 1) * (L + 1) + 3) / 4 * 4;
}
// launch_evaluate's identity kernel with the calibration counts (no loss).  Device pointers.
cudaError_t launch_evaluate_calibration(const float* probs, const uint8_t* labels, const uint8_t* ccs_ids, int B,
                                        int L, uint8_t* exact, int32_t* pred_counts, int32_t* ccs_counts,
                                        const EvalCalibOut& calib, cudaStream_t st);
// labels u8 [n] (device) copied to out with every id above 4 replaced by 0; *bad (zeroed by the caller) is set to 1 when
// there was one, so that the evaluation kernels index only inside their tables and the call can refuse the labels
void launch_copy_label_ids(const uint8_t* labels, uint8_t* out, size_t n, int* bad, cudaStream_t st);
// AlignmentLoss per window with its gradient: loss [B], d loss / d probs [B, L, 5] and the soft alignment matches
// [B, L, L] (both nullable).  `tables` is loss_grad_table_bytes(L, ctas) of device scratch, ctas from loss_grad_grid(B)
// (persistent grid on the current device).  Device pointers.
cudaError_t loss_grad_grid(int B, int* ctas);
size_t loss_grad_table_bytes(int L, int ctas);
cudaError_t launch_loss_grad(const float* probs, const uint8_t* labels, int B, int L, float del_cost, float loss_reg,
                             int hard_min, float* tables, int ctas, float* loss, float* grad, float* matches,
                             cudaStream_t st);
// DistillationLoss per window from teacher / student logits [B, L, 5]; logit_loss 0 = mean squared error, 1 = KL
// divergence (DCB_LOGIT_LOSS_*).  When grad is not null, also its gradient d loss / d student [B, L, 5] with the
// teacher held constant; the loss bits are the same either way.  Device pointers.
cudaError_t launch_distill_loss_grad(const float* teacher, const float* student, int B, int L, float temperature,
                                     int logit_loss, float* loss, float* grad, cudaStream_t st);

// ---- strict-fp32 path (strict_kernels.cu): row-major float32 activations, windows packed back to back
void launch_strict_embed(const float* rows, int R, int L, int E, int nwindows, const StrictEmbedRow* meta,
                         const float* tables, float* emb, int* status, cudaStream_t st);
void launch_strict_gemm(const float* A, const float* B, float* C, int M, int N, int K, const StrictEpi& ep,
                        cudaStream_t st);
void launch_strict_layernorm(const float* x, float* y, int M, const float* g, const float* b, cudaStream_t st);
void launch_strict_attention(const float* q, const float* k, const float* v, float* o, int nwindows, int L, int win,
                             cudaStream_t st);
void launch_strict_head(const float* x, int M, const HeadParams& hp, cudaStream_t st);

// ---- tf32x3 path (tf32x3_kernels.cu): the strict path's GEMM on the tensor cores, same arguments and epilogue, with
// W [K][N] (row-major float32) given as its tf32x3_image
cudaError_t tf32x3_init();
size_t tf32x3_image_elems(int K, int N);
std::vector<float> tf32x3_image(const float* W, int K, int N);
void launch_tf32x3_gemm(const float* A, const float* Wimg, float* C, int M, int N, int K, const StrictEpi& ep,
                        cudaStream_t st);

}  // namespace dcb
