/* dcb200 -- C ABI of the H100-native (sm_90a) DeepConsensus model path.
 *
 * This is the drop-in boundary for the one hot path of google/deepconsensus (v1.2.0):
 *
 *   quick_inference.initialize_model()          deepconsensus/inference/quick_inference.py:485-532
 *   quick_inference.run_model_on_examples()     deepconsensus/inference/quick_inference.py:341-415
 *     -> model.predict(rows)                    deepconsensus/models/networks.py:357-365 (:221-345, :436-520)
 *     -> argmax / Phred / calibration / clip    quick_inference.py:377-389, quality_calibration/calibration_lib.py:77-99
 *     -> per-window base + quality strings      quick_inference.py:390-414, utils/utils.py:60-62
 *
 * The reference has no FFI (it is pure Python on TensorFlow); the binding a maintainer adds
 * is a ctypes stub -- see INTEGRATION.md and deepconsensus_b200/engine.py.
 *
 * Conventions: plain C, no exceptions across the boundary.  Every function returns
 * DCB_OK (0) or a negative error code; dcb_last_error() gives the message.  All buffers are
 * caller-owned and caller-sized.  One engine per device, not re-entrant (the reference
 * touches the model from its main thread only).  Results are deterministic (no atomics in
 * any reduction).
 */
#ifndef DCB200_H_
#define DCB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DCB_OK 0
#define DCB_ERR_INVALID (-1)     /* bad argument / unsupported configuration */
#define DCB_ERR_CUDA (-2)        /* CUDA runtime error (message has the detail) */
#define DCB_ERR_WEIGHTS (-3)     /* missing / mis-shaped variable */
#define DCB_ERR_STATE (-4)       /* call order (e.g. forward before load_weights) */
#define DCB_ERR_INPUT_RANGE (-5) /* an embedding id was out of range (TF would raise); output still produced with clamped ids */

typedef struct dcb_engine dcb_engine;

/* Model + inference options.  Field names follow params.json / InferenceOptions
 * (models/model_configs.py:76-139,272-338; quick_inference.py:238-275). */
typedef struct dcb_config {
  int32_t struct_size;        /* sizeof(dcb_config), for ABI checking */
  int32_t device;             /* CUDA device ordinal */
  /* input geometry (data_providers.py:61-113) */
  int32_t max_passes;
  int32_t max_length;
  int32_t use_ccs_bq;
  /* transformer (transformer_basic_params.py:33-67 merged under model_configs.py) */
  int32_t hidden_size;        /* must be 280 */
  int32_t num_heads;          /* must be 2 */
  int32_t num_hidden_layers;
  int32_t filter_size;        /* multiple of 128, <= 2048 */
  int32_t attn_win_size;      /* 0 => full attention (params.attn_win_size None) */
  int32_t rezero;             /* 1: x + alpha*f(x); 0: x + f(LayerNorm(x)) (encoder_stack.py:72-93) */
  int32_t add_pos_encoding;
  int32_t condense_transformer_input; /* must be 1 (transformer_input_size == hidden_size) */
  /* embedding widths and vocabularies (networks.py:375-421) */
  int32_t per_base_hidden_size, pw_hidden_size, ip_hidden_size, strand_hidden_size,
      ccs_bq_hidden_size, sn_hidden_size;
  int32_t pw_max, ip_max, sn_max, ccs_bq_max, strand_max;
  /* post-processing (quick_inference.py:377-389) */
  int32_t max_base_quality;   /* 93 */
  int32_t calibration_enabled;
  double calibration_threshold, calibration_w, calibration_b;
  /* engine sizing */
  int32_t max_batch;          /* largest B a single dcb_forward call will see */
  int32_t chunk_tiles;        /* 128-token tiles processed per pass through the layer stack; 0 = auto */
  int32_t precision;          /* DCB_PRECISION_BF16 (default), DCB_PRECISION_FP32 or DCB_PRECISION_TF32X3: which
                                 arithmetic dcb_forward uses when the call does not say (see DCB_STRICT_FP32) */
  int32_t reserved[5];
} dcb_config;

/* Arithmetic of the forward pass.
 *   DCB_PRECISION_BF16  tensor-core path: bf16 operands, float32 accumulation / residual / LayerNorm / softmax.
 *                       Logits differ from the reference's float32 graph by the operand rounding (0.02-0.1 on
 *                       random-weight models), so the argmax can flip at near-ties.
 *   DCB_PRECISION_FP32  the reference's own arithmetic (float32 operands and accumulation, networks.py:506-507):
 *                       differs from the reference by summation order only (~1e-5 on logits); identical bases wherever
 *                       the float32 top-2 logit margin exceeds 1e-3.  CUDA-core kernels, ~25x slower.
 *   DCB_PRECISION_TF32X3 the DCB_PRECISION_FP32 forward with its GEMMs on the tensor cores: every float32 operand is
 *                       split into two tf32 parts and three products are accumulated in float32 (3xTF32), which loses
 *                       ~2^-22 relative per operand.  The same accuracy gates as DCB_PRECISION_FP32; its split weight
 *                       images are built only for engines created with this precision.  DCB_STRICT_FP32 and
 *                       DCB_FAST_BF16 still select those paths per call. */
#define DCB_PRECISION_BF16 0
#define DCB_PRECISION_FP32 1
#define DCB_PRECISION_TF32X3 2

/* A named host tensor in the reference checkpoint's layout, e.g.
 * "model/encoder_stack/layers/0/0/layer/query_dense_layer/kernel" float32 [280,2,140]. */
typedef struct dcb_tensor {
  const char* name;
  const float* data;   /* host pointer, C-contiguous float32 */
  int32_t ndim;
  int64_t shape[4];
} dcb_tensor;

/* flags for dcb_forward */
#define DCB_ROWS_ON_DEVICE 1u   /* `rows` is a device pointer (already resident in HBM); must be 16-byte aligned */
#define DCB_OUT_ON_DEVICE 2u    /* output pointers are device pointers */
#define DCB_STRICT_FP32 4u      /* this call runs in float32 (DCB_PRECISION_FP32) whatever dcb_config.precision says */
#define DCB_FAST_BF16 8u        /* this call runs the bf16 tensor-core path whatever dcb_config.precision says */
#define DCB_LABELS_ON_DEVICE 16u /* dcb_evaluate: `labels` and `ccs_ids` are device arrays (e.g. dcb_features_eval's) */

/* Create an engine on cfg->device.  Replaces model construction in initialize_model
 * (quick_inference.py:515-526). */
int dcb_create(const dcb_config* cfg, dcb_engine** out);

/* Load all variables (host fp32, reference shapes); the engine pads, folds (query scale,
 * ReZero alpha) and casts into its device layouts.  Replaces checkpoint.restore(...)
 * (quick_inference.py:527-529).  Unknown names are ignored (expect_partial); every variable
 * the configured model needs must be present. */
int dcb_load_weights(dcb_engine* e, const dcb_tensor* tensors, int32_t n);

/* The hot path: rows float32 [B, total_rows, max_length] (the [B,R,L,1] tensor of
 * quick_inference.py:363 with the channel axis dropped; NOT pre-clipped -- format_rows'
 * clipping happens on the device) -> per position base character (' ', 'A', 'T', 'C', 'G')
 * and Phred+33 quality character.  probs_out / logits_out ([B, L, 5] float32) may be NULL. */
int dcb_forward(dcb_engine* e, const float* rows, int32_t batch, uint32_t flags,
                uint8_t* bases_out, uint8_t* quals_out, float* probs_out, float* logits_out);

/* ---- packed input rows (the feature-construction side of the path) ----------------------------------------------------
 * The float32 [B, R, L] rows of quick_inference.py:363 hold small integers: bases / ccs in 0..4, pw / ip from uint8
 * BAM tags (pre_lib.py:221-226,704-744), strand in 0..2, ccs_bq in -1..93, plus four float SN values per window that
 * extract_features repeats along L (pre_lib.py:741-742).  The packed form keeps exactly that information in
 * dcb_packed_window_bytes() bytes per window (7,344 B instead of 40,800 B for 20 x 120) -- per window, in this order:
 *     u8 [P][L]   bits 0-2 = base id of subread p (row p), bits 3-4 = its strand id (row 3P + p)
 *     u8 [P][L]   pw (rows P..2P-1),   clipped to [0, 255] and truncated, as format_rows + tf.cast would
 *     u8 [P][L]   ip (rows 2P..3P-1),  same
 *     u8 [L]      ccs base id (row 4P)
 *     u8 [L]      ccs_bq + 1 (row 4P+1; only when use_ccs_bq) -- the embedding id itself (networks.py:495)
 *     padding to a multiple of 16 bytes
 *     f32 [4]     the window's SN values (rows R-4..R-1, taken at position 0; not clipped)
 * The engine turns packed bytes into table ids inside its embedding kernel (PW_MAX / IP_MAX / SN_MAX clipping included);
 * results are bit-identical to dcb_forward on the float32 rows the packed form was made from.
 *
 * dcb_pack_rows: host helper (needs no GPU and no engine -- it belongs to the producer of the rows; only max_passes,
 * max_length, use_ccs_bq and the *_max fields of `cfg` are read), float32 rows [B, R, L] -> packed.  Returns DCB_ERR_INPUT_RANGE (and still writes
 * clamped output) if a base / strand / ccs / ccs_bq value is outside its vocabulary -- the values TensorFlow's gather
 * would raise on -- or an SN row is not constant along L; DCB_ERR_INVALID if the configuration cannot be packed:
 * PW_MAX or IP_MAX above 255, STRAND_MAX above 3 (two bits) or CCS_BQ_MAX above 256 (its largest id, CCS_BQ_MAX - 1,
 * must fit a byte).  The packed entry points refuse such an engine with DCB_ERR_INVALID too. */
size_t dcb_packed_window_bytes(const dcb_config* cfg);
int dcb_pack_rows(const dcb_config* cfg, const float* rows, int32_t batch, uint8_t* packed_out);
/* dcb_forward / dcb_submit on packed rows (host pointer, or device pointer with DCB_ROWS_ON_DEVICE: 16-byte aligned). */
int dcb_forward_packed(dcb_engine* e, const uint8_t* packed, int32_t batch, uint32_t flags,
                       uint8_t* bases_out, uint8_t* quals_out, float* probs_out, float* logits_out);
int dcb_submit_packed(dcb_engine* e, const uint8_t* packed, int32_t batch, uint32_t flags,
                      uint8_t* bases_out, uint8_t* quals_out, float* probs_out, float* logits_out, int64_t* ticket);

/* Pipelined form of dcb_forward for a stream of batches (the `for batch in batches: model.predict(batch)` loop of
 * quick_inference.py:352-368): dcb_submit enqueues the host->device copy of `rows` on a copy stream, the kernels and
 * the device->host copy of the results, and returns a ticket without waiting; dcb_wait(ticket) blocks until that
 * batch's outputs are in the caller's buffers and returns its status (DCB_ERR_INPUT_RANGE etc.).  At most TWO
 * submissions may be in flight, so the copy of batch i+1 overlaps the kernels of batch i; tickets must be waited for in
 * order.  `rows` and the output buffers must stay valid (and should be page-locked, dcb_alloc_host) until dcb_wait
 * returns.  dcb_forward == dcb_submit + dcb_wait. */
int dcb_submit(dcb_engine* e, const float* rows, int32_t batch, uint32_t flags,
               uint8_t* bases_out, uint8_t* quals_out, float* probs_out, float* logits_out, int64_t* ticket);
int dcb_wait(dcb_engine* e, int64_t ticket);

/* The first stage of stitch_utils.stitch_to_fastq for a batch of reads -- get_full_sequence + remove_gaps
 * (stitch_utils.py:51-98) -- on the device: the windows [zmw_start[z], zmw_start[z+1]) of `bases` / `quals`
 * ([n_windows, L] bytes exactly as dcb_forward writes them, sorted by window position) are concatenated and the gap
 * character ' ' is dropped together with the quality character under it.  Read z is written at offset
 * zmw_start[z] * L of seq_out / qual_out (each n_windows * L bytes) and len_out[z] receives its length.  zmw_start is a
 * host array of n_zmw + 1 non-decreasing window indices.  flags: DCB_ROWS_ON_DEVICE => bases/quals are device
 * pointers (e.g. the DCB_OUT_ON_DEVICE outputs of dcb_forward); DCB_OUT_ON_DEVICE => seq_out/qual_out/len_out are
 * device pointers.  The missing-window check and the empty / quality / length filters stay with the caller
 * (deepconsensus_b200/stitch_gpu.py), which has the window positions and read names. */
int dcb_stitch(dcb_engine* e, const uint8_t* bases, const uint8_t* quals, int32_t n_windows, int32_t L,
               const int32_t* zmw_start, int32_t n_zmw, uint32_t flags,
               uint8_t* seq_out, uint8_t* qual_out, int32_t* len_out);

/* ---- the rest of the post-model stage on the device --------------------------------------------------------------------
 * dcb_stitch_fastq = stitch_utils.stitch_to_fastq for a batch of reads (stitch_utils.py:131-189): dcb_stitch, then per
 * read the missing-window check of get_full_sequence (window i must not start beyond i * L, stitch_utils.py:60-78), the
 * only-gaps check, the quality filter round(avg_phred(quals), 5) >= min_quality (utils.py:88-106,
 * stitch_utils.py:101-109), the length filter, and for the reads that pass the FASTQ record
 * '@' name '\n' sequence "\n+\n" quality '\n' (stitch_utils.py:112-119) written at rec_off[z] of fastq_out.
 *   window_pos [n_windows]   DCModelOutput.window_pos of every window (sorted within a read)
 *   names / name_off         the read names, concatenated; read z is names[name_off[z] .. name_off[z+1])
 *   fastq_out, fastq_cap     caller-sized; names + 2 * n_windows * L + 6 * n_zmw bytes always suffice
 *   rec_off [n_zmw + 1]      byte offset of every read's record (rec_off[n_zmw] = total bytes written)
 *   outcome [n_zmw]          DCB_READ_* -- the OutcomeCounter field the reference would bump
 *   avg_q [n_zmw]            the read's average Phred (float64)
 * bases / quals are host arrays, or device arrays with DCB_ROWS_ON_DEVICE (e.g. dcb_forward's DCB_OUT_ON_DEVICE
 * outputs); every output is a host array.  A read whose average quality lies within 1e-7 of the filter threshold is
 * reported with DCB_READ_BORDERLINE or-ed in (its record IS written): the caller re-evaluates that read with the
 * reference's own float64 expression, because NumPy's pairwise sum and the histogram sum used here may differ in the
 * last bits (deepconsensus_b200/stitch_gpu.py does). */
#define DCB_READ_OK 0
#define DCB_READ_EMPTY 1          /* OutcomeCounter.empty_sequence (a window is missing) */
#define DCB_READ_ONLY_GAPS 2      /* OutcomeCounter.only_gaps */
#define DCB_READ_LOW_QUALITY 3    /* OutcomeCounter.failed_quality_filter */
#define DCB_READ_TOO_SHORT 4      /* OutcomeCounter.failed_length_filter */
#define DCB_READ_BORDERLINE 0x80  /* flag: quality within 1e-7 of the threshold, caller decides */
int dcb_stitch_fastq(dcb_engine* e, const uint8_t* bases, const uint8_t* quals, int32_t n_windows, int32_t L,
                     const int32_t* zmw_start, int32_t n_zmw, const int32_t* window_pos,
                     const uint8_t* names, const int32_t* name_off, double min_quality, int32_t min_length,
                     uint32_t flags, uint8_t* fastq_out, int64_t fastq_cap, int64_t* rec_off, int32_t* outcome,
                     double* avg_q);

/* The skip decision of inference_on_n_zmws (quick_inference.py:663-672) for a batch of windows:
 * mask[w] = avg_phred(ccs_bq[w, :]) > skip_windows_above (entries < 0 are spacing and are dropped, utils.py:88-106);
 * 2 = within 1e-7 of the threshold, caller decides.  ccs_bq: host int16 [n_windows, L]. */
int dcb_skip_mask(dcb_engine* e, const int16_t* ccs_bq, int32_t n_windows, int32_t L, double skip_windows_above,
                  uint8_t* mask_out, double* avg_out /* nullable */);

/* process_skipped_window (quick_inference.py:567-594) for k windows that bypass the model: window j adopts the CCS
 * bases (ccs_ids, host u8 [k, L], ids 0..4 -> ' ATCG') and the CCS base qualities (ccs_bq, host int16 [k, L]) after
 * calibrate_quality_scores (calibration_lib.py:77-99; float64) / min(., max_base_quality) / int32 truncation / +33,
 * and is written to row dst_window[j] of bases / quals ([*, L]; device arrays with DCB_OUT_ON_DEVICE -- e.g. the arrays
 * dcb_forward filled for the scored windows, so that dcb_stitch_fastq can run on them without a host round trip). */
int dcb_fill_skipped(dcb_engine* e, const uint8_t* ccs_ids, const int16_t* ccs_bq, const int32_t* dst_window, int32_t k,
                     int32_t L, int32_t calibration_enabled, double calibration_threshold, double calibration_w,
                     double calibration_b, uint32_t flags, uint8_t* bases, uint8_t* quals);

/* ---- windows of different widths (CCS smart windows: overflow windows keep their full width) ------------------------
 * The same three calls on windows laid out back to back at any width: window w is bytes win_off[w] .. win_off[w + 1]
 * of bases / quals (win_off: host int64 [n_windows + 1], win_off[0] = 0, non-decreasing).  dcb_stitch,
 * dcb_stitch_fastq and dcb_fill_skipped are these calls with win_off[w] = w * L; they run the same kernels.
 *   dcb_stitch_ragged        read z is written at win_off[zmw_start[z]] of seq_out / qual_out (win_off[n_windows] bytes)
 *   dcb_stitch_fastq_ragged  the missing-window check still counts windows: window i of a read is missing when its
 *                            window_pos exceeds i * L, whatever the widths before it (stitch_utils.py:60-78); fastq_cap:
 *                            names + 2 * win_off[n_windows] + 6 * n_zmw bytes always suffice
 *   dcb_fill_skipped_ragged  skipped window j is src_off[j] .. src_off[j + 1] of ccs_ids / ccs_bq (src_off [k + 1]) and
 *                            goes to window dst_window[j] of the output arrays, whose windows are dst_off [n_dst + 1];
 *                            the two widths must agree */
int dcb_stitch_ragged(dcb_engine* e, const uint8_t* bases, const uint8_t* quals, const int64_t* win_off, int32_t n_windows,
                      const int32_t* zmw_start, int32_t n_zmw, uint32_t flags, uint8_t* seq_out, uint8_t* qual_out,
                      int32_t* len_out);
int dcb_stitch_fastq_ragged(dcb_engine* e, const uint8_t* bases, const uint8_t* quals, const int64_t* win_off,
                            int32_t n_windows, int32_t L, const int32_t* zmw_start, int32_t n_zmw, const int32_t* window_pos,
                            const uint8_t* names, const int32_t* name_off, double min_quality, int32_t min_length,
                            uint32_t flags, uint8_t* fastq_out, int64_t fastq_cap, int64_t* rec_off, int32_t* outcome,
                            double* avg_q);
int dcb_fill_skipped_ragged(dcb_engine* e, const uint8_t* ccs_ids, const int16_t* ccs_bq, const int64_t* src_off,
                            const int32_t* dst_window, int32_t k, const int64_t* dst_off, int32_t n_dst,
                            int32_t calibration_enabled, double calibration_threshold, double calibration_w,
                            double calibration_b, uint32_t flags, uint8_t* bases, uint8_t* quals);

/* ---- evaluation of labelled windows ---------------------------------------------------------------------------------
 * What model_inference.py (models/model_inference.py:79-120 -> model_utils.run_inference_and_write_results,
 * model_utils.py:379-421) has `model.evaluate` compute per window, and the identity of the training loop's metrics
 * (model_utils.get_deepconsensus_metrics, model_utils.py:69-96), for a batch of B windows of length L <= 256:
 *   loss_out [B]         AlignmentLoss.eval with width=None (losses_and_metrics.py:306-411,549-595): label left-shifted
 *                        (:92-115), probs renormalised to sum to 1, xentropy substitution / insertion costs clipped at
 *                        1e-7 (:123-143,191-207), constant del_cost, soft-min -loss_reg * logsumexp(-t / loss_reg) --
 *                        or the hard min when loss_reg <= 0 (params.loss_reg None) -- read at anti-diagonal
 *                        seq_len + L, row seq_len.  float32, as the reference.
 *   exact_out [B]        PerExampleAccuracy (losses_and_metrics.py:37-65): 1 when the left-shifted argmax prediction
 *                        equals the left-shifted label at all L positions.
 *   pred_counts [B][5]   AlignmentMetric.alignment (losses_and_metrics.py:704-1043) of the label against the
 *                        argmax-decoded prediction: num_matches, num_insertions, num_deletions, num_correct_matches,
 *                        alignment_length (affine gaps: match +2, mismatch -5, open 5+4, extend 4; ties go to the
 *                        first of [match, ins, del]).
 *   ccs_counts [B][5]    the same against the window's CCS row (get_batch_identity_ccs_pred,
 *                        losses_and_metrics.py:1061-1098; the row is model_utils.get_ccs_from_example,
 *                        model_utils.py:128-139, i.e. row 4 * max_passes of data_providers.get_indices).
 * probs float32 [B, L, 5]: a host array, or with DCB_ROWS_ON_DEVICE a device array (e.g. the DCB_OUT_ON_DEVICE probs_out
 * of dcb_forward / dcb_forward_packed, so that the probabilities never leave the GPU).  labels / ccs_ids: host u8 [B, L],
 * ids 0..4 over ' ATCG' (labels outside 0..4 are DCB_ERR_INVALID; a CCS id outside 0..4 counts as a gap, as its
 * all-zero one-hot row decodes); with DCB_LABELS_ON_DEVICE both are device arrays, read in place, and the label check
 * runs on the device (the kernels then see no label id above 4, and the call still returns DCB_ERR_INVALID).  band_width >= 0 (the banded AlignmentLoss, params.band_width set) is DCB_ERR_INVALID;
 * pass DCB_BAND_WIDTH_NONE.  Outputs are host arrays; ms_out (nullable) receives the device time of the evaluation
 * kernels.  Deterministic: repeated calls give identical bits. */
#define DCB_BAND_WIDTH_NONE (-1)
int dcb_evaluate(dcb_engine* e, const float* probs, const uint8_t* labels, const uint8_t* ccs_ids, int32_t batch,
                 int32_t L, double del_cost, double loss_reg, int32_t band_width, uint32_t flags, float* loss_out,
                 uint8_t* exact_out, int32_t* pred_counts, int32_t* ccs_counts, float* ms_out);

/* Base-quality calibration counts of labelled windows: the traceback of dcb_evaluate's AlignmentMetric counts
 * classifies every base of the left-shifted argmax prediction and of the left-shifted CCS row, and each base's quality
 * is binned by that class, as calculate_baseq_calibration bins a read's M / I / D operations:
 *   an edge-1 base equal to its label base        match
 *   an edge-1 base that differs, an edge-2/3 base  mismatch (an inserted base is unaligned)
 *   a label base on edge 4/5                       a deletion: no quality, only counted
 * The prediction's quality is the head's epilogue without calibration, -10 log10(1 - p_max) of the probability row
 * the base was decoded from, capped at 93 and rounded half to even (the quality byte minus 33 of a forward with
 * calibration skipped); the CCS row's is ccs_bq u8 [B, L], its raw base quality.  A quality stays with its base through
 * the left shift.  Per window, sum match = num_correct_matches, sum mismatch = num_matches - num_correct_matches +
 * num_insertions, deletions = num_deletions.
 *   counts_out int64 [2][DCB_CALIB_BINS][2]   [prediction, CCS][quality][match, mismatch] of the batch
 *   deletions_out int64 [2]                   label bases deleted against the prediction and against the CCS row
 *   pred_counts, ccs_counts int32 [B][5]      bitwise dcb_evaluate's
 * probs, labels, ccs_ids, flags and the argument checks are dcb_evaluate's (no loss is computed, so there is no
 * del_cost, loss_reg or band_width); with DCB_LABELS_ON_DEVICE ccs_bq is a device array too.  A binned CCS quality
 * above DCB_CALIB_BINS - 1 is DCB_ERR_INVALID naming the window.  Outputs are host arrays; ms_out (nullable) receives
 * the kernel's device time.  The counts are integer sums: they do not depend on how windows are split into calls. */
#define DCB_CALIB_BINS 100
int dcb_evaluate_calibration(dcb_engine* e, const float* probs, const uint8_t* labels, const uint8_t* ccs_ids,
                             const uint8_t* ccs_bq, int32_t batch, int32_t L, uint32_t flags, int64_t* counts_out,
                             int64_t* deletions_out, int32_t* pred_counts, int32_t* ccs_counts, float* ms_out);

/* The gradient of the alignment loss, for training: AlignmentLoss.eval(return_matches=True)
 * (losses_and_metrics.py:549-595, width=None) and the gradient the training loop's tape takes of the per-window loss
 * with respect to y_pred (model_train_custom_loop.py, model_distillation.py).  For B windows of length L <= 256, probs
 * float32 [B, L, 5] and labels u8 [B, L] (ids 0..4 over ' ATCG'):
 *   loss_out [B]            the loss, bitwise equal to dcb_evaluate's loss_out on the same arguments
 *   grad_out [B, L, 5]      d loss[b] / d probs[b] (nullable): float32, with TensorFlow's gradient semantics -- the
 *                           soft-min's gradient is softmax(-t / loss_reg), the hard min's splits equally among exactly
 *                           tied minima, clip_by_value passes at its bounds and is zero outside, xlogy is zero where
 *                           the one-hot label is zero, probs are renormalised to sum to 1 on the way in
 *   matches_out [B, L, L]   d loss[b] / d substitution cost [i][j] (nullable): the soft alignment of left-shifted label
 *                           position i to prediction position j; rows at or beyond the label's length are 0
 * loss_reg <= 0 is the hard min (params.loss_reg None); band_width >= 0 is DCB_ERR_INVALID (pass DCB_BAND_WIDTH_NONE).
 * probs / labels are host arrays, or device arrays with DCB_ROWS_ON_DEVICE; outputs are host arrays, or device arrays
 * with DCB_OUT_ON_DEVICE.  The engine keeps every DP cell of each window in device scratch it grows on demand ((L + 1)^2
 * floats per resident CTA).  ms_out (nullable) receives the kernel's device time.  Returns once the work on the engine's
 * stream has finished.  DCB_ERR_INVALID for batch < 0, L outside 1..256, a label id above 4, or a null probs / labels /
 * loss_out with batch > 0; batch == 0 does nothing.  Deterministic: no atomics; repeated calls, and host vs device
 * pointers, give identical bits. */
int dcb_alignment_loss_grad(dcb_engine* e, const float* probs, const uint8_t* labels, int32_t batch, int32_t L,
                            double del_cost, double loss_reg, int32_t band_width, uint32_t flags, float* loss_out,
                            float* grad_out, float* matches_out, float* ms_out);

/* The distillation term of a distilled student's loss: DistillationLoss.call (losses_and_metrics.py:1170-1213), which
 * the distillation loop's eval step adds to the student's AlignmentLoss (model_distillation.py:242-270,320-349:
 * per example student_alpha * AlignmentLoss + distill_alpha * DistillationLoss).  For a batch of B windows of length
 * L <= 256, teacher_logits / student_logits float32 [B, L, 5]:
 *   t = softmax(teacher / T), s = softmax(student / T) over the 5 classes (tf.nn.softmax: divide by T, subtract the
 *   max, exp, sum, divide), then per position the Keras logit loss with the teacher as y_true --
 *     DCB_LOGIT_LOSS_MSE  mean_squared_error: mean_c (s_c - t_c)^2 (the transformer_learn_values_distill default,
 *                         model_configs.py:150-190)
 *     DCB_LOGIT_LOSS_KL   kl_divergence: both clipped to [1e-7, 1], sum_c t_c * log(t_c / s_c) (DistillationLoss's
 *                         own default)
 *   and loss_out[b] = the mean over all L positions, padding included.  float32 throughout.
 * Both logits arrays are host arrays, or with DCB_ROWS_ON_DEVICE device arrays (e.g. the DCB_OUT_ON_DEVICE logits_out of
 * two engines on the same device, a teacher and a student, once both forwards have been waited for).  loss_out is a
 * host array; ms_out (nullable) receives the kernel's device time.  DCB_ERR_INVALID for batch < 0, L outside 1..256, a
 * temperature that is not finite and > 0 (in float32), an unknown logit-loss id, or a null pointer with batch > 0;
 * batch == 0 does nothing.  Deterministic: repeated calls, and host vs device inputs, give identical bits. */
#define DCB_LOGIT_LOSS_MSE 0
#define DCB_LOGIT_LOSS_KL 1
int dcb_distill_loss(dcb_engine* e, const float* teacher_logits, const float* student_logits, int32_t batch,
                     int32_t L, double temperature, int32_t logit_loss, uint32_t flags, float* loss_out,
                     float* ms_out);

/* The distillation term with its gradient, for training a student (model_distillation.py:281-318, whose tape holds the
 * teacher's logits constant):
 *   loss_out [B]          the loss, bitwise equal to dcb_distill_loss's loss_out on the same arguments
 *   grad_out [B, L, 5]    d loss[b] / d student_logits[b] (nullable), float32, with TensorFlow's gradient semantics:
 *                         per position the logit loss's gradient with respect to s -- MSE 2 (s_c - t_c) / 5, KL
 *                         -t'_c / s'_c (t', s' clipped to [1e-7, 1]; 0 where s_c lies outside [1e-7, 1], as
 *                         clip_by_value passes at its bounds and blocks outside them) -- times 1 / L (the mean over
 *                         the window), then the softmax backward (g_c - sum_c' g_c' s_c') s_c and the division by T
 * Arguments and checks as dcb_distill_loss.  Inputs are host arrays, or device arrays with DCB_ROWS_ON_DEVICE; outputs
 * are host arrays, or device arrays with DCB_OUT_ON_DEVICE.  ms_out (nullable) receives the kernel's device time.
 * Returns once the work on the engine's stream has finished.  Deterministic: no atomics; repeated calls, and host vs
 * device pointers, give identical bits. */
int dcb_distill_loss_grad(dcb_engine* e, const float* teacher_logits, const float* student_logits, int32_t batch,
                          int32_t L, double temperature, int32_t logit_loss, uint32_t flags, float* loss_out,
                          float* grad_out, float* ms_out);

/* ---- feature construction from BAM (host C++, htslib-free, needs no GPU) -----------------------------------------------
 * What `deepconsensus run` does in front of the model: stream the subreads-to-CCS BAM ZMW by ZMW (SubreadGrouper,
 * pre_lib.py:50-91), expand / clip / indent every subread (expand_clip_indent with trim_insertions, :1061-1239), fetch
 * the CCS read (:966-998,1322-1330), space all reads out (space_out_subreads, :1242-1276), cut windows of max_length
 * columns (DcExample.iter_examples, :625-697) and lay the feature rows out (extract_features, :704-744) -- as float32
 * rows and / or directly as packed rows.  Errors: negative return code, message from dcb_prep_last_error(). */
typedef struct dcb_prep dcb_prep;
typedef struct dcb_zmw_info {
  int32_t n_windows;          /* windows of this ZMW (examples without any CCS position are dropped, as the reference does) */
  int32_t n_subreads;         /* mapped subreads in the BAM (the first max_passes are used) */
  const char* name;           /* CCS read name = reference name of the subread alignments; valid until the next call */
  int32_t has_ec, has_np, has_rq;
  float ec, rq;               /* aux tags of the CCS read (construct_ccs_read) */
  int32_t np_num_passes;
  const char* rg;             /* RG tag or NULL */
  int32_t ccs_length, spaced_width;
} dcb_zmw_info;
int dcb_prep_open(const char* subreads_to_ccs_bam, const char* ccs_bam, int32_t max_passes, int32_t max_length,
                  int32_t use_ccs_bq, int32_t ins_trim, dcb_prep** out);
/* Process ZMWs on n_threads worker threads plus one BAM-decoding thread (results still come out in file order); call
 * before the first dcb_prep_next_zmw.  n_threads <= 0: everything on the calling thread. */
int dcb_prep_set_threads(dcb_prep* p, int32_t n_threads);
int dcb_prep_next_zmw(dcb_prep* p, dcb_zmw_info* info);   /* 1 = a ZMW is loaded, 0 = end of file, < 0 = error */
/* The windows of the loaded ZMW; every output may be NULL.  rows float32 [n, R, L]; packed [n, dcb_packed_window_bytes];
 * window_pos / num_passes int32 [n]; overflow u8 [n]; ccs_bq int16 [n, L] (-1 at gaps and padding). */
int dcb_prep_get_windows(dcb_prep* p, float* rows, uint8_t* packed, int32_t* window_pos, uint8_t* overflow,
                         int16_t* ccs_bq, int32_t* num_passes);
/* CCS smart windows (`deepconsensus run --use_ccs_smart_windows`, pre_lib.py:625-650,1329-1331): enabled before the first
 * dcb_prep_next_zmw, each ZMW's windows are cut at the widths of its CCS record's `wl` tag (B array, any integer
 * subtype) instead of every max_length columns.  Window j takes wl[j] CCS bases plus the gap columns before the last of
 * them; an entry of 0 gives no window.  A window at most max_length wide is padded like the last fixed-width window; a
 * wider one is an overflow window (overflow = 1): it is never scored, its rows / packed rows / ccs_bq hold only its
 * first max_length columns, and dcb_prep_get_overflow_ccs hands out its CCS at full width.  dcb_prep_next_zmw fails
 * with DCB_ERR_INVALID naming the ZMW on a missing or non-integer wl tag, a negative entry, or sum(wl) != CCS length
 * (where the reference raises), and on an overflow window in a CCS read without any non-zero base quality (the
 * reference slices the unspaced quality array by spaced columns there, and its output goes out of step).  In raw-record
 * mode the tag is checked the same way and handed out by dcb_prep_get_window_lengths (for dcb_features_layout_smart).
 * dcb_prep_get_window_widths: spaced width of every window, int32 [n_windows] (with fixed-width windows, the columns
 * before the padding).
 * dcb_prep_get_overflow_ccs: the CCS ids (u8, 0..4 = ' ATCG') and base qualities (int16, -1 at gap columns) of every
 * overflow window at full width, windows back to back in window order; either output may be NULL. */
int dcb_prep_use_ccs_smart_windows(dcb_prep* p, int32_t enabled);
int dcb_prep_get_window_widths(dcb_prep* p, int32_t* width);
int dcb_prep_get_overflow_ccs(dcb_prep* p, uint8_t* ccs_ids, int16_t* ccs_bq);
/* Raw-record mode with smart windows: the loaded ZMW's `wl` tag; *n always receives its length, wl (nullable) int32 [n]. */
int dcb_prep_get_window_lengths(dcb_prep* p, int32_t* n, int32_t* wl);
/* Raw-record mode, for feature construction on the device (dcb_features_layout below): enabled before the first
 * dcb_prep_next_zmw, the stream decodes and validates each ZMW and keeps its records as they are -- no trimming, spacing
 * or windows (dcb_zmw_info.n_windows and spaced_width are 0, dcb_prep_get_windows is DCB_ERR_STATE), so the worker
 * threads only decode, validate and export.  Every check expand_clip_indent makes (pre_lib.py:1128-1239: implausible
 * cigar / position, cigar vs sequence length, pw / ip length, missing sn tag, pad operations, an aligned part that
 * cannot be located) is made here with the same message, on what trim_insertions (pre_lib.py:1061-1125) would leave of
 * the record; the export also refuses hard clips and reference skips, which subread alignments to a CCS read do not
 * contain.  dcb_prep_get_records writes nothing for a ZMW that failed.
 * dcb_prep_get_records, for the loaded ZMW -- every array may be NULL, so a first call sizes the second:
 *   sizes [DCB_RECORD_SIZES]    subreads, cigar operations, query bases, CCS length, 1 when any CCS quality is non-zero
 *                               (spacing of the qualities only applies then, pre_lib.py:247-250)
 *   read_meta [n][DCB_READ_META] per mapped subread, ALL of them (space_out_subreads runs over every subread before
 *                               extract_features keeps the first max_passes, pre_lib.py:1242-1276,704-744): offset and
 *                               count of its cigar operations, offset and count of its query bases, pos, reverse flag,
 *                               first and one-past-last alignment column (after trimming) that survive the soft clips,
 *                               insertion columns left after trimming, 0.  Offsets are relative to this ZMW's arrays.
 *   read_sn [n][4]              the sn tag
 *   cigar                       u32 per operation, op | len << 4, as stored in the BAM (untrimmed)
 *   bases / pw / ip             per query base, in the BAM's order: base id over ' ATCG' (others 0), and the kinetics
 *                               cast to uint8 as expand_clip_indent does (pre_lib.py:1166-1167)
 *   ccs_bases / ccs_bq          the CCS read's base ids and base qualities */
#define DCB_READ_META 10
#define DCB_RECORD_SIZES 5
int dcb_prep_export_records(dcb_prep* p, int32_t enabled);
int dcb_prep_get_records(dcb_prep* p, int64_t* sizes, int32_t* read_meta, float* read_sn, uint32_t* cigar, uint8_t* bases,
                         uint8_t* pw, uint8_t* ip, uint8_t* ccs_bases, uint8_t* ccs_bq);
/* Training mode (`preprocess` with a truth alignment): dcb_prep_open_truth opens the truth alignment to the CCS reads
 * and its index (path + ".bai"), before the first dcb_prep_next_zmw.  Every ZMW then fetches, on the stream's decoding
 * side, what next(truth_to_ccs.fetch(ccs_name)) gives (pre_lib.py:1001-1014): the first record of the reference named
 * after the CCS read.  dcb_prep_get_label hands it out for the loaded ZMW; info [DCB_LABEL_INFO] is always written:
 *   status (DCB_LABEL_*), cigar operations, bases, pos (the indent), ccs0 (CCS index of the first cigar column),
 *   leading and trailing soft clip lengths, flag
 * and with DCB_LABEL_FOUND cigar u32 [n] / bases u8 [n] (nullable) receive what expand_clip_indent keeps of the record
 * (pre_lib.py:1128-1239, no ins_trim): hard clips dropped, and with any soft clip the soft clips and the deletions
 * between them and the aligned bases removed, so the cigar holds M / I / D / = / X only; bases are ids 1..4 over
 * ' ATCG'.  An unmapped record, reference skips, pads, inner soft clips, a cigar that disagrees with the sequence or a
 * base outside ACGT is DCB_ERR_INVALID naming the ZMW (the reference leaves such label entries uninitialised). */
#define DCB_LABEL_FOUND 0
#define DCB_LABEL_NOT_FOUND 1
#define DCB_LABEL_SUPPLEMENTARY 2
#define DCB_LABEL_INFO 8
int dcb_prep_open_truth(dcb_prep* p, const char* truth_to_ccs_bam);
int dcb_prep_get_label(dcb_prep* p, int32_t* info, uint32_t* cigar, uint8_t* bases);
const char* dcb_prep_ccs_header(dcb_prep* p);             /* SAM header text of the CCS BAM */
void dcb_prep_close(dcb_prep* p);
const char* dcb_prep_last_error(void);
/* Unaligned BAM output as quick_inference.py:742-760,892-897 writes it (flag 4, mapq 255, tags ec:f np:i rq:f RG:Z zm:i). */
typedef struct dcb_bamw dcb_bamw;
int dcb_bamw_open(const char* path, const char* header_text, dcb_bamw** out);
int dcb_bamw_write(dcb_bamw* w, const char* name, const uint8_t* seq, const uint8_t* qual_phred33, int32_t len,
                   int32_t has_ec, float ec, int32_t np_num_passes, float rq, const char* rg);
int dcb_bamw_close(dcb_bamw* w);

/* ---- feature construction on the device ---------------------------------------------------------------------------------
 * trim_insertions, expand_clip_indent, space_out_subreads, the window cut and the packed rows (pre_lib.py:1061-1276,
 * 625-744) from the records of a batch of ZMWs, in two phases so that rows are only laid out for the windows the model
 * will score.  dcb_records is dcb_prep_get_records' arrays of n_zmw ZMWs concatenated (host pointers): read_meta's
 * offsets made relative to the concatenated cigar / base arrays, ZMW z owning reads [zmw_read_off[z],
 * zmw_read_off[z + 1]) and CCS bases [zmw_ccs_off[z], zmw_ccs_off[z + 1]).  Records must come from
 * dcb_prep_get_records or hold what it guarantees; the engine checks every offset and sizes its scratch from read_meta,
 * and a cigar that disagrees with its read_meta ends in DCB_ERR_INVALID.
 *
 * dcb_features_layout (phase A) spaces the batch and returns, dense over the batch and ZMW by ZMW, exactly what
 * dcb_prep_get_windows returns apart from the rows: zmw_windows [n_zmw] (windows per ZMW; windows without a CCS
 * position are dropped, pre_lib.py:625-697), window_pos / num_passes int32 [n], overflow u8 [n], ccs_bq int16 [n, L]
 * (-1 at gaps and padding), ccs_ids u8 [n, L] (the CCS row, pre_lib.py:739) -- what the skip decision
 * (dcb_skip_mask) and dcb_fill_skipped need.  *n_windows_out receives n; max_windows is the capacity of the per-window
 * arrays, and sum over ZMWs of ceil((max(ccs_len, max_r(pos + col_end - col_begin)) + sum_r insertion columns + 32) / L)
 * always suffices.  The spaced reads stay in engine scratch until the next call; a batch whose spaced reads would
 * exceed 2 GiB is DCB_ERR_INVALID (pass fewer ZMWs), and the engine stays usable after any error.
 *
 * dcb_features_pack (phase B) writes the packed rows (above) of windows[0..n) -- indices into phase A's n windows, any
 * order, repeats allowed -- to packed_out [n, dcb_packed_window_bytes]: a host array, or with DCB_OUT_ON_DEVICE a
 * 16-byte-aligned device array that dcb_forward_packed(..., DCB_ROWS_ON_DEVICE) reads in place.  Byte for byte the
 * `packed` of dcb_prep_get_windows.  ms_out (nullable): device time of the kernels.  Deterministic, no atomics. */
typedef struct dcb_records {
  int32_t n_zmw, n_cigar, n_query, reserved;
  const int32_t* zmw_read_off;     /* [n_zmw + 1] */
  const int32_t* zmw_ccs_off;      /* [n_zmw + 1] */
  const int32_t* zmw_ccs_bq_any;   /* [n_zmw] */
  const int32_t* read_meta;        /* [n_reads, DCB_READ_META] */
  const float* read_sn;            /* [n_reads, 4] */
  const uint32_t* cigar;           /* [n_cigar] */
  const uint8_t *bases, *pw, *ip;  /* [n_query] */
  const uint8_t *ccs_bases, *ccs_bq;
} dcb_records;
int dcb_features_layout(dcb_engine* e, const dcb_records* rec, int32_t ins_trim, int32_t max_windows, int32_t* zmw_windows,
                        int32_t* window_pos, uint8_t* overflow, int16_t* ccs_bq, int32_t* num_passes, uint8_t* ccs_ids,
                        int32_t* n_windows_out, float* ms_out);
int dcb_features_pack(dcb_engine* e, const int32_t* windows, int32_t n, uint32_t flags, uint8_t* packed_out, float* ms_out);
/* CCS smart windows on the device (`run --use_ccs_smart_windows --features gpu`): dcb_features_layout with each ZMW's
 * windows cut at its `wl` tag (wl: host int32, ZMW z's lengths at wl[wl_off[z] .. wl_off[z + 1]), wl_off [n_zmw + 1]
 * starting at 0) as dcb_prep_use_ccs_smart_windows cuts them on the host: window j holds CCS bases [S, S + wl[j]), S the
 * sum of the lengths before it, with the gap columns in front of the last of them; a length of 0 gives no window.
 * window_width int32 [n] receives every window's spaced width, overflow = width > L.  ccs_bq / ccs_ids and the packed
 * rows of dcb_features_pack hold a window's first min(width, L) columns and padding after them.  Negative lengths,
 * lengths that do not sum to the CCS length, or an overflow window in a CCS read without base qualities return
 * DCB_ERR_INVALID and leave no layout; the engine stays usable.
 * dcb_features_ccs: the CCS ids (0..4) and base qualities (-1 at gap columns) of the layout's windows[0..n) at full
 * width, window i at off[i] .. off[i + 1] of ccs_ids / ccs_bq (host arrays; off [n + 1] starts at 0 and must follow the
 * windows' widths) -- what an overflow window adopts.  ms_out (nullable): device time of the kernel. */
int dcb_features_layout_smart(dcb_engine* e, const dcb_records* rec, const int32_t* wl_off, const int32_t* wl, int32_t ins_trim,
                              int32_t max_windows, int32_t* zmw_windows, int32_t* window_pos, uint8_t* overflow,
                              int32_t* window_width, int16_t* ccs_bq, int32_t* num_passes, uint8_t* ccs_ids,
                              int32_t* n_windows_out, float* ms_out);
int dcb_features_ccs(dcb_engine* e, const int32_t* windows, int32_t n, const int64_t* off, uint8_t* ccs_ids, int16_t* ccs_bq,
                     float* ms_out);
/* Training labels on the device, after dcb_features_layout on the same batch: labels holds one label per ZMW of that
 * batch (host arrays; label_meta [n_zmw, DCB_LABEL_META] = cigar offset, cigar count, base offset, base count, pos,
 * ccs0 of dcb_prep_get_label, offsets relative to the concatenated cigar / bases, the cigar ranges in ZMW order and
 * disjoint; a label with no operations is all gaps).  labels_out u8 [n, L] receives the label row of windows[0..n) over ' ATCG' as bases_encoded gives it
 * (pre_lib.py:652-697): the label columns whose CCS index lies in the window's inclusive CCS bounds and everything
 * between them, padded with gaps to L; longer than L, its gaps removed (status 1, n_examples_adjusted_label); still
 * longer, a row of gaps (status 2, n_examples_label_overflow: the window is dropped).  status_out u8 [n]: 0 kept,
 * 1 adjusted, 2 overflow.  ccs_width_out (nullable) int32 [n_zmw]: DcExample.ccs_width of every ZMW of the layout
 * (its spaced CCS read without trailing gaps), which iter_examples' window count follows.  Labels the engine cannot index, operations other than M / I / D / = / X, a cigar that
 * disagrees with its base count or base ids outside 1..4 are DCB_ERR_INVALID; the engine and the layout stay usable.
 * ms_out (nullable): device time of the kernels.  Deterministic, no atomics. */
#define DCB_LABEL_META 6
typedef struct dcb_labels {
  int32_t n_zmw, n_cigar, n_bases, reserved;
  const int32_t* label_meta;       /* [n_zmw, DCB_LABEL_META] */
  const uint32_t* cigar;           /* [n_cigar] */
  const uint8_t* bases;            /* [n_bases] */
} dcb_labels;
int dcb_features_labels(dcb_engine* e, const dcb_labels* labels, const int32_t* windows, int32_t n, uint8_t* labels_out,
                        uint8_t* status_out, int32_t* ccs_width_out, float* ms_out);

/* Evaluation inputs on the device, after dcb_features_layout on the same batch: the label rows and statuses of every
 * window of the layout (dcb_features_labels' rows, from the same `labels`), then the kept windows -- label status != 2
 * and keep_zmw[z] != 0 for their ZMW (host u8 [n_keep], n_keep the layout's ZMW count) -- compacted in ZMW and window
 * order by a block scan (no atomics), and for each of them, in that order, written to caller-given device arrays:
 *   packed_out [k, dcb_packed_window_bytes]  16-byte aligned, the packed rows dcb_forward_packed(..., DCB_ROWS_ON_DEVICE)
 *                                            reads in place -- byte for byte dcb_features_pack's
 *   labels_out u8 [k, L], ccs_out u8 [k, L]  label rows and CCS rows (the layout's ccs_ids), which dcb_evaluate reads in
 *                                            place with DCB_LABELS_ON_DEVICE
 * capacity is the room of these arrays in windows.  Host outputs: *k_out, k (written even when it exceeds capacity);
 * status_out u8 [n] (nullable) the status of every window of the layout (0 kept, 1 adjusted, 2 overflow);
 * ccs_width_out int32 [n_zmw] (nullable) as dcb_features_labels; windows_out int32 [capacity] (nullable) the layout
 * index of every kept window.  DCB_ERR_INVALID for k > capacity (nothing beyond capacity is written), a keep mask of
 * another length, and every label dcb_features_labels refuses; the engine and the layout stay usable.  ms_out
 * (nullable): device time of the kernels.  Deterministic. */
int dcb_features_eval(dcb_engine* e, const dcb_labels* labels, const uint8_t* keep_zmw, int32_t n_keep, int32_t capacity,
                      uint8_t* packed_out, uint8_t* labels_out, uint8_t* ccs_out, uint8_t* status_out, int32_t* ccs_width_out,
                      int32_t* windows_out, int32_t* k_out, float* ms_out);

/* ---- base-quality calibration (calculate_baseq_calibration.py) ----------------------------------------------------------
 * Per predicted quality, how many bases of reads aligned to a truth assembly match it and how many do not.
 *
 * The reader (host C++, needs no GPU).  dcb_calib_open opens a coordinate-sorted BAM with its index (path + ".bai"; a
 * missing index is DCB_ERR_INVALID) and a plain FASTA file, through its .fai when there is one, else an index built in
 * memory (a compressed FASTA is refused).  n_threads >= 1 threads decode and validate each batch.
 * dcb_calib_contigs: "name\tlength\n" per contig of the BAM header (fasta = 0) or of the FASTA file (fasta = 1).
 * dcb_calib_fetch_reference: the FASTA bases [start, stop) of a contig as the file holds them, clipped at its end;
 * *n receives their count, out (nullable) needs stop - start bytes.
 * dcb_calib_query starts a fetch of [start, stop) on a contig: what AlignmentFile.fetch returns (htslib's overlap
 * test, pos < stop and bam_endpos > start), minus records with pos < min_pos, duplicate, qcfail, secondary, unmapped or
 * supplementary records, and records with mapping quality < min_mapq.  dcb_calib_next_batch reads on until the batch
 * holds at least max_bases bases (or the fetch ends): returns 1 with sizes [3] = reads, cigar operations, bases, or 0
 * when nothing is left; a record without SEQ or QUAL, or whose cigar disagrees with its SEQ, is DCB_ERR_INVALID naming
 * it.  dcb_calib_get_batch copies the batch out (every array nullable): read_meta int32 [reads, DCB_CALIB_META] = pos,
 * endpos, cigar offset, cigar count, base offset, base count; cigar [operations] as the BAM stores it; seq [bases] the
 * 4-bit codes of "=ACMGRSVTWYHKDBN"; qual [bases] Phred values.  dcb_calib_read_name: the name of read i of the batch.
 * Errors: dcb_prep_last_error.
 *
 * The count (engine, sm_90a): dcb_calib_count walks every read of a batch on the device and returns in counts int64
 * [100][2] how many (match, mismatch) events each quality bin received over every interval of the regions on the
 * contig -- each region [start, stop] cut into intervals [s, min(stop, s + interval_length)], both ends inclusive, each
 * counting the reads it fetches.  failure int64 [3] receives (read index, reference position, DCB_CALIB_*) of the
 * lowest read of the batch that has a counted event the reference would fail on, or (-1, 0, 0): a base past the
 * contig's end, a quality whose bin lies outside [-100, 100), or (DCB_CALIB_BAD_INPUT) bases the call was not given.
 * ref_bases (host) are the contig's bases [ref_start, ref_start + ref_count); NULL keeps the previous call's, which
 * must then have the same ref_start and ref_count.  ms_out (nullable): device time of the kernels.  The counts are sums
 * of integers, so they do not depend on the order of the work; there are no global atomics. */
#define DCB_CALIB_META 6
#define DCB_CALIB_PAST_CONTIG 1
#define DCB_CALIB_BAD_QUALITY 2
#define DCB_CALIB_BAD_INPUT 3
typedef struct dcb_calib dcb_calib;
int dcb_calib_open(const char* bam, const char* fasta, int32_t n_threads, dcb_calib** out);
const char* dcb_calib_contigs(dcb_calib* p, int32_t fasta);
int dcb_calib_fetch_reference(dcb_calib* p, const char* contig, int64_t start, int64_t stop, uint8_t* out, int64_t* n);
int dcb_calib_query(dcb_calib* p, const char* contig, int64_t start, int64_t stop, int64_t min_pos, int32_t min_mapq);
int dcb_calib_next_batch(dcb_calib* p, int64_t max_bases, int64_t* sizes);
int dcb_calib_get_batch(dcb_calib* p, int32_t* read_meta, uint32_t* cigar, uint8_t* seq, uint8_t* qual);
const char* dcb_calib_read_name(dcb_calib* p, int64_t i);
void dcb_calib_close(dcb_calib* p);
typedef struct dcb_calib_input {
  int32_t n_reads, n_regions;
  int64_t n_cigar, n_bases;
  const int32_t* read_meta;        /* [n_reads, DCB_CALIB_META] */
  const uint32_t* cigar;           /* [n_cigar] */
  const uint8_t *seq, *qual;       /* [n_bases] */
  const int64_t* regions;          /* [n_regions, 2]: start, stop */
  int64_t interval_length;         /* > 0 */
  const uint8_t* ref_bases;        /* [ref_count] or NULL */
  int64_t ref_start, ref_count, contig_length;
  int32_t calibration_enabled, reserved;
  double threshold, w, b;          /* calibrate_quality_scores' threshold, w, b */
} dcb_calib_input;
int dcb_calib_count(dcb_engine* e, const dcb_calib_input* in, int64_t* counts, int64_t* failure, float* ms_out);

/* ---- read identity (read_yield.py) --------------------------------------------------------------------------------------
 * dcb_read_identity walks every read of a batch from dcb_calib_get_batch against the truth assembly on the device and
 * returns per read, in counts int64 [n_reads][5]: matches, mismatches, insertions, deletions and soft-clipped bases.
 * An M, = or X base is a match when it equals the upper-cased reference base and both are A, C, G or T, else a
 * mismatch; I, D and S count their lengths; H and P count nothing.  avg_q [n_reads] receives avg_phred of the read's
 * qualities (float64, an exact histogram times the engine's 10^(-q/10) table from the host's libm pow), and status
 * [n_reads] one DCB_IDENTITY_* code:
 *   OK          the counts are valid;
 *   PAST_CONTIG the read has a reference base at or past contig_length: it is not counted (counts 0);
 *   SKIP_OP     the cigar has an N operation, which has no meaning for identity (counts 0);
 *   BORDERLINE  as OK, but avg_q lies within 1e-7 of q - 5e-6 for an integer q, where round(avg_q, 5) >= q turns: the
 *               caller re-decides the quality filter with NumPy's own sum;
 *   BAD_INPUT   ref_bases do not cover one of the read's bases inside the contig (counts 0).
 * ref_bases (host) are the contig's bases [ref_start, ref_start + ref_count).  ms_out (nullable): device time of the
 * kernel.  The results do not depend on how the reads are split into batches; there are no global atomics. */
#define DCB_IDENTITY_COUNTS 5
#define DCB_IDENTITY_OK 0
#define DCB_IDENTITY_PAST_CONTIG 1
#define DCB_IDENTITY_SKIP_OP 2
#define DCB_IDENTITY_BORDERLINE 3
#define DCB_IDENTITY_BAD_INPUT 4
typedef struct dcb_identity_input {
  int32_t n_reads, reserved;
  int64_t n_cigar, n_bases;
  const int32_t* read_meta;        /* [n_reads, DCB_CALIB_META] */
  const uint32_t* cigar;           /* [n_cigar] */
  const uint8_t *seq, *qual;       /* [n_bases] */
  const uint8_t* ref_bases;        /* [ref_count] */
  int64_t ref_start, ref_count, contig_length;
} dcb_identity_input;
int dcb_read_identity(dcb_engine* e, const dcb_identity_input* in, int64_t* counts, double* avg_q, int32_t* status,
                      float* ms_out);

/* ---- read errors (read_yield.py --error_profile) ---------------------------------------------------------------------
 * dcb_read_errors walks the same batch as dcb_read_identity and returns per read, in errors int64
 * [n_reads][DCB_ERRORS_COLS], its errors by type and homopolymer length: six tables of DCB_ERRORS_BINS bins h = 0..20
 * at the DCB_ERRORS_* column offsets, then the 5 x 5 substitution matrix (rows the truth class, columns the read
 * class, in the order A, C, G, T, other).
 *   hp(r)         the length of the maximal run of one base of A, C, G, T (upper-cased first) that holds truth
 *                 position r, measured over the whole contig; 0 for any other byte, which breaks runs.  h = min(hp, 20).
 *   substitutions an M, = or X base that dcb_read_identity counts as a mismatch at r: 1 in SUB[hp(r)] and in
 *                 MATRIX[truth class][read class of the 4-bit SEQ code].
 *   deletions     a D of n bases at [r, r + n): 1 in DEL_EVENTS[h], n in DEL_BASES[h], h = hp(r) when the n truth
 *                 bases are one base of A, C, G, T, else 0.
 *   insertions    an I of n bases where the walk has reached r: 1 in INS_EVENTS[h], n in INS_BASES[h].  When the n
 *                 bases are one base b of A, C, G, T: h = hp(r - 1) if r >= 1 and truth[r - 1] is b, else hp(r) if
 *                 r < contig_length and truth[r] is b; otherwise h = 0.
 *   runs          RUNS[h]: the maximal runs that lie inside the read's truth span [pos, endpos); RUNS[0] is 0.
 * Adjacent I (or D) operations are separate events; S, H and P count nothing.  A read that dcb_read_identity gives
 * PAST_CONTIG, SKIP_OP or BAD_INPUT has a zero row.  ref_bases must hold, for every read, [max(pos - 1, 0),
 * min(endpos + 1, contig_length)) and the whole runs at both ends of the slice (the kernel takes the slice's edges
 * as run ends); a batch whose slice does not reach that far is refused.  ms_out (nullable): device time of the
 * kernels.  The results do not depend on how the reads are split into batches; there are no global atomics. */
#define DCB_ERRORS_BINS 21
#define DCB_ERRORS_SUB 0
#define DCB_ERRORS_INS_EVENTS 21
#define DCB_ERRORS_INS_BASES 42
#define DCB_ERRORS_DEL_EVENTS 63
#define DCB_ERRORS_DEL_BASES 84
#define DCB_ERRORS_RUNS 105
#define DCB_ERRORS_MATRIX 126
#define DCB_ERRORS_COLS 151
int dcb_read_errors(dcb_engine* e, const dcb_identity_input* in, int64_t* errors, float* ms_out);

/* ---- k-mer QV (kmer_qv.py) -----------------------------------------------------------------------------------------
 * A sequential reader of FASTA, FASTQ or BAM files (the format comes from the content; text may be plain or gzip):
 * dcb_seq_next_batch reads whole records until the batch holds at least max_bases bases (at least one record), sets
 * sizes[0] = reads and sizes[1] = bases, and returns 1, or 0 at the end of the file (< 0: error, dcb_prep_last_error;
 * a gzip stream that is corrupt or ends early is an error, naming the file).
 * dcb_seq_get_batch copies out the concatenated upper-cased bases [n_bases], the Phred qualities [n_bases] (0 where a
 * read has none), the offsets [n_reads + 1] and has_qual [n_reads] (0 for FASTA records and BAM QUAL 0xFF).  A BAM is
 * read in file order without an index; its secondary (0x100) and supplementary (0x800) records are skipped, and a
 * record without SEQ is refused.  FASTA records may span lines. */
typedef struct dcb_seq_reader dcb_seq_reader;
int dcb_seq_open(const char* path, dcb_seq_reader** out);
int dcb_seq_next_batch(dcb_seq_reader* r, int64_t max_bases, int64_t* sizes);
int dcb_seq_get_batch(dcb_seq_reader* r, uint8_t* bases, uint8_t* qual, int64_t* offsets, uint8_t* has_qual);
const char* dcb_seq_read_name(dcb_seq_reader* r, int64_t i);
void dcb_seq_close(dcb_seq_reader* r);

/* The engine's k-mer table: an open-addressing table of canonical k-mer codes (2 bits per base, A=0 C=1 G=2 T=3, first
 * base most significant; canonical = the smaller of the k-mer's and its reverse complement's code) with a uint32 count
 * per key.  A key's slot is the low bits of splitmix64's finalizer of the key, probed linearly; the key belongs to
 * partition (mix >> 32) % n_partitions.  Any byte other than A, C, G or T breaks the k-mers that contain it.
 *   dcb_kmer_table_init   allocates capacity slots, the largest power of two that fits table_bytes (12 bytes a slot;
 *                         table_bytes <= 0: half the device's free memory), for 1 <= k <= 31.
 *   dcb_kmer_table_clear  empties it for the keys of one partition.
 *   dcb_kmer_count        counts every k-mer of the batch's reads that belongs to the partition (both strands to one
 *                         key; counts saturate near 2^32).  When the number of distinct keys exceeds 0.8 x capacity the
 *                         table stops accepting keys and reports overflow in dcb_kmer_table_stats: the caller repeats
 *                         the work with more partitions.
 *   dcb_kmer_query        per read of the batch: the k-mer positions of the partition (counts[2r]) and how many of
 *                         them have a count below min_count (counts[2r + 1]).  With with_quality, also avg_phred of the
 *                         read's qualities (the engine's 10^(-q/10) table, as dcb_read_identity) in avg_q[r] and
 *                         borderline[r] = 1 where it lies within 1e-7 of q - 5e-6 for an integer q; reads without
 *                         qualities get avg_q 0.
 * dcb_kmer_count and dcb_kmer_query enqueue their work on pipeline slot 0 or 1 and return; dcb_kmer_wait waits for
 * the slot's work, writes its query outputs (host arrays of the batch's n_reads; NULL for a count) and its device time.
 * Two slots may be in flight at once, so the host reads the next batch while the device works on the last.
 * dcb_kmer_table_stats (after a wait): stats[DCB_KMER_STATS] = capacity, distinct keys claimed, overflow, k-mers
 * counted, their probe steps, k-mers queried, their probe steps; histogram[DCB_KMER_HIST + 1]: [c] = keys with count
 * c for c = 1..255, [256] = keys with count >= 256.  Every output is an integer, so none depends on the batch split,
 * the insertion order or the number of partitions. */
#define DCB_KMER_STATS 7
#define DCB_KMER_HIST 256
typedef struct dcb_kmer_batch {
  int32_t n_reads, reserved;
  int64_t n_bases;
  const uint8_t* bases;            /* [n_bases] */
  const uint8_t* qual;             /* [n_bases] Phred; dcb_kmer_query with with_quality only */
  const int64_t* offsets;          /* [n_reads + 1], offsets[0] = 0 */
  const uint8_t* has_qual;         /* [n_reads]; dcb_kmer_query with with_quality only */
} dcb_kmer_batch;
int dcb_kmer_table_init(dcb_engine* e, int64_t table_bytes, int32_t k, int64_t* capacity);
int dcb_kmer_table_clear(dcb_engine* e, int32_t partition, int32_t n_partitions);
int dcb_kmer_count(dcb_engine* e, const dcb_kmer_batch* b, int32_t slot);
int dcb_kmer_query(dcb_engine* e, const dcb_kmer_batch* b, int32_t min_count, int32_t with_quality, int32_t slot);
int dcb_kmer_wait(dcb_engine* e, int32_t slot, int64_t* counts, double* avg_q, int32_t* borderline, float* ms_out);
int dcb_kmer_table_stats(dcb_engine* e, int64_t* stats, int64_t* histogram);

/* The copy-number spectrum (`kmer_qv --spectrum`): a second table, the set table, counts the evaluated reads' own
 * k-mers with the table's layout, slot and partition rule and k, and a scan bins every distinct key of one partition
 * by its count in both tables.
 *   dcb_kmer_set_init   allocates the set table as dcb_kmer_table_init sizes the table (after dcb_kmer_table_init).
 *   dcb_kmer_set_clear  empties it for the keys of one partition.
 *   dcb_kmer_set_count  counts the k-mers of the partition of the reads r with keep[r] != 0 (host [n_reads]) into the
 *                       set table, as dcb_kmer_count counts.  It reuses the bases and offsets that the last
 *                       dcb_kmer_query (or dcb_kmer_count) on the same slot staged; b must be that batch, and only its
 *                       sizes are checked.  It overflows as the table does.  Waited on with dcb_kmer_wait, which writes
 *                       nothing but the device time.
 *   dcb_kmer_spectrum   (both tables holding the same partition) matrix[c * DCB_KMER_SPECTRUM_BINS + m] = distinct
 *                       keys of the partition with table count min(c, 256) and set count min(m, 256): the set's keys
 *                       for m >= 1, the table's keys the set lacks in column 0; [0][0] is 0.  stats
 *                       [DCB_KMER_SPECTRUM_STATS] = the set table's capacity, distinct keys claimed, overflow, k-mers
 *                       counted, their probe steps.  Exact integers, whatever the thread order: the host sums the
 *                       partitions. */
#define DCB_KMER_SPECTRUM_BINS 257
#define DCB_KMER_SPECTRUM_STATS 5
int dcb_kmer_set_init(dcb_engine* e, int64_t table_bytes, int64_t* capacity);
int dcb_kmer_set_clear(dcb_engine* e, int32_t partition, int32_t n_partitions);
int dcb_kmer_set_count(dcb_engine* e, const dcb_kmer_batch* b, const uint8_t* keep, int32_t slot);
int dcb_kmer_spectrum(dcb_engine* e, int64_t* matrix, int64_t* stats);

/* Device time of the last dcb_forward (milliseconds, CUDA events on the engine's stream). */
int dcb_last_forward_ms(dcb_engine* e, float* ms);
/* Number of engine kernels launched by the last dcb_forward. */
int dcb_last_forward_launches(dcb_engine* e, int32_t* n);

/* Per-kernel timing of the dominant stage (the FFN GEMMs): when enabled, every launch is bracketed by CUDA events on the
 * engine's stream; dcb_get_profile returns the FFN stages' accumulated device time, count and tokens processed since
 * dcb_set_profile. */
int dcb_set_profile(dcb_engine* e, int32_t enabled);
int dcb_get_profile(dcb_engine* e, float* ffn_ms_total, int32_t* ffn_launches, int64_t* ffn_tokens);
/* Device time (ms) and launch count per kernel class since dcb_set_profile: [0] embed, [1] row GEMM
 * (condenser / out-projection), [2] QKV GEMM, [3] attention, [4] FFN, [5] head. */
int dcb_get_profile_kernels(dcb_engine* e, float* ms6, int32_t* n6);

/* Pinned host memory helpers (for callers that want async H2D/D2H). */
int dcb_alloc_host(size_t bytes, void** out);
int dcb_free_host(void* p);
/* Device memory helpers so a host language can keep inputs resident (bench `value`). */
int dcb_alloc_device(dcb_engine* e, size_t bytes, void** out);
int dcb_free_device(dcb_engine* e, void* p);
int dcb_memcpy_h2d(dcb_engine* e, void* dst_dev, const void* src_host, size_t bytes);
int dcb_memcpy_d2h(dcb_engine* e, void* dst_host, const void* src_dev, size_t bytes);
int dcb_synchronize(dcb_engine* e);

const char* dcb_last_error(const dcb_engine* e); /* e may be NULL: last create() error */
const char* dcb_version(void);
void dcb_destroy(dcb_engine* e);

#ifdef __cplusplus
}
#endif
#endif /* DCB200_H_ */
