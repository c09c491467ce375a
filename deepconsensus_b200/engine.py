"""ctypes binding of the dcb200 C-ABI (include/dcb200.h) and the model object built on it.

`B200Model` stands where the reference's `tf.keras.Model` stands in
`quick_inference.run_model_on_examples` (quick_inference.py:341-415):

  * `model.predict(rows)` -> object with `.numpy()` giving softmax output [B, L, 5]
    (the contract quick_inference.py:368-370 relies on), and
  * `model.forward(rows)` -> base / quality characters straight from the device epilogue
    (what quick_inference.py:377-414 computes on the host).

There is no CPU fallback: if the CUDA library is missing or no sm_90 GPU is present,
construction raises.
"""
from __future__ import annotations

import ctypes
import os
from typing import Any, Callable, Dict, Iterable, Iterator, List, Optional, Tuple

import numpy as np

from deepconsensus_b200 import calibration as calibration_lib
from deepconsensus_b200 import params as params_lib
from deepconsensus_b200 import weights as weights_lib

# DCB200_LIB: developer override to load an experiment build of the same library (never a different implementation)
_LIB_PATH = os.environ.get("DCB200_LIB") or os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc",
                                                         "libdcb200.so")
_lib = None

DCB_ROWS_ON_DEVICE = 1
DCB_OUT_ON_DEVICE = 2
DCB_STRICT_FP32 = 4
DCB_FAST_BF16 = 8
DCB_LABELS_ON_DEVICE = 16
DCB_PRECISION_BF16 = 0
DCB_PRECISION_FP32 = 1
DCB_PRECISION_TF32X3 = 2
# precision name -> dcb_config.precision
PRECISIONS = {"bf16": DCB_PRECISION_BF16, "fp32": DCB_PRECISION_FP32, "tf32x3": DCB_PRECISION_TF32X3}
# per-read outcome codes of dcb_stitch_fastq (the OutcomeCounter field the reference would bump)
DCB_READ_OK, DCB_READ_EMPTY, DCB_READ_ONLY_GAPS, DCB_READ_LOW_QUALITY, DCB_READ_TOO_SHORT = 0, 1, 2, 3, 4
DCB_READ_BORDERLINE = 0x80
DCB_BAND_WIDTH_NONE = -1
# dcb_calib_count: per-read meta columns, quality bins, and the kinds of failure it reports
CALIB_META, CALIB_BINS = 6, 100
DCB_CALIB_PAST_CONTIG, DCB_CALIB_BAD_QUALITY, DCB_CALIB_BAD_INPUT = 1, 2, 3
# dcb_read_identity: per-read counts (matches, mismatches, insertions, deletions, soft clips) and status codes
IDENTITY_COUNTS = 5
(DCB_IDENTITY_OK, DCB_IDENTITY_PAST_CONTIG, DCB_IDENTITY_SKIP_OP, DCB_IDENTITY_BORDERLINE,
 DCB_IDENTITY_BAD_INPUT) = range(5)
# dcb_read_errors: per-read rows of six ERRORS_BINS-bin tables at these column offsets, then the 5 x 5 substitution matrix
ERRORS_BINS = 21
(ERRORS_SUB, ERRORS_INS_EVENTS, ERRORS_INS_BASES, ERRORS_DEL_EVENTS, ERRORS_DEL_BASES, ERRORS_RUNS,
 ERRORS_MATRIX) = range(0, 7 * ERRORS_BINS, ERRORS_BINS)
ERRORS_COLS = ERRORS_MATRIX + 25
# dcb_kmer_table_stats: its stats entries and the count histogram's last bin (counts >= DCB_KMER_HIST)
KMER_STAT_KEYS = ("capacity", "claimed", "overflow", "count_kmers", "count_probes", "query_kmers", "query_probes")
KMER_HIST = 256
# dcb_kmer_spectrum: its stats entries and the bins of each axis (counts 0..256, 256 meaning >= 256)
KMER_SET_STAT_KEYS = ("capacity", "claimed", "overflow", "count_kmers", "count_probes")
KMER_SPECTRUM_BINS = 257
DCB_LOGIT_LOSS_MSE, DCB_LOGIT_LOSS_KL = 0, 1
# Keras loss identifiers (tf.keras.losses.get) of the two logit losses DistillationLoss is used with
LOGIT_LOSS_IDS = {"mean_squared_error": DCB_LOGIT_LOSS_MSE, "mse": DCB_LOGIT_LOSS_MSE, "MSE": DCB_LOGIT_LOSS_MSE,
                  "kl_divergence": DCB_LOGIT_LOSS_KL, "kullback_leibler_divergence": DCB_LOGIT_LOSS_KL,
                  "kld": DCB_LOGIT_LOSS_KL, "KLD": DCB_LOGIT_LOSS_KL}
# columns of dcb_evaluate's per-window alignment counts (AlignmentMetric.alignment's metric_values)
EVAL_COUNT_KEYS = ("num_matches", "num_insertions", "num_deletions", "num_correct_matches", "alignment_length")


class DcbError(RuntimeError):
  def __init__(self, code: int, message: str):
    super().__init__("dcb200 error %d: %s" % (code, message))
    self.code = code


class DcbConfig(ctypes.Structure):
  _fields_ = [
      ("struct_size", ctypes.c_int32), ("device", ctypes.c_int32),
      ("max_passes", ctypes.c_int32), ("max_length", ctypes.c_int32),
      ("use_ccs_bq", ctypes.c_int32),
      ("hidden_size", ctypes.c_int32), ("num_heads", ctypes.c_int32),
      ("num_hidden_layers", ctypes.c_int32), ("filter_size", ctypes.c_int32),
      ("attn_win_size", ctypes.c_int32), ("rezero", ctypes.c_int32),
      ("add_pos_encoding", ctypes.c_int32), ("condense_transformer_input", ctypes.c_int32),
      ("per_base_hidden_size", ctypes.c_int32), ("pw_hidden_size", ctypes.c_int32),
      ("ip_hidden_size", ctypes.c_int32), ("strand_hidden_size", ctypes.c_int32),
      ("ccs_bq_hidden_size", ctypes.c_int32), ("sn_hidden_size", ctypes.c_int32),
      ("pw_max", ctypes.c_int32), ("ip_max", ctypes.c_int32), ("sn_max", ctypes.c_int32),
      ("ccs_bq_max", ctypes.c_int32), ("strand_max", ctypes.c_int32),
      ("max_base_quality", ctypes.c_int32), ("calibration_enabled", ctypes.c_int32),
      ("calibration_threshold", ctypes.c_double), ("calibration_w", ctypes.c_double),
      ("calibration_b", ctypes.c_double),
      ("max_batch", ctypes.c_int32), ("chunk_tiles", ctypes.c_int32),
      ("precision", ctypes.c_int32),
      ("reserved", ctypes.c_int32 * 5),
  ]


class DcbTensor(ctypes.Structure):
  _fields_ = [("name", ctypes.c_char_p), ("data", ctypes.POINTER(ctypes.c_float)),
              ("ndim", ctypes.c_int32), ("shape", ctypes.c_int64 * 4)]


READ_META = 10   # DCB_READ_META: int32 fields per subread in the raw records


LABEL_META = 6  # DCB_LABEL_META: int32 fields per label in dcb_labels


class DcbLabels(ctypes.Structure):
  """dcb_labels: one training label per ZMW of a dcb_features_layout batch (include/dcb200.h)."""
  _fields_ = [("n_zmw", ctypes.c_int32), ("n_cigar", ctypes.c_int32), ("n_bases", ctypes.c_int32), ("reserved", ctypes.c_int32),
              ("label_meta", ctypes.c_void_p), ("cigar", ctypes.c_void_p), ("bases", ctypes.c_void_p)]


class DcbRecords(ctypes.Structure):
  """dcb_records: the raw records of a batch of ZMWs (include/dcb200.h "feature construction on the device")."""
  _fields_ = [("n_zmw", ctypes.c_int32), ("n_cigar", ctypes.c_int32), ("n_query", ctypes.c_int32), ("reserved", ctypes.c_int32)] + [
      (k, ctypes.c_void_p) for k in ("zmw_read_off", "zmw_ccs_off", "zmw_ccs_bq_any", "read_meta", "read_sn", "cigar", "bases",
                                     "pw", "ip", "ccs_bases", "ccs_bq")]


class DcbCalibInput(ctypes.Structure):
  """dcb_calib_input: one batch of aligned reads and the regions of one contig (include/dcb200.h "base-quality
  calibration")."""
  _fields_ = [("n_reads", ctypes.c_int32), ("n_regions", ctypes.c_int32), ("n_cigar", ctypes.c_int64),
              ("n_bases", ctypes.c_int64), ("read_meta", ctypes.c_void_p), ("cigar", ctypes.c_void_p),
              ("seq", ctypes.c_void_p), ("qual", ctypes.c_void_p), ("regions", ctypes.c_void_p),
              ("interval_length", ctypes.c_int64), ("ref_bases", ctypes.c_void_p), ("ref_start", ctypes.c_int64),
              ("ref_count", ctypes.c_int64), ("contig_length", ctypes.c_int64), ("calibration_enabled", ctypes.c_int32),
              ("reserved", ctypes.c_int32), ("threshold", ctypes.c_double), ("w", ctypes.c_double), ("b", ctypes.c_double)]


class DcbIdentityInput(ctypes.Structure):
  """dcb_identity_input: one batch of aligned reads and the reference bases they cover (include/dcb200.h "read
  identity")."""
  _fields_ = [("n_reads", ctypes.c_int32), ("reserved", ctypes.c_int32), ("n_cigar", ctypes.c_int64),
              ("n_bases", ctypes.c_int64), ("read_meta", ctypes.c_void_p), ("cigar", ctypes.c_void_p),
              ("seq", ctypes.c_void_p), ("qual", ctypes.c_void_p), ("ref_bases", ctypes.c_void_p),
              ("ref_start", ctypes.c_int64), ("ref_count", ctypes.c_int64), ("contig_length", ctypes.c_int64)]


class DcbKmerBatch(ctypes.Structure):
  """dcb_kmer_batch: one batch of concatenated sequences (include/dcb200.h "k-mer QV")."""
  _fields_ = [("n_reads", ctypes.c_int32), ("reserved", ctypes.c_int32), ("n_bases", ctypes.c_int64),
              ("bases", ctypes.c_void_p), ("qual", ctypes.c_void_p), ("offsets", ctypes.c_void_p),
              ("has_qual", ctypes.c_void_p)]


# Every symbol include/dcb200.h declares; tests check the built library exports all of them.
ABI_SYMBOLS = (
    "dcb_create", "dcb_load_weights", "dcb_forward", "dcb_submit", "dcb_wait", "dcb_stitch", "dcb_last_forward_ms",
    "dcb_packed_window_bytes", "dcb_pack_rows", "dcb_forward_packed", "dcb_submit_packed",
    "dcb_stitch_fastq", "dcb_skip_mask", "dcb_fill_skipped", "dcb_stitch_ragged", "dcb_stitch_fastq_ragged",
    "dcb_fill_skipped_ragged", "dcb_evaluate", "dcb_evaluate_calibration", "dcb_distill_loss",
    "dcb_alignment_loss_grad", "dcb_distill_loss_grad", "dcb_prep_open", "dcb_prep_set_threads", "dcb_prep_next_zmw", "dcb_prep_get_windows", "dcb_prep_ccs_header", "dcb_prep_close",
    "dcb_prep_last_error", "dcb_prep_export_records", "dcb_prep_get_records", "dcb_prep_use_ccs_smart_windows",
    "dcb_prep_get_window_widths", "dcb_prep_get_overflow_ccs", "dcb_features_layout", "dcb_features_pack",
    "dcb_features_layout_smart", "dcb_features_ccs", "dcb_prep_get_window_lengths", "dcb_prep_open_truth",
    "dcb_prep_get_label", "dcb_features_labels", "dcb_features_eval",
    "dcb_calib_open", "dcb_calib_contigs", "dcb_calib_fetch_reference", "dcb_calib_query", "dcb_calib_next_batch",
    "dcb_calib_get_batch", "dcb_calib_read_name", "dcb_calib_close", "dcb_calib_count", "dcb_read_identity",
    "dcb_read_errors",
    "dcb_seq_open", "dcb_seq_next_batch", "dcb_seq_get_batch", "dcb_seq_read_name", "dcb_seq_close",
    "dcb_kmer_table_init", "dcb_kmer_table_clear", "dcb_kmer_count", "dcb_kmer_query", "dcb_kmer_wait",
    "dcb_kmer_table_stats", "dcb_kmer_set_init", "dcb_kmer_set_clear", "dcb_kmer_set_count", "dcb_kmer_spectrum",
    "dcb_bamw_open", "dcb_bamw_write", "dcb_bamw_close",
    "dcb_last_forward_launches", "dcb_set_profile", "dcb_get_profile", "dcb_get_profile_kernels", "dcb_alloc_host",
    "dcb_free_host", "dcb_alloc_device", "dcb_free_device", "dcb_memcpy_h2d", "dcb_memcpy_d2h",
    "dcb_synchronize", "dcb_last_error", "dcb_version", "dcb_destroy",
)
# include/dcb200_debug.h: developer / test hooks, not part of the drop-in boundary
DEBUG_SYMBOLS = ("dcb_set_debug", "dcb_debug_residual", "dcb_debug_operand", "dcb_debug_f32", "dcb_debug_head_epilogue")
# dcb_debug_operand's image ids (DCB_DEBUG_*)
DEBUG_OPERANDS = {"embed": 0, "xb": 1, "qkv": 2, "att": 3, "hid": 4}
# dcb_debug_f32's image ids (DCB_DEBUG_F32_*)
DEBUG_F32 = {"emb": 0, "x": 1, "y": 2, "q": 3, "k": 4, "v": 5, "att": 6, "hid": 7}


def library_path() -> str:
  return _LIB_PATH


def load_library() -> ctypes.CDLL:
  """Loads libdcb200.so (built in-tree by `__graft_entry__.build()` / csrc/build.sh)."""
  global _lib
  if _lib is None:
    _lib = _load(_LIB_PATH)
  return _lib


_dev_lib = None


def load_dev_library() -> ctypes.CDLL:
  """libdcb200_dev.so: the same sources built with -DDCB_DEV_SWITCHES, where DCB_ALIGN=0 selects the alternative
  token layout (tests and scripts only; pass as B200Model(..., library=...))."""
  global _dev_lib
  if _dev_lib is None:
    _dev_lib = _load(os.path.join(os.path.dirname(_LIB_PATH), "libdcb200_dev.so"))
  return _dev_lib


def _load(path: str) -> ctypes.CDLL:
  if not os.path.exists(path):
    raise FileNotFoundError(
        "%s not found: build the CUDA extension first (python -c 'import __graft_entry__ as g; "
        "g.build()'); the dcb200 engine has no CPU fallback" % path)
  lib = ctypes.CDLL(path)
  vp, i32, u32 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_uint32
  lib.dcb_create.argtypes = [ctypes.POINTER(DcbConfig), ctypes.POINTER(vp)]
  lib.dcb_load_weights.argtypes = [vp, ctypes.POINTER(DcbTensor), i32]
  lib.dcb_forward.argtypes = [vp, vp, i32, u32, vp, vp, vp, vp]
  lib.dcb_submit.argtypes = [vp, vp, i32, u32, vp, vp, vp, vp, ctypes.POINTER(ctypes.c_int64)]
  lib.dcb_wait.argtypes = [vp, ctypes.c_int64]
  lib.dcb_packed_window_bytes.argtypes = [ctypes.POINTER(DcbConfig)]
  lib.dcb_packed_window_bytes.restype = ctypes.c_size_t
  lib.dcb_pack_rows.argtypes = [ctypes.POINTER(DcbConfig), vp, i32, vp]
  lib.dcb_forward_packed.argtypes = [vp, vp, i32, u32, vp, vp, vp, vp]
  lib.dcb_submit_packed.argtypes = [vp, vp, i32, u32, vp, vp, vp, vp, ctypes.POINTER(ctypes.c_int64)]
  lib.dcb_stitch.argtypes = [vp, vp, vp, i32, i32, vp, i32, u32, vp, vp, vp]
  f64 = ctypes.c_double
  lib.dcb_stitch_fastq.argtypes = [vp, vp, vp, i32, i32, vp, i32, vp, vp, vp, f64, i32, u32, vp, ctypes.c_int64, vp, vp, vp]
  lib.dcb_skip_mask.argtypes = [vp, vp, i32, i32, f64, vp, vp]
  lib.dcb_fill_skipped.argtypes = [vp, vp, vp, vp, i32, i32, i32, f64, f64, f64, u32, vp, vp]
  lib.dcb_stitch_ragged.argtypes = [vp, vp, vp, vp, i32, vp, i32, u32, vp, vp, vp]
  lib.dcb_stitch_fastq_ragged.argtypes = [vp, vp, vp, vp, i32, i32, vp, i32, vp, vp, vp, f64, i32, u32, vp, ctypes.c_int64, vp,
                                          vp, vp]
  lib.dcb_fill_skipped_ragged.argtypes = [vp, vp, vp, vp, vp, i32, vp, i32, i32, f64, f64, f64, u32, vp, vp]
  lib.dcb_evaluate.argtypes = [vp, vp, vp, vp, i32, i32, f64, f64, i32, u32, vp, vp, vp, vp,
                               ctypes.POINTER(ctypes.c_float)]
  lib.dcb_evaluate_calibration.argtypes = [vp, vp, vp, vp, vp, i32, i32, u32, vp, vp, vp, vp, ctypes.POINTER(ctypes.c_float)]
  lib.dcb_distill_loss.argtypes = [vp, vp, vp, i32, i32, f64, i32, u32, vp, ctypes.POINTER(ctypes.c_float)]
  lib.dcb_distill_loss_grad.argtypes = [vp, vp, vp, i32, i32, f64, i32, u32, vp, vp, ctypes.POINTER(ctypes.c_float)]
  lib.dcb_alignment_loss_grad.argtypes = [vp, vp, vp, i32, i32, f64, f64, i32, u32, vp, vp, vp,
                                          ctypes.POINTER(ctypes.c_float)]
  lib.dcb_features_layout.argtypes = [vp, ctypes.POINTER(DcbRecords), i32, i32, vp, vp, vp, vp, vp, vp, ctypes.POINTER(i32),
                                      ctypes.POINTER(ctypes.c_float)]
  lib.dcb_features_pack.argtypes = [vp, vp, i32, u32, vp, ctypes.POINTER(ctypes.c_float)]
  lib.dcb_features_layout_smart.argtypes = [vp, ctypes.POINTER(DcbRecords), vp, vp, i32, i32, vp, vp, vp, vp, vp, vp, vp,
                                            ctypes.POINTER(i32), ctypes.POINTER(ctypes.c_float)]
  lib.dcb_features_ccs.argtypes = [vp, vp, i32, vp, vp, vp, ctypes.POINTER(ctypes.c_float)]
  lib.dcb_features_labels.argtypes = [vp, ctypes.POINTER(DcbLabels), vp, i32, vp, vp, vp, ctypes.POINTER(ctypes.c_float)]
  lib.dcb_features_eval.argtypes = [vp, ctypes.POINTER(DcbLabels), vp, i32, i32, vp, vp, vp, vp, vp, vp, ctypes.POINTER(i32),
                                    ctypes.POINTER(ctypes.c_float)]
  lib.dcb_calib_count.argtypes = [vp, ctypes.POINTER(DcbCalibInput), vp, vp, ctypes.POINTER(ctypes.c_float)]
  lib.dcb_read_identity.argtypes = [vp, ctypes.POINTER(DcbIdentityInput), vp, vp, vp, ctypes.POINTER(ctypes.c_float)]
  lib.dcb_read_errors.argtypes = [vp, ctypes.POINTER(DcbIdentityInput), vp, ctypes.POINTER(ctypes.c_float)]
  lib.dcb_kmer_table_init.argtypes = [vp, ctypes.c_int64, i32, ctypes.POINTER(ctypes.c_int64)]
  lib.dcb_kmer_table_clear.argtypes = [vp, i32, i32]
  lib.dcb_kmer_count.argtypes = [vp, ctypes.POINTER(DcbKmerBatch), i32]
  lib.dcb_kmer_query.argtypes = [vp, ctypes.POINTER(DcbKmerBatch), i32, i32, i32]
  lib.dcb_kmer_wait.argtypes = [vp, i32, vp, vp, vp, ctypes.POINTER(ctypes.c_float)]
  lib.dcb_kmer_table_stats.argtypes = [vp, vp, vp]
  lib.dcb_kmer_set_init.argtypes = [vp, ctypes.c_int64, ctypes.POINTER(ctypes.c_int64)]
  lib.dcb_kmer_set_clear.argtypes = [vp, i32, i32]
  lib.dcb_kmer_set_count.argtypes = [vp, ctypes.POINTER(DcbKmerBatch), vp, i32]
  lib.dcb_kmer_spectrum.argtypes = [vp, vp, vp]
  lib.dcb_last_forward_ms.argtypes = [vp, ctypes.POINTER(ctypes.c_float)]
  lib.dcb_last_forward_launches.argtypes = [vp, ctypes.POINTER(i32)]
  lib.dcb_set_debug.argtypes = [vp, i32]
  lib.dcb_set_profile.argtypes = [vp, i32]
  lib.dcb_get_profile.argtypes = [vp, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(i32),
                                  ctypes.POINTER(ctypes.c_int64)]
  lib.dcb_get_profile_kernels.argtypes = [vp, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(i32)]
  lib.dcb_debug_residual.argtypes = [vp, i32, vp, ctypes.c_int64]
  lib.dcb_debug_operand.argtypes = [vp, i32, i32, vp, ctypes.c_int64]
  lib.dcb_debug_f32.argtypes = [vp, i32, i32, vp, ctypes.c_int64]
  lib.dcb_debug_head_epilogue.argtypes = [vp, vp, ctypes.c_int64, vp, vp, vp]
  lib.dcb_alloc_host.argtypes = [ctypes.c_size_t, ctypes.POINTER(vp)]
  lib.dcb_free_host.argtypes = [vp]
  lib.dcb_alloc_device.argtypes = [vp, ctypes.c_size_t, ctypes.POINTER(vp)]
  lib.dcb_free_device.argtypes = [vp, vp]
  lib.dcb_memcpy_h2d.argtypes = [vp, vp, vp, ctypes.c_size_t]
  lib.dcb_memcpy_d2h.argtypes = [vp, vp, vp, ctypes.c_size_t]
  lib.dcb_synchronize.argtypes = [vp]
  lib.dcb_last_error.argtypes = [vp]
  lib.dcb_last_error.restype = ctypes.c_char_p
  lib.dcb_version.restype = ctypes.c_char_p
  lib.dcb_destroy.argtypes = [vp]
  lib.dcb_destroy.restype = None
  return lib


def make_config(params: params_lib.Params, max_batch: int, device: int = 0,
                max_base_quality: int = 93,
                calibration: Optional[calibration_lib.QualityCalibrationValues] = None,
                chunk_tiles: int = 0, precision: str = "bf16") -> DcbConfig:
  """params (params.json surface) + InferenceOptions fields -> dcb_config."""
  if precision not in PRECISIONS:
    raise ValueError("precision must be 'bf16' (tensor cores), 'fp32' (strict, the reference's arithmetic) or "
                     "'tf32x3' (the strict forward with its GEMMs on the tensor cores), got %r" % (precision,))
  c = DcbConfig()
  c.struct_size = ctypes.sizeof(DcbConfig)
  c.device = device
  c.max_passes, c.max_length = int(params.max_passes), int(params.max_length)
  c.use_ccs_bq = int(bool(params.use_ccs_bq))
  c.hidden_size, c.num_heads = int(params.hidden_size), int(params.num_heads)
  c.num_hidden_layers, c.filter_size = int(params.num_hidden_layers), int(params.filter_size)
  c.attn_win_size = int(params.attn_win_size or 0)
  c.rezero = int(bool(params.rezero))
  c.add_pos_encoding = int(bool(params.add_pos_encoding))
  c.condense_transformer_input = int(bool(params.condense_transformer_input))
  for f in ("per_base", "pw", "ip", "strand", "ccs_bq", "sn"):
    setattr(c, f + "_hidden_size", int(params[f + "_hidden_size"]))
  c.pw_max, c.ip_max, c.sn_max = int(params.PW_MAX), int(params.IP_MAX), int(params.SN_MAX)
  c.ccs_bq_max, c.strand_max = int(params.CCS_BQ_MAX), int(params.STRAND_MAX)
  c.max_base_quality = int(max_base_quality)
  if calibration is not None and calibration.enabled:
    c.calibration_enabled = 1
    c.calibration_threshold = float(calibration.threshold)
    c.calibration_w, c.calibration_b = float(calibration.w), float(calibration.b)
  c.max_batch = int(max_batch)
  c.chunk_tiles = int(chunk_tiles)
  c.precision = PRECISIONS[precision]
  for need in ("use_bases", "use_pw", "use_ip", "use_strand", "use_ccs", "use_sn"):
    if not params.get(need, True):
      raise DcbError(-1, "params.%s=False is not supported by the dcb200 engine" % need)
  return c


class _Prediction:
  """Stand-in for the EagerTensor `model.predict` returns (quick_inference.py:368-370)."""

  def __init__(self, array: np.ndarray):
    self._array = array

  def numpy(self) -> np.ndarray:
    return self._array


def _ptr(x: Any) -> Optional[ctypes.c_void_p]:
  """A void* argument: an ndarray's data, or an integer address (0 or None: NULL)."""
  if isinstance(x, np.ndarray):
    return x.ctypes.data_as(ctypes.c_void_p)
  return ctypes.c_void_p(int(x)) if x else None


def _arg(x: Any, dtype: Any, on_device: bool = False) -> Tuple[Optional[ctypes.c_void_p], Optional[np.ndarray]]:
  """A host-or-device input: with on_device a device address, else x as a C-contiguous `dtype` array.  Returns the
  pointer and the array it points into (None for an address), which must stay alive until the call returns."""
  if on_device:
    return _ptr(x), None
  a = np.ascontiguousarray(x, dtype=dtype)
  return _ptr(a), a


def ccs_bq_bytes(ccs_bq: Any) -> np.ndarray:
  """CCS base qualities (int16 from a tf.Example or the feature layout) as the uint8 rows dcb_evaluate_calibration reads:
  a value outside 0..255, such as a gap's -1, becomes 255, which the call refuses wherever a base carries it."""
  q = np.asarray(ccs_bq)
  return np.ascontiguousarray(np.where((q < 0) | (q > 255), 255, q), dtype=np.uint8)


def _outputs(out: Optional[Dict[str, int]], shapes: Dict[str, Optional[Tuple[int, ...]]]):
  """float32 outputs of a call that can write device memory; shapes[k] is None for an output not wanted.  With `out`, a
  dict of device addresses, the results go there (DCB_OUT_ON_DEVICE) and come back as None; otherwise host arrays are
  allocated.  Returns (flag, pointers in the order of `shapes`, result dict)."""
  res: Dict[str, Any] = dict.fromkeys(shapes)
  if out is not None:
    return DCB_OUT_ON_DEVICE, [None if shape is None else _ptr(out[k]) for k, shape in shapes.items()], res
  for k, shape in shapes.items():
    if shape is not None:
      res[k] = np.zeros(shape, np.float32)
  return 0, [_ptr(res[k]) for k in shapes], res


def _rows3(params: params_lib.Params, rows: np.ndarray) -> np.ndarray:
  """float32 rows [B, R, L(,1)] of `params`' geometry as a C-contiguous float32 [B, R, L] array."""
  rows = np.asarray(rows)
  if rows.ndim == 4:
    if rows.shape[-1] != 1:
      raise ValueError("rows must be [B, R, L, 1]")
    rows = rows[..., 0]
  R, L = params_lib.get_total_rows(params.max_passes, params.use_ccs_bq), int(params.max_length)
  if rows.ndim != 3 or rows.shape[1] != R or rows.shape[2] != L:
    raise ValueError("rows must be [B, %d, %d(, 1)], got %s" % (R, L, rows.shape))
  return np.ascontiguousarray(rows, dtype=np.float32)


class B200Model:
  """The encoder-only learned-values transformer on one H100, behind the C-ABI."""

  def __init__(self, params: params_lib.Params, weights: weights_lib.Weights, max_batch: int = 1024,
               device: int = 0, max_base_quality: int = 93,
               calibration: Optional[calibration_lib.QualityCalibrationValues] = None,
               chunk_tiles: int = 0, precision: str = "bf16", library: Optional[ctypes.CDLL] = None):
    """precision: "bf16" = tensor-core path (default); "fp32" = strict path, the reference's float32 arithmetic
    (identical bases wherever the float32 top-2 logit margin exceeds 1e-3; ~25x slower); "tf32x3" = the strict
    path's forward with its GEMMs on the tensor cores, each float32 operand split into two tf32 parts (the same
    accuracy gates as "fp32").  Any of them can be overridden per call with forward(..., strict=True/False), which
    selects the "fp32" / "bf16" path."""
    self._lib = library if library is not None else load_library()
    self._handle = ctypes.c_void_p()
    self.params = params
    self.max_batch = max_batch
    self.device = int(device)
    self.max_length = int(params.max_length)
    self.total_rows = params_lib.get_total_rows(params.max_passes, params.use_ccs_bq)
    self._layout_windows = 0   # windows of the last successful features_layout
    cfg = make_config(params, max_batch, device, max_base_quality, calibration, chunk_tiles, precision)
    rc = self._lib.dcb_create(ctypes.byref(cfg), ctypes.byref(self._handle))
    if rc:
      msg = self._lib.dcb_last_error(None).decode()
      self._handle = ctypes.c_void_p()
      raise DcbError(rc, msg)
    self.load_weights(weights)

  # -- lifecycle ---------------------------------------------------------------------------
  def close(self) -> None:
    if getattr(self, "_handle", None) and self._handle.value:
      self._lib.dcb_destroy(self._handle)
      self._handle = ctypes.c_void_p()
      for st in getattr(self, "_stage", {}).values():
        for addr in st["addrs"]:
          free_pinned(addr)
      self._stage = {}

  def __del__(self):
    try:
      self.close()
    except Exception:  # interpreter shutdown
      pass

  def _check(self, rc: int, tolerate: Tuple[int, ...] = ()) -> int:
    if rc and rc not in tolerate:
      raise DcbError(rc, self._lib.dcb_last_error(self._handle).decode())
    return rc

  def load_weights(self, weights: weights_lib.Weights) -> None:
    weights_lib.check_weights(self.params, weights)
    keep, tensors = [], (DcbTensor * len(weights))()
    for i, (name, arr) in enumerate(weights.items()):
      shape = np.shape(arr)                      # 0-d for the ReZero alphas
      a = np.ascontiguousarray(np.asarray(arr, dtype=np.float32)).reshape(-1)
      keep.append(a)
      tensors[i].name = name.encode()
      tensors[i].data = a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
      tensors[i].ndim = len(shape)
      for d, s in enumerate(shape):
        tensors[i].shape[d] = s
    self._check(self._lib.dcb_load_weights(self._handle, tensors, len(weights)))

  # -- the hot path ------------------------------------------------------------------------
  @staticmethod
  def _precision_flag(strict: Optional[bool]) -> int:
    return 0 if strict is None else (DCB_STRICT_FP32 if strict else DCB_FAST_BF16)

  def forward(self, rows: np.ndarray, want_probs: bool = False, want_logits: bool = False,
              strict_input: bool = True, strict: Optional[bool] = None) -> Dict[str, np.ndarray]:
    """rows float32 [B, R, L(,1)] -> dict(bases u8 [B,L], quals u8 [B,L], [probs], [logits]).

    Batches larger than `max_batch` are split, like `batch_examples` does with
    `options.batch_size` (quick_inference.py:304-338).
    """
    return self._forward_chunks(self._lib.dcb_forward, _rows3(self.params, rows), want_probs, want_logits,
                                strict_input, strict)

  def _forward_chunks(self, fn, x: np.ndarray, want_probs: bool, want_logits: bool, strict_input: bool,
                      strict: Optional[bool]) -> Dict[str, np.ndarray]:
    """forward() / forward_packed() on validated input x [B, ...]: dcb_forward or dcb_forward_packed (`fn`) per
    max_batch chunk into host arrays."""
    B, L = x.shape[0], self.max_length
    out = dict(bases=np.empty((B, L), np.uint8), quals=np.empty((B, L), np.uint8))
    if want_probs:
      out["probs"] = np.empty((B, L, 5), np.float32)
    if want_logits:
      out["logits"] = np.empty((B, L, 5), np.float32)
    ms, launches = 0.0, 0
    for b0 in range(0, B, self.max_batch):
      b1 = min(B, b0 + self.max_batch)
      part = [out[k][b0:b1] if k in out else None for k in ("bases", "quals", "probs", "logits")]
      self._forward_chunk(fn, x[b0:b1], self._precision_flag(strict), *part, strict_input=strict_input)
      ms += self.last_forward_ms()
      launches += self.last_forward_launches()
    self.last_ms, self.last_launches = ms, launches
    return out

  def _forward_chunk(self, fn, x: np.ndarray, flags: int, bases, quals, probs, logits, strict_input: bool) -> None:
    """One dcb_forward / dcb_forward_packed call on at most max_batch windows; outputs are host arrays or device
    addresses (per `flags`), None for one not wanted."""
    rc = fn(self._handle, _ptr(x), x.shape[0], flags, _ptr(bases), _ptr(quals), _ptr(probs), _ptr(logits))
    self._check(rc, tolerate=() if strict_input else (-5,))

  # -- packed input rows (include/dcb200.h "packed input rows")1) -------------------------
  @property
  def packed_window_bytes(self) -> int:
    return packed_window_bytes(self.params)

  def pack_rows(self, rows: np.ndarray, out: Optional[np.ndarray] = None, strict_input: bool = True) -> np.ndarray:
    return pack_rows(self.params, rows, out, strict_input)

  def forward_packed(self, packed: np.ndarray, want_probs: bool = False, want_logits: bool = False,
                     strict_input: bool = True, strict: Optional[bool] = None) -> Dict[str, np.ndarray]:
    """forward() on packed rows uint8 [B, packed_window_bytes]: bit-identical to forward() on the float32 rows they
    were packed from."""
    packed = np.ascontiguousarray(packed, dtype=np.uint8)
    if packed.ndim != 2 or packed.shape[1] != self.packed_window_bytes:
      raise ValueError("packed rows must be uint8 [B, %d]" % self.packed_window_bytes)
    return self._forward_chunks(self._lib.dcb_forward_packed, packed, want_probs, want_logits, strict_input, strict)

  def submit_packed_raw(self, packed_ptr: int, batch: int, flags: int, bases_ptr: int, quals_ptr: int,
                        probs_ptr: int = 0, logits_ptr: int = 0) -> int:
    """dcb_submit_packed on caller-managed pointers; returns the ticket for wait_raw()."""
    ticket = ctypes.c_int64(-1)
    self._check(self._lib.dcb_submit_packed(self._handle, _ptr(packed_ptr), batch, flags, _ptr(bases_ptr),
                                            _ptr(quals_ptr), _ptr(probs_ptr), _ptr(logits_ptr), ctypes.byref(ticket)))
    return int(ticket.value)

  # -- the hot path, pipelined over a stream of batches ----------------------------------------
  # dcb_submit / dcb_wait: the host->device copy of batch i+1 overlaps the kernels of batch i.  Page-locked staging
  # (two sets, allocated on first use) is owned here so that callers can stack their windows straight into it.
  def staging_rows(self, slot: int) -> np.ndarray:
    """Pinned float32 [max_batch, R, L] buffer of pipeline slot 0/1 (fill [:batch], then submit(slot=...))."""
    return self._staging(slot, "rows")

  def _staging(self, slot: int, key: str) -> np.ndarray:
    """Pinned buffer `key` (rows, bases, quals, probs or logits) of pipeline slot 0/1, allocated on first use."""
    st = self.__dict__.setdefault("_stage", {}).setdefault(slot, {"addrs": []})
    if key not in st:
      mb, R, L = self.max_batch, self.total_rows, self.max_length
      shape, dtype = {"rows": ((mb, R, L), np.float32), "bases": ((mb, L), np.uint8), "quals": ((mb, L), np.uint8),
                      "probs": ((mb, L, 5), np.float32), "logits": ((mb, L, 5), np.float32)}[key]
      n = int(np.prod(shape)) * np.dtype(dtype).itemsize
      addr, raw = alloc_pinned(max(n, 1))
      st["addrs"].append(addr)
      st[key] = raw[:n].view(dtype).reshape(shape)
    return st[key]

  def submit(self, rows: Optional[np.ndarray] = None, batch: Optional[int] = None, slot: Optional[int] = None,
             want_probs: bool = False, want_logits: bool = False, strict: Optional[bool] = None) -> Dict[str, Any]:
    """Enqueue one batch (<= max_batch windows) and return a handle for wait().  Either pass `rows` (copied into the
    slot's pinned staging) or fill staging_rows(slot)[:batch] yourself and pass `batch`.  At most two handles may be
    outstanding and they must be waited for in submission order."""
    busy = self.__dict__.setdefault("_slot_busy", {0: False, 1: False})
    if slot is None:
      slot = 1 - getattr(self, "_last_slot", 1)
      if busy[slot] and not busy[1 - slot]:
        slot = 1 - slot
    if busy[slot]:   # its pinned staging may still be read by the copy engine: refuse before touching it
      raise DcbError(-4, "two submissions in flight: wait() for the oldest first")
    self._last_slot = slot
    staged = self._staging(slot, "rows")
    if rows is not None:
      rows = _rows3(self.params, rows)
      batch = rows.shape[0]
      if batch > self.max_batch:
        raise ValueError("submit(): batch %d > max_batch %d" % (batch, self.max_batch))
      staged[:batch] = rows
    elif batch is None:
      raise ValueError("submit(): rows or batch required")
    out = [self._staging(slot, k) if want else None
           for k, want in (("bases", True), ("quals", True), ("probs", want_probs), ("logits", want_logits))]
    ticket = ctypes.c_int64(-1)
    self._check(self._lib.dcb_submit(self._handle, _ptr(staged), batch, self._precision_flag(strict),
                                     *(_ptr(a) for a in out), ctypes.byref(ticket)))
    busy[slot] = True
    return dict(ticket=int(ticket.value), slot=slot, batch=batch, probs=want_probs, logits=want_logits)

  def wait(self, handle: Dict[str, Any], strict_input: bool = True) -> Dict[str, np.ndarray]:
    """Block until the submission's results are on the host; returns the same dict as forward()."""
    rc = self._lib.dcb_wait(self._handle, handle["ticket"])
    if rc != -4:   # anything but "not in flight" retires the slot
      self._slot_busy[handle["slot"]] = False
    self._check(rc, tolerate=() if strict_input else (-5,))
    keys = ["bases", "quals"] + [k for k in ("probs", "logits") if handle[k]]
    out = {k: self._staging(handle["slot"], k)[:handle["batch"]].copy() for k in keys}
    self.last_ms, self.last_launches = self.last_forward_ms(), self.last_forward_launches()
    return out

  def drain(self, *handles) -> None:
    """Retire outstanding submissions whose results are no longer wanted (error paths): waits for each handle and
    swallows its status, so the engine's and this object's pipeline slots are free again."""
    for h in handles:
      if h is None:
        continue
      try:
        self.wait(h, strict_input=False)
      except DcbError:
        pass

  def forward_batches(self, batches, want_probs: bool = False, want_logits: bool = False,
                      strict_input: bool = True, strict: Optional[bool] = None):
    """Pipelined forward over an iterable of row batches; yields one output dict per batch, in order."""
    submit = lambda rows: self.submit(rows, want_probs=want_probs, want_logits=want_logits, strict=strict)
    for _, out in pipelined(batches, submit, lambda h: self.wait(h, strict_input), self.drain):
      yield out

  # -- stitch: per-read window concatenation + gap compaction on the device -------------------------
  def stitch(self, bases, quals, zmw_start: np.ndarray, n_windows: Optional[int] = None,
             on_device: bool = False, length: Optional[int] = None, win_off: Optional[np.ndarray] = None
             ) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """dcb_stitch: bases/quals are uint8 [n_windows, L] arrays (or device addresses when `on_device`); read z is the
    windows [zmw_start[z], zmw_start[z+1]).  Returns (seq, qual, lengths): read z's compacted characters are
    seq[zmw_start[z] * L : zmw_start[z] * L + lengths[z]] (same for qual).  With `win_off` (int64 [n_windows + 1]),
    dcb_stitch_ragged: window w is bytes win_off[w] .. win_off[w + 1] of the flat bases / quals, and read z starts at
    win_off[zmw_start[z]]."""
    zs = np.ascontiguousarray(zmw_start, dtype=np.int32)
    nz = int(zs.shape[0]) - 1
    L = int(length) if length is not None else self.max_length   # characters per window
    if on_device and n_windows is None and win_off is None:
      raise ValueError("stitch(on_device=True) needs n_windows")
    b_ptr, bases = _arg(bases, np.uint8, on_device)
    q_ptr, quals = _arg(quals, np.uint8, on_device)
    flags = DCB_ROWS_ON_DEVICE if on_device else 0
    lens = np.zeros(max(nz, 0), np.int32)
    if win_off is not None:
      off = np.ascontiguousarray(win_off, dtype=np.int64)
      seq, qual = np.empty(int(off[-1]), np.uint8), np.empty(int(off[-1]), np.uint8)
      self._check(self._lib.dcb_stitch_ragged(self._handle, b_ptr, q_ptr, _ptr(off), len(off) - 1, _ptr(zs), nz, flags,
                                              _ptr(seq), _ptr(qual), _ptr(lens)))
      return seq, qual, lens
    if not on_device:
      n_windows = int(bases.shape[0])
    seq = np.empty(n_windows * L, np.uint8)
    qual = np.empty(n_windows * L, np.uint8)
    self._check(self._lib.dcb_stitch(self._handle, b_ptr, q_ptr, n_windows, L, _ptr(zs), nz, flags, _ptr(seq), _ptr(qual),
                                     _ptr(lens)))
    return seq, qual, lens

  def stitch_fastq(self, bases, quals, zmw_start: np.ndarray, window_pos, names, min_quality: float, min_length: int,
                   n_windows: Optional[int] = None, on_device: bool = False, length: Optional[int] = None,
                   win_off: Optional[np.ndarray] = None):
    """dcb_stitch_fastq: stitch_utils.stitch_to_fastq for a batch of reads on the device.  Returns (fastq bytes,
    rec_off int64 [n_zmw + 1], outcome int32 [n_zmw], avg_q float64 [n_zmw]); read z's record is
    fastq[rec_off[z]:rec_off[z + 1]] (empty unless outcome[z] & 0x7f == DCB_READ_OK).  With `win_off` (int64
    [n_windows + 1]), dcb_stitch_fastq_ragged on windows of any width (see `stitch`)."""
    zs = np.ascontiguousarray(zmw_start, dtype=np.int32)
    nz = int(zs.shape[0]) - 1
    L = int(length) if length is not None else self.max_length
    if on_device and n_windows is None and win_off is None:
      raise ValueError("stitch_fastq(on_device=True) needs n_windows")
    b_ptr, bases = _arg(bases, np.uint8, on_device)
    q_ptr, quals = _arg(quals, np.uint8, on_device)
    off = None if win_off is None else np.ascontiguousarray(win_off, dtype=np.int64)
    if off is not None:
      n_windows = len(off) - 1
    elif not on_device:
      n_windows = int(bases.shape[0])
    pos = np.ascontiguousarray(window_pos, dtype=np.int32)
    if pos.shape[0] != n_windows:
      raise ValueError("window_pos must have one entry per window")
    enc = [n.encode("latin-1") if isinstance(n, str) else bytes(n) for n in names]
    if len(enc) != nz:
      raise ValueError("names must have one entry per read")
    name_off = np.zeros(nz + 1, np.int32)
    if nz:
      name_off[1:] = np.cumsum([len(x) for x in enc])
    blob = np.frombuffer(b"".join(enc) or b"\0", np.uint8)
    cap = int(name_off[-1]) + 2 * (n_windows * L if off is None else int(off[-1])) + 6 * nz + 16
    fastq = np.empty(cap, np.uint8)
    rec_off = np.zeros(nz + 1, np.int64)
    outcome = np.zeros(max(nz, 0), np.int32)
    avg_q = np.zeros(max(nz, 0), np.float64)
    tail = (_ptr(zs), nz, _ptr(pos), _ptr(blob), _ptr(name_off), float(min_quality), int(min_length),
            DCB_ROWS_ON_DEVICE if on_device else 0, _ptr(fastq), cap, _ptr(rec_off), _ptr(outcome), _ptr(avg_q))
    if off is None:
      self._check(self._lib.dcb_stitch_fastq(self._handle, b_ptr, q_ptr, n_windows, L, *tail))
    else:
      self._check(self._lib.dcb_stitch_fastq_ragged(self._handle, b_ptr, q_ptr, _ptr(off), n_windows, L, *tail))
    return fastq[:int(rec_off[-1])].tobytes(), rec_off, outcome, avg_q

  def skip_mask(self, ccs_base_quality_scores: np.ndarray, skip_windows_above: float) -> Tuple[np.ndarray, np.ndarray]:
    """dcb_skip_mask: per window avg_phred(ccs_base_quality_scores) > skip_windows_above on the device
    (quick_inference.py:663-672).  Returns (mask uint8 [n] with 2 = within 1e-7 of the threshold, avg float64 [n])."""
    bq = np.ascontiguousarray(ccs_base_quality_scores, dtype=np.int16)
    if bq.ndim != 2:
      raise ValueError("ccs_base_quality_scores must be [n_windows, L]")
    n, L = bq.shape
    mask, avg = np.zeros(n, np.uint8), np.zeros(n, np.float64)
    self._check(self._lib.dcb_skip_mask(self._handle, _ptr(bq), n, L, float(skip_windows_above), _ptr(mask), _ptr(avg)))
    return mask, avg

  def fill_skipped(self, ccs_ids: np.ndarray, ccs_base_quality_scores: np.ndarray, dst_window: np.ndarray,
                   bases, quals, calibration: Optional[calibration_lib.QualityCalibrationValues] = None,
                   on_device: bool = False) -> None:
    """dcb_fill_skipped: process_skipped_window (quick_inference.py:567-594) for k windows on the device; window j
    lands in row dst_window[j] of `bases` / `quals` (uint8 [*, L] arrays, or device addresses with on_device)."""
    ids = np.ascontiguousarray(ccs_ids, dtype=np.uint8)
    bq = np.ascontiguousarray(ccs_base_quality_scores, dtype=np.int16)
    dst = np.ascontiguousarray(dst_window, dtype=np.int32)
    k, L = ids.shape
    if bq.shape != (k, L) or dst.shape != (k,):
      raise ValueError("fill_skipped: ccs_ids / ccs_base_quality_scores [k, L] and dst_window [k] expected")
    cal = calibration
    en = int(bool(cal is not None and cal.enabled))
    if not on_device:   # written in place: no copy may stand in for the caller's arrays
      if not (bases.flags.c_contiguous and quals.flags.c_contiguous and bases.dtype == np.uint8 and quals.dtype == np.uint8):
        raise ValueError("fill_skipped: bases / quals must be C-contiguous uint8 arrays")
      if k and int(dst.max()) >= bases.shape[0]:
        raise ValueError("fill_skipped: destination window outside the output arrays")
    self._check(self._lib.dcb_fill_skipped(self._handle, _ptr(ids), _ptr(bq), _ptr(dst), k, L, en,
                                           float(cal.threshold) if en else 0.0, float(cal.w) if en else 1.0,
                                           float(cal.b) if en else 0.0, DCB_OUT_ON_DEVICE if on_device else 0,
                                           _ptr(bases), _ptr(quals)))

  def fill_skipped_ragged(self, ccs_ids: np.ndarray, ccs_base_quality_scores: np.ndarray, src_off: np.ndarray,
                          dst_window: np.ndarray, dst_off: np.ndarray, bases: np.ndarray, quals: np.ndarray,
                          calibration: Optional[calibration_lib.QualityCalibrationValues] = None) -> None:
    """dcb_fill_skipped_ragged: `fill_skipped` on windows of any width.  Skipped window j is ccs_ids /
    ccs_base_quality_scores[src_off[j]:src_off[j + 1]] (flat uint8 / int16) and is written to window dst_window[j] of
    the flat `bases` / `quals`, whose windows are dst_off (int64 [n_dst + 1]); the two widths must agree."""
    ids = np.ascontiguousarray(ccs_ids, dtype=np.uint8).reshape(-1)
    bq = np.ascontiguousarray(ccs_base_quality_scores, dtype=np.int16).reshape(-1)
    so, do = np.ascontiguousarray(src_off, dtype=np.int64), np.ascontiguousarray(dst_off, dtype=np.int64)
    dst = np.ascontiguousarray(dst_window, dtype=np.int32)
    k = len(so) - 1
    if ids.shape != bq.shape or len(ids) != int(so[-1]) or dst.shape != (k,):
      raise ValueError("fill_skipped_ragged: ccs_ids / ccs_base_quality_scores [src_off[-1]] and dst_window [k] expected")
    if not (bases.flags.c_contiguous and quals.flags.c_contiguous and bases.dtype == np.uint8 and quals.dtype == np.uint8):
      raise ValueError("fill_skipped_ragged: bases / quals must be C-contiguous uint8 arrays")
    if bases.size < int(do[-1]) or quals.size < int(do[-1]):
      raise ValueError("fill_skipped_ragged: bases / quals smaller than dst_off[-1]")
    cal = calibration
    en = int(bool(cal is not None and cal.enabled))
    self._check(self._lib.dcb_fill_skipped_ragged(self._handle, _ptr(ids), _ptr(bq), _ptr(so), _ptr(dst), k, _ptr(do),
                                                  len(do) - 1, en, float(cal.threshold) if en else 0.0,
                                                  float(cal.w) if en else 1.0, float(cal.b) if en else 0.0, 0,
                                                  _ptr(bases), _ptr(quals)))

  # -- feature construction on the device (include/dcb200.h "feature construction on the device") -----------------
  def features_layout(self, records: Dict[str, np.ndarray], ins_trim: int = 5) -> Dict[str, Any]:
    """dcb_features_layout (phase A) on a batch of raw records (`concat_records` of
    `preprocess.BamFeatureStream.next_zmw_records()` bundles): spaces the reads of every ZMW on the device and returns
    what dcb_prep_get_windows returns apart from the rows, dense over the batch -- dict(zmw_windows [n_zmw], window_pos
    [n], overflow [n], num_passes [n], ccs_bq int16 [n, L], ccs_ids uint8 [n, L], ms).  The spaced reads stay on the
    device for features_pack.  When the records carry `wl` / `wl_off` (CCS smart windows), dcb_features_layout_smart
    cuts the windows at those lengths and the result also has window_width [n]."""
    L = self.max_length
    spec = dict(zmw_read_off=np.int32, zmw_ccs_off=np.int32, zmw_ccs_bq_any=np.int32, read_meta=np.int32, read_sn=np.float32,
                cigar=np.uint32, bases=np.uint8, pw=np.uint8, ip=np.uint8, ccs_bases=np.uint8, ccs_bq=np.uint8)
    held = {k: _arg(records[k], dt) for k, dt in spec.items()}
    rec = DcbRecords(n_zmw=len(held["zmw_ccs_bq_any"][1]), n_cigar=held["cigar"][1].size, n_query=held["bases"][1].size)
    for k, (ptr, _) in held.items():
      setattr(rec, k, ptr)
    # a capacity that always suffices: the spaced width is at most the longest read plus every insertion column
    meta = held["read_meta"][1].reshape(-1, READ_META)
    ro = held["zmw_read_off"][1]
    smart = "wl" in records
    cap = 0
    for z in range(rec.n_zmw):
      m = meta[ro[z]:ro[z + 1]]
      longest = max(int(np.diff(held["zmw_ccs_off"][1])[z]), int((m[:, 4] + m[:, 7] - m[:, 6]).max(initial=0)))
      cap += (longest + int(m[:, 8].sum()) + 32 + L - 1) // L
    if smart:                                          # at most one window per length
      wl_off, wl = (np.ascontiguousarray(records[k], np.int32) for k in ("wl_off", "wl"))
      cap = len(wl)
    out = dict(zmw_windows=np.zeros(rec.n_zmw, np.int32), window_pos=np.zeros(cap, np.int32), overflow=np.zeros(cap, np.uint8),
               ccs_bq=np.zeros((cap, L), np.int16), num_passes=np.zeros(cap, np.int32), ccs_ids=np.zeros((cap, L), np.uint8))
    n, ms = ctypes.c_int32(0), ctypes.c_float(0)
    if smart:
      out["window_width"] = np.zeros(cap, np.int32)
      self._check(self._lib.dcb_features_layout_smart(
          self._handle, ctypes.byref(rec), _ptr(wl_off), _ptr(wl), int(ins_trim), cap, _ptr(out["zmw_windows"]),
          _ptr(out["window_pos"]), _ptr(out["overflow"]), _ptr(out["window_width"]), _ptr(out["ccs_bq"]),
          _ptr(out["num_passes"]), _ptr(out["ccs_ids"]), ctypes.byref(n), ctypes.byref(ms)))
    else:
      self._check(self._lib.dcb_features_layout(self._handle, ctypes.byref(rec), int(ins_trim), cap, _ptr(out["zmw_windows"]),
                                                _ptr(out["window_pos"]), _ptr(out["overflow"]), _ptr(out["ccs_bq"]),
                                                _ptr(out["num_passes"]), _ptr(out["ccs_ids"]), ctypes.byref(n), ctypes.byref(ms)))
    res: Dict[str, Any] = {k: (v if k == "zmw_windows" else v[:n.value]) for k, v in out.items()}
    res["ms"] = float(ms.value)
    self._layout_windows = int(n.value)
    return res

  def features_pack(self, windows: np.ndarray, out: Optional[int] = None) -> Dict[str, Any]:
    """dcb_features_pack (phase B): packed rows of the listed windows of the last features_layout, in the list's order.
    Returns dict(packed uint8 [k, packed_window_bytes], ms); with `out`, a 16-byte-aligned device address, the rows are
    written there (ready for forward_packed_raw with DCB_ROWS_ON_DEVICE) and `packed` is None."""
    idx = np.ascontiguousarray(windows, dtype=np.int32).reshape(-1)
    packed = None if out is not None else np.empty((len(idx), self.packed_window_bytes), np.uint8)
    ms = ctypes.c_float(0)
    self._check(self._lib.dcb_features_pack(self._handle, _ptr(idx), len(idx), DCB_OUT_ON_DEVICE if out is not None else 0,
                                            _ptr(out) if out is not None else _ptr(packed), ctypes.byref(ms)))
    return dict(packed=packed, ms=float(ms.value))

  def features_ccs(self, windows: np.ndarray, widths: np.ndarray) -> Dict[str, Any]:
    """dcb_features_ccs: the CCS ids and qualities of the listed windows of the last features_layout at full width
    (`widths`: their window_width).  Returns dict(ccs_ids uint8, ccs_bq int16, off int64 [n + 1], ms); window i is
    [off[i], off[i + 1])."""
    idx = np.ascontiguousarray(windows, dtype=np.int32).reshape(-1)
    off = np.zeros(len(idx) + 1, np.int64)
    np.cumsum(np.asarray(widths, np.int64).reshape(-1), out=off[1:])
    ids, bq = np.zeros(int(off[-1]), np.uint8), np.zeros(int(off[-1]), np.int16)
    ms = ctypes.c_float(0)
    self._check(self._lib.dcb_features_ccs(self._handle, _ptr(idx), len(idx), _ptr(off), _ptr(ids), _ptr(bq), ctypes.byref(ms)))
    return dict(ccs_ids=ids, ccs_bq=bq, off=off, ms=float(ms.value))

  def features_labels(self, labels: Dict[str, np.ndarray], windows: np.ndarray) -> Dict[str, Any]:
    """dcb_features_labels: the training label rows of the listed windows of the last features_layout.  `labels` is
    `concat_labels` of one label per ZMW of that batch.  Returns dict(labels uint8 [k, L] over ' ATCG', status uint8 [k]
    (0 kept, 1 gaps removed, 2 overflow), ccs_width int32 [n_zmw] (DcExample.ccs_width per ZMW of the batch), ms)."""
    idx = np.ascontiguousarray(windows, dtype=np.int32).reshape(-1)
    meta, cig, bases = (np.ascontiguousarray(labels[k], dt) for k, dt in (("label_meta", np.int32), ("cigar", np.uint32),
                                                                         ("bases", np.uint8)))
    lab = DcbLabels(n_zmw=meta.reshape(-1, LABEL_META).shape[0], n_cigar=cig.size, n_bases=bases.size,
                    label_meta=_ptr(meta), cigar=_ptr(cig), bases=_ptr(bases))
    out = dict(labels=np.zeros((len(idx), self.max_length), np.uint8), status=np.zeros(len(idx), np.uint8),
               ccs_width=np.zeros(lab.n_zmw, np.int32))
    ms = ctypes.c_float(0)
    self._check(self._lib.dcb_features_labels(self._handle, ctypes.byref(lab), _ptr(idx), len(idx), _ptr(out["labels"]),
                                              _ptr(out["status"]), _ptr(out["ccs_width"]), ctypes.byref(ms)))
    out["ms"] = float(ms.value)
    return out

  def features_eval(self, labels: Dict[str, np.ndarray], keep_zmw: np.ndarray, capacity: int, packed_ptr: int,
                    labels_ptr: int, ccs_ptr: int) -> Dict[str, Any]:
    """dcb_features_eval: the evaluation inputs of the last features_layout's windows.  `labels` is `concat_labels` of
    one label per ZMW of that batch, keep_zmw one flag per ZMW.  The kept windows (label status != 2, ZMW kept) go, in
    window order, to the device arrays at packed_ptr (uint8 [capacity, packed_window_bytes], 16-byte aligned),
    labels_ptr and ccs_ptr (uint8 [capacity, L] each).  Returns dict(k, status uint8 [n] of every window of the layout,
    ccs_width int32 [n_zmw], windows int32 [k] (layout index of every kept window), ms).  DcbError(-1) when k exceeds
    capacity."""
    meta, cig, bases = (np.ascontiguousarray(labels[k], dt) for k, dt in (("label_meta", np.int32), ("cigar", np.uint32),
                                                                         ("bases", np.uint8)))
    lab = DcbLabels(n_zmw=meta.reshape(-1, LABEL_META).shape[0], n_cigar=cig.size, n_bases=bases.size,
                    label_meta=_ptr(meta), cigar=_ptr(cig), bases=_ptr(bases))
    keep = np.ascontiguousarray(keep_zmw, np.uint8).reshape(-1)
    n = self._layout_windows
    out = dict(status=np.zeros(n, np.uint8), ccs_width=np.zeros(lab.n_zmw, np.int32),
               windows=np.zeros(max(int(capacity), 0), np.int32))
    k, ms = ctypes.c_int32(0), ctypes.c_float(0)
    self._check(self._lib.dcb_features_eval(self._handle, ctypes.byref(lab), _ptr(keep), len(keep), int(capacity),
                                            _ptr(packed_ptr), _ptr(labels_ptr), _ptr(ccs_ptr), _ptr(out["status"]),
                                            _ptr(out["ccs_width"]), _ptr(out["windows"]), ctypes.byref(k), ctypes.byref(ms)))
    out["k"] = int(k.value)
    out["windows"] = out["windows"][:out["k"]]
    out["ms"] = float(ms.value)
    return out

  def calib_count(self, batch: Dict[str, np.ndarray], regions: np.ndarray, interval_length: int,
                  ref_bases: Optional[np.ndarray], ref_start: int, ref_count: int, contig_length: int,
                  calibration: Optional[calibration_lib.QualityCalibrationValues] = None) -> Dict[str, Any]:
    """dcb_calib_count: the (match, mismatch) events per quality bin of one batch of reads (dict of read_meta int32
    [n, CALIB_META], cigar uint32, seq uint8 4-bit codes, qual uint8) over every interval of `regions` (int64 [k, 2],
    start and stop on one contig).  ref_bases: the contig's bases [ref_start, ref_start + ref_count), or None to keep
    the previous call's.  Returns dict(counts int64 [100, 2], failure (read index, position, DCB_CALIB_*) with read
    index -1 when no counted event fails, ms)."""
    meta = np.ascontiguousarray(batch["read_meta"], np.int32).reshape(-1, CALIB_META)
    cig, seq, qual = (np.ascontiguousarray(batch[k], dt) for k, dt in (("cigar", np.uint32), ("seq", np.uint8),
                                                                       ("qual", np.uint8)))
    reg = np.ascontiguousarray(regions, np.int64).reshape(-1, 2)
    # an empty array still has to reach the call as a non-NULL pointer: NULL keeps the previous call's bases
    ref = None if ref_bases is None else np.ascontiguousarray(ref_bases, np.uint8) if len(ref_bases) else np.zeros(1, np.uint8)
    cal = calibration
    en = bool(cal is not None and cal.enabled)
    arg = DcbCalibInput(n_reads=len(meta), n_regions=len(reg), n_cigar=cig.size, n_bases=seq.size, read_meta=_ptr(meta),
                        cigar=_ptr(cig), seq=_ptr(seq), qual=_ptr(qual), regions=_ptr(reg),
                        interval_length=int(interval_length), ref_bases=None if ref is None else _ptr(ref),
                        ref_start=int(ref_start), ref_count=int(ref_count), contig_length=int(contig_length),
                        calibration_enabled=int(en), threshold=float(cal.threshold) if en else 0.0,
                        w=float(cal.w) if en else 1.0, b=float(cal.b) if en else 0.0)
    counts, failure, ms = np.zeros((CALIB_BINS, 2), np.int64), np.zeros(3, np.int64), ctypes.c_float(0)
    self._check(self._lib.dcb_calib_count(self._handle, ctypes.byref(arg), _ptr(counts), _ptr(failure), ctypes.byref(ms)))
    return dict(counts=counts, failure=tuple(int(x) for x in failure), ms=float(ms.value))

  def read_identity(self, batch: Dict[str, np.ndarray], ref: np.ndarray, ref_start: int,
                    contig_length: int) -> Dict[str, Any]:
    """dcb_read_identity: per read of one batch (dict of read_meta int32 [n, CALIB_META], cigar uint32, seq uint8 4-bit
    codes, qual uint8) against `ref`, the contig's bases [ref_start, ref_start + len(ref)) as uint8 characters.
    Returns dict(counts int64 [n, IDENTITY_COUNTS] (matches, mismatches, insertions, deletions, soft clips), avg_q
    float64 [n], status int32 [n] (DCB_IDENTITY_*), ms)."""
    meta = np.ascontiguousarray(batch["read_meta"], np.int32).reshape(-1, CALIB_META)
    cig, seq, qual = (np.ascontiguousarray(batch[k], dt) for k, dt in (("cigar", np.uint32), ("seq", np.uint8),
                                                                       ("qual", np.uint8)))
    ref = np.ascontiguousarray(ref, np.uint8)
    n = len(meta)
    arg = DcbIdentityInput(n_reads=n, n_cigar=cig.size, n_bases=seq.size, read_meta=_ptr(meta), cigar=_ptr(cig),
                           seq=_ptr(seq), qual=_ptr(qual), ref_bases=_ptr(ref), ref_start=int(ref_start),
                           ref_count=ref.size, contig_length=int(contig_length))
    counts, avg_q, status = np.zeros((n, IDENTITY_COUNTS), np.int64), np.zeros(n, np.float64), np.zeros(n, np.int32)
    ms = ctypes.c_float(0)
    self._check(self._lib.dcb_read_identity(self._handle, ctypes.byref(arg), _ptr(counts), _ptr(avg_q), _ptr(status),
                                            ctypes.byref(ms)))
    return dict(counts=counts, avg_q=avg_q, status=status, ms=float(ms.value))

  def read_errors(self, batch: Dict[str, np.ndarray], ref: np.ndarray, ref_start: int,
                  contig_length: int) -> Dict[str, Any]:
    """dcb_read_errors: per read of one batch (as read_identity takes it) its errors by type and homopolymer length
    against `ref`, the contig's bases [ref_start, ref_start + len(ref)), which must hold every read's [pos - 1,
    endpos + 1) within the contig and the whole runs at both of its ends.  Returns dict(errors int64 [n, ERRORS_COLS],
    ms)."""
    meta = np.ascontiguousarray(batch["read_meta"], np.int32).reshape(-1, CALIB_META)
    cig, seq, qual = (np.ascontiguousarray(batch[k], dt) for k, dt in (("cigar", np.uint32), ("seq", np.uint8),
                                                                       ("qual", np.uint8)))
    ref = np.ascontiguousarray(ref, np.uint8)
    n = len(meta)
    arg = DcbIdentityInput(n_reads=n, n_cigar=cig.size, n_bases=seq.size, read_meta=_ptr(meta), cigar=_ptr(cig),
                           seq=_ptr(seq), qual=_ptr(qual), ref_bases=_ptr(ref), ref_start=int(ref_start),
                           ref_count=ref.size, contig_length=int(contig_length))
    errors, ms = np.zeros((n, ERRORS_COLS), np.int64), ctypes.c_float(0)
    self._check(self._lib.dcb_read_errors(self._handle, ctypes.byref(arg), _ptr(errors), ctypes.byref(ms)))
    return dict(errors=errors, ms=float(ms.value))

  # -- k-mer QV (include/dcb200.h "k-mer QV") ---------------------------------------------------------------------
  def kmer_table_init(self, table_bytes: int, k: int) -> int:
    """dcb_kmer_table_init: an empty k-mer table in at most table_bytes of device memory (<= 0: half the free
    memory); returns its capacity in slots."""
    cap = ctypes.c_int64(0)
    self._check(self._lib.dcb_kmer_table_init(self._handle, int(table_bytes), int(k), ctypes.byref(cap)))
    return int(cap.value)

  def kmer_table_clear(self, partition: int, n_partitions: int) -> None:
    self._check(self._lib.dcb_kmer_table_clear(self._handle, int(partition), int(n_partitions)))

  def kmer_submit(self, batch: Dict[str, np.ndarray], slot: int, min_count: int = 0, with_quality: bool = False
                  ) -> Tuple[int, int, DcbKmerBatch, Tuple[np.ndarray, ...]]:
    """dcb_kmer_count (min_count 0) or dcb_kmer_query of one batch (dict of bases uint8, offsets int64 [n + 1],
    qual uint8 and has_qual uint8 [n]) on pipeline slot 0 / 1.  Returns the handle kmer_wait takes."""
    arrays = tuple(np.ascontiguousarray(batch[k], dt) for k, dt in (("bases", np.uint8), ("offsets", np.int64),
                                                                    ("qual", np.uint8), ("has_qual", np.uint8)))
    bases, offsets, qual, has_qual = arrays
    arg = DcbKmerBatch(n_reads=len(offsets) - 1, n_bases=bases.size, bases=_ptr(bases), qual=_ptr(qual),
                       offsets=_ptr(offsets), has_qual=_ptr(has_qual))
    if min_count:
      self._check(self._lib.dcb_kmer_query(self._handle, ctypes.byref(arg), int(min_count), int(with_quality), int(slot)))
    else:
      self._check(self._lib.dcb_kmer_count(self._handle, ctypes.byref(arg), int(slot)))
    return int(slot), int(min_count), arg, arrays

  def kmer_wait(self, handle) -> Dict[str, Any]:
    """dcb_kmer_wait for a kmer_submit: dict(ms) and, for a query, counts int64 [n, 2] (k-mers of the partition,
    unsupported), avg_q float64 [n] and borderline bool [n]."""
    slot, query, arg, _ = handle
    n = arg.n_reads
    counts, avg_q, border = np.zeros((n, 2), np.int64), np.zeros(n, np.float64), np.zeros(n, np.int32)
    ms = ctypes.c_float(0)
    self._check(self._lib.dcb_kmer_wait(self._handle, slot, _ptr(counts), _ptr(avg_q), _ptr(border), ctypes.byref(ms)))
    out: Dict[str, Any] = dict(ms=float(ms.value))
    if query:
      out.update(counts=counts, avg_q=avg_q, borderline=border.astype(bool))
    return out

  def kmer_retire(self, handle) -> None:
    try:
      self.kmer_wait(handle)
    except DcbError:
      pass

  def kmer_table_stats(self, histogram: bool = True) -> Dict[str, Any]:
    """dcb_kmer_table_stats: dict of KMER_STAT_KEYS and, with `histogram`, histogram int64 [KMER_HIST + 1] ([c] = keys
    with count c, [KMER_HIST] = keys with count >= KMER_HIST)."""
    stats, hist = np.zeros(len(KMER_STAT_KEYS), np.int64), np.zeros(KMER_HIST + 1, np.int64)
    self._check(self._lib.dcb_kmer_table_stats(self._handle, _ptr(stats), _ptr(hist) if histogram else None))
    out: Dict[str, Any] = {k: int(v) for k, v in zip(KMER_STAT_KEYS, stats)}
    if histogram:
      out["histogram"] = hist
    return out

  def kmer_set_init(self, table_bytes: int) -> int:
    """dcb_kmer_set_init: an empty set table (the evaluated reads' k-mers) in at most table_bytes of device memory
    (<= 0: half the free memory), after kmer_table_init; returns its capacity in slots."""
    cap = ctypes.c_int64(0)
    self._check(self._lib.dcb_kmer_set_init(self._handle, int(table_bytes), ctypes.byref(cap)))
    return int(cap.value)

  def kmer_set_clear(self, partition: int, n_partitions: int) -> None:
    self._check(self._lib.dcb_kmer_set_clear(self._handle, int(partition), int(n_partitions)))

  def kmer_set_submit(self, handle, keep: np.ndarray) -> Tuple[int, int, DcbKmerBatch, Tuple[np.ndarray, ...]]:
    """dcb_kmer_set_count of the batch a kmer_submit `handle` (already waited for) staged, on the same slot, for the
    reads with keep[r] (bool or uint8 [n]).  Returns the handle kmer_wait takes."""
    slot, _, arg, arrays = handle
    keep = np.ascontiguousarray(keep, np.uint8)
    if keep.shape != (arg.n_reads,):
      raise ValueError("keep must have one entry per read of the batch, got shape %s" % (keep.shape,))
    self._check(self._lib.dcb_kmer_set_count(self._handle, ctypes.byref(arg), _ptr(keep), int(slot)))
    return int(slot), 0, arg, arrays + (keep,)

  def kmer_spectrum(self) -> Dict[str, Any]:
    """dcb_kmer_spectrum of the partition both tables hold: dict(matrix int64 [KMER_SPECTRUM_BINS,
    KMER_SPECTRUM_BINS] ([c][m] = distinct k-mers with table count c and set count m, 256 meaning >= 256), stats dict
    of KMER_SET_STAT_KEYS)."""
    b = KMER_SPECTRUM_BINS
    matrix, stats = np.zeros((b, b), np.int64), np.zeros(len(KMER_SET_STAT_KEYS), np.int64)
    self._check(self._lib.dcb_kmer_spectrum(self._handle, _ptr(matrix), _ptr(stats)))
    return dict(matrix=matrix, stats={k: int(v) for k, v in zip(KMER_SET_STAT_KEYS, stats)})

  def stitch_raw(self, bases_ptr: int, quals_ptr: int, n_windows: int, zmw_start: np.ndarray, flags: int,
                 seq_ptr: int, qual_ptr: int, len_ptr: int, length: Optional[int] = None) -> None:
    """dcb_stitch on caller-managed pointers (host or device per `flags`)."""
    zs = np.ascontiguousarray(zmw_start, dtype=np.int32)
    self._check(self._lib.dcb_stitch(self._handle, _ptr(bases_ptr), _ptr(quals_ptr), n_windows,
                                     int(length) if length is not None else self.max_length, _ptr(zs),
                                     int(zs.shape[0]) - 1, flags, _ptr(seq_ptr), _ptr(qual_ptr), _ptr(len_ptr)))

  # -- evaluation of labelled windows (include/dcb200.h "evaluation of labelled windows") -------------------------
  def _eval_args(self, del_cost, loss_reg, band_width):
    p = self.params
    del_cost = float(p.get("del_cost", 10.0) if del_cost is None else del_cost)
    loss_reg = p.get("loss_reg", 0.1) if loss_reg == "params" else loss_reg
    band_width = p.get("band_width") if band_width == "params" else band_width
    return (del_cost, 0.0 if loss_reg is None else float(loss_reg),
            DCB_BAND_WIDTH_NONE if band_width is None else int(band_width))

  def evaluate_windows(self, probs, labels: np.ndarray, ccs_ids: np.ndarray, del_cost: Optional[float] = None,
                       loss_reg: Any = "params", band_width: Any = "params", on_device: bool = False,
                       batch: Optional[int] = None, labels_on_device: bool = False) -> Dict[str, Any]:
    """dcb_evaluate: per-window AlignmentLoss, PerExampleAccuracy flag and AlignmentMetric counts of the prediction and
    of the CCS row.  probs float32 [B, L, 5] (host array, or a device address with on_device=True and `batch`);
    labels / ccs_ids uint8 [B, L] (host arrays, or with labels_on_device=True and `batch` device addresses of
    [batch, max_length], e.g. features_eval's).  del_cost / loss_reg / band_width default to params.json's
    (loss_reg=None: hard min; band_width set: DcbError -1).  Returns loss float32 [B], exact uint8 [B], pred_counts /
    ccs_counts int32 [B, 5] (columns EVAL_COUNT_KEYS) and ms, the device time of the evaluation kernels."""
    if labels_on_device:
      if batch is None:
        raise ValueError("evaluate_windows(labels_on_device=True) needs batch")
      B, L = int(batch), self.max_length
    else:
      labels = np.ascontiguousarray(labels, dtype=np.uint8)
      ccs_ids = np.ascontiguousarray(ccs_ids, dtype=np.uint8)
      if labels.ndim != 2 or ccs_ids.shape != labels.shape:
        raise ValueError("labels and ccs_ids must both be uint8 [B, L]")
      B, L = labels.shape
    if on_device and (batch is None or int(batch) != B):
      raise ValueError("evaluate_windows(on_device=True) needs batch == labels.shape[0]")
    p_ptr, probs = _arg(probs, np.float32, on_device)
    if not on_device and probs.shape != (B, L, 5):
      raise ValueError("probs must be float32 [%d, %d, 5], got %s" % (B, L, probs.shape))
    dc, reg, bw = self._eval_args(del_cost, loss_reg, band_width)
    out = _empty_eval(B)
    ms = ctypes.c_float()
    flags = (DCB_ROWS_ON_DEVICE if on_device else 0) | (DCB_LABELS_ON_DEVICE if labels_on_device else 0)
    self._check(self._lib.dcb_evaluate(self._handle, p_ptr, _ptr(labels), _ptr(ccs_ids), B, L, dc, reg, bw,
                                       flags, _ptr(out["loss"]), _ptr(out["exact"]),
                                       _ptr(out["pred_counts"]), _ptr(out["ccs_counts"]), ctypes.byref(ms)))
    out["ms"] = float(ms.value)
    return out

  def evaluate_calibration(self, probs, labels, ccs_ids, ccs_bq, on_device: bool = False,
                           batch: Optional[int] = None, labels_on_device: bool = False) -> Dict[str, Any]:
    """dcb_evaluate_calibration: base-quality calibration counts of the prediction and of the CCS row, from the
    traceback of evaluate_windows()'s AlignmentMetric counts.  probs / labels / ccs_ids as in evaluate_windows();
    ccs_bq uint8 [B, L] (ccs_bq_bytes) beside ccs_ids, host or, with labels_on_device, device.  Returns counts int64
    [2, CALIB_BINS, 2] ([prediction, CCS][quality][match, mismatch]), deletions int64 [2], pred_counts / ccs_counts
    int32 [B, 5] (bitwise evaluate_windows()'s) and ms, the kernel's device time."""
    if labels_on_device:
      if batch is None:
        raise ValueError("evaluate_calibration(labels_on_device=True) needs batch")
      B, L = int(batch), self.max_length
    else:
      labels = np.ascontiguousarray(labels, dtype=np.uint8)
      ccs_ids = np.ascontiguousarray(ccs_ids, dtype=np.uint8)
      ccs_bq = np.ascontiguousarray(ccs_bq, dtype=np.uint8)
      if labels.ndim != 2 or ccs_ids.shape != labels.shape or ccs_bq.shape != labels.shape:
        raise ValueError("labels, ccs_ids and ccs_bq must all be uint8 [B, L]")
      B, L = labels.shape
    if on_device and (batch is None or int(batch) != B):
      raise ValueError("evaluate_calibration(on_device=True) needs batch == labels.shape[0]")
    p_ptr, probs = _arg(probs, np.float32, on_device)
    if not on_device and probs.shape != (B, L, 5):
      raise ValueError("probs must be float32 [%d, %d, 5], got %s" % (B, L, probs.shape))
    out = dict(counts=np.zeros((2, CALIB_BINS, 2), np.int64), deletions=np.zeros(2, np.int64),
               pred_counts=np.zeros((B, 5), np.int32), ccs_counts=np.zeros((B, 5), np.int32))
    ms = ctypes.c_float()
    flags = (DCB_ROWS_ON_DEVICE if on_device else 0) | (DCB_LABELS_ON_DEVICE if labels_on_device else 0)
    self._check(self._lib.dcb_evaluate_calibration(self._handle, p_ptr, _ptr(labels), _ptr(ccs_ids), _ptr(ccs_bq), B, L,
                                                   flags, _ptr(out["counts"]), _ptr(out["deletions"]),
                                                   _ptr(out["pred_counts"]), _ptr(out["ccs_counts"]),
                                                   ctypes.byref(ms)))
    out["ms"] = float(ms.value)
    return out

  def distill_loss(self, teacher_logits, student_logits, temperature: float = 1.0, logit_loss: Any = "kl_divergence",
                   on_device: bool = False, batch: Optional[int] = None,
                   length: Optional[int] = None) -> Dict[str, Any]:
    """Per-window DistillationLoss between teacher and student logits float32 [B, L, 5] (host arrays, or device
    addresses with on_device=True, `batch` and optionally `length`, default max_length): distill_loss_grad() without
    the gradient, so dcb_distill_loss_grad computes it.  logit_loss is a Keras identifier (LOGIT_LOSS_IDS) or a
    DCB_LOGIT_LOSS_* id.  Returns loss float32 [B] and ms, the kernel's device time."""
    if on_device and batch is None:
      raise ValueError("distill_loss(on_device=True) needs batch")
    r = self.distill_loss_grad(teacher_logits, student_logits, temperature, logit_loss, want_grad=False,
                               on_device=on_device, batch=batch, length=length)
    return dict(loss=r["loss"], ms=r["ms"])

  def distill_loss_grad(self, teacher_logits, student_logits, temperature: float = 1.0,
                        logit_loss: Any = "kl_divergence", want_grad: bool = True, on_device: bool = False,
                        batch: Optional[int] = None, length: Optional[int] = None,
                        out: Optional[Dict[str, int]] = None) -> Dict[str, Any]:
    """dcb_distill_loss_grad: per-window DistillationLoss (bitwise equal to dcb_distill_loss's) and its gradient with
    respect to the student's logits, the teacher held constant.  Logits float32 [B, L, 5] are host arrays, or device
    addresses with on_device=True, `batch` and optionally `length` (default max_length).  Returns loss float32 [B],
    grad float32 [B, L, 5] (None unless want_grad) and ms, the kernel's device time.  With `out`, a dict of device
    addresses for "loss" and, if wanted, "grad", the results are written there instead and returned as None."""
    lid = logit_loss_id(logit_loss)
    if on_device and batch is None:
      raise ValueError("distill_loss_grad(on_device=True) needs batch")
    t_ptr, teacher = _arg(teacher_logits, np.float32, on_device)
    s_ptr, student = _arg(student_logits, np.float32, on_device)
    if on_device:
      B, L = int(batch), int(length) if length is not None else self.max_length
    elif teacher.ndim != 3 or teacher.shape[2] != 5 or student.shape != teacher.shape:
      raise ValueError("teacher and student logits must both be float32 [B, L, 5], got %s and %s" %
                       (teacher.shape, student.shape))
    else:
      B, L = teacher.shape[:2]
    out_flag, ptrs, res = _outputs(out, dict(loss=(B,), grad=(B, L, 5) if want_grad else None))
    ms = ctypes.c_float()
    self._check(self._lib.dcb_distill_loss_grad(self._handle, t_ptr, s_ptr, B, L, float(temperature), lid,
                                                (DCB_ROWS_ON_DEVICE if on_device else 0) | out_flag, *ptrs,
                                                ctypes.byref(ms)))
    res["ms"] = float(ms.value)
    return res

  def alignment_loss_grad(self, probs, labels, del_cost: Optional[float] = None, loss_reg: Any = "params",
                          band_width: Any = "params", want_grad: bool = True, want_matches: bool = False,
                          on_device: bool = False, batch: Optional[int] = None, length: Optional[int] = None,
                          out: Optional[Dict[str, int]] = None) -> Dict[str, Any]:
    """dcb_alignment_loss_grad: per-window AlignmentLoss, its gradient with respect to probs and the soft alignment
    matches (AlignmentLoss.eval(return_matches=True)).  probs float32 [B, L, 5] and labels uint8 [B, L] are host arrays,
    or device addresses with on_device=True, `batch` and optionally `length` (default max_length).  del_cost / loss_reg
    / band_width default to params.json's, as in evaluate_windows.  Returns loss float32 [B], grad float32 [B, L, 5]
    (None unless want_grad), matches float32 [B, L, L] (None unless want_matches) and ms, the kernel's device time.
    With `out`, a dict of device addresses for "loss" and, as wanted, "grad" / "matches", the results are written
    there instead and returned as None."""
    if on_device and batch is None:
      raise ValueError("alignment_loss_grad(on_device=True) needs batch")
    l_ptr, labels = _arg(labels, np.uint8, on_device)
    if on_device:
      B, L = int(batch), int(length) if length is not None else self.max_length
    elif labels.ndim != 2:
      raise ValueError("labels must be uint8 [B, L], got %s" % (labels.shape,))
    else:
      B, L = labels.shape
    p_ptr, probs = _arg(probs, np.float32, on_device)
    if not on_device and probs.shape != (B, L, 5):
      raise ValueError("probs must be float32 [%d, %d, 5], got %s" % (B, L, probs.shape))
    dc, reg, bw = self._eval_args(del_cost, loss_reg, band_width)
    out_flag, ptrs, res = _outputs(out, dict(loss=(B,), grad=(B, L, 5) if want_grad else None,
                                             matches=(B, L, L) if want_matches else None))
    ms = ctypes.c_float()
    self._check(self._lib.dcb_alignment_loss_grad(self._handle, p_ptr, l_ptr, B, L, dc, reg, bw,
                                                  (DCB_ROWS_ON_DEVICE if on_device else 0) | out_flag, *ptrs,
                                                  ctypes.byref(ms)))
    res["ms"] = float(ms.value)
    return res

  def ccs_ids(self, rows_or_packed: np.ndarray) -> np.ndarray:
    """The CCS row of every window as ids uint8 [B, L] (model_utils.get_ccs_from_example: row 4 * max_passes)."""
    return ccs_ids_from_input(self.params, rows_or_packed)

  def evaluate(self, rows_or_packed: np.ndarray, labels: np.ndarray, strict: Optional[bool] = None,
               del_cost: Optional[float] = None, loss_reg: Any = "params", band_width: Any = "params",
               strict_input: bool = True) -> Dict[str, Any]:
    """Forward + evaluation of labelled windows: float32 rows [B, R, L(,1)] or packed rows uint8 [B, packed bytes],
    labels uint8 [B, L].  The forward writes its probabilities to device memory and dcb_evaluate reads them there;
    they never come back to the host.  Returns evaluate_windows()'s dict (concatenated over max_batch chunks) plus
    forward_ms / eval_ms, the summed device times."""
    x = np.asarray(rows_or_packed)
    packed = x.dtype == np.uint8 and x.ndim == 2
    if packed:
      x = np.ascontiguousarray(x)
      if x.shape[1] != self.packed_window_bytes:
        raise ValueError("packed rows must be uint8 [B, %d]" % self.packed_window_bytes)
    else:
      x = _rows3(self.params, x)
    B, L = x.shape[0], self.max_length
    labels = np.ascontiguousarray(labels, dtype=np.uint8)
    if labels.shape != (B, L):
      raise ValueError("labels must be uint8 [%d, %d]" % (B, L))
    ccs = self.ccs_ids(x)
    mb = min(self.max_batch, max(B, 1))
    d_probs = self.alloc_device(mb * L * 5 * 4)
    d_bq = self.alloc_device(2 * mb * L)
    parts = []
    fwd_ms = eval_ms = 0.0
    try:
      fn = self._lib.dcb_forward_packed if packed else self._lib.dcb_forward
      for b0 in range(0, B, mb):
        b1 = min(B, b0 + mb)
        self._forward_chunk(fn, x[b0:b1], DCB_OUT_ON_DEVICE | self._precision_flag(strict), d_bq, d_bq + mb * L,
                            d_probs, None, strict_input)
        fwd_ms += self.last_forward_ms()
        r = self.evaluate_windows(d_probs, labels[b0:b1], ccs[b0:b1], del_cost, loss_reg, band_width, on_device=True,
                                  batch=b1 - b0)
        eval_ms += r.pop("ms")
        parts.append(r)
    finally:
      self.free_device(d_probs)
      self.free_device(d_bq)
    out = _concat_eval(parts)
    out["forward_ms"], out["eval_ms"] = fwd_ms, eval_ms
    return out

  def predict(self, rows: np.ndarray) -> _Prediction:
    """Softmax output [B, L, 5], shaped like `EncoderOnlyTransformer.predict` (networks.py:357-365)."""
    return _Prediction(self.forward(rows, want_probs=True)["probs"])

  # -- introspection -----------------------------------------------------------------------
  def last_forward_ms(self) -> float:
    v = ctypes.c_float()
    self._check(self._lib.dcb_last_forward_ms(self._handle, ctypes.byref(v)))
    return float(v.value)

  def last_forward_launches(self) -> int:
    v = ctypes.c_int32()
    self._check(self._lib.dcb_last_forward_launches(self._handle, ctypes.byref(v)))
    return int(v.value)

  def set_profile(self, enabled: bool = True) -> None:
    self._check(self._lib.dcb_set_profile(self._handle, int(enabled)))

  def get_profile(self) -> Dict[str, float]:
    ms, n, tok = ctypes.c_float(), ctypes.c_int32(), ctypes.c_int64()
    self._check(self._lib.dcb_get_profile(self._handle, ctypes.byref(ms), ctypes.byref(n),
                                          ctypes.byref(tok)))
    ms6, n6 = (ctypes.c_float * 6)(), (ctypes.c_int32 * 6)()
    self._check(self._lib.dcb_get_profile_kernels(self._handle, ms6, n6))
    names = ("embed", "row_gemm", "qkv_gemm", "attention", "ffn", "head")
    return dict(ffn_ms_total=float(ms.value), ffn_launches=int(n.value), ffn_tokens=int(tok.value),
                kernels={k: dict(ms=float(ms6[i]), launches=int(n6[i])) for i, k in enumerate(names)})

  def set_debug(self, enabled: bool = True) -> None:
    self._check(self._lib.dcb_set_debug(self._handle, int(enabled)))

  def debug_residual(self, stage: int, tokens: int) -> np.ndarray:
    out = np.empty((tokens, 280), np.float32)
    self._check(self._lib.dcb_debug_residual(self._handle, stage, _ptr(out), out.size))
    return out

  def debug_operand(self, stage: int, which: str, tokens: int) -> np.ndarray:
    """dcb_debug_operand: bf16 operand image `which` (a DEBUG_OPERANDS key) captured at `stage`, as raw bf16 bits
    uint16 [tokens, width] at the image's padded width."""
    width = {"embed": (params_lib.embedded_width(self.params) + 15) // 16 * 16, "xb": 288, "qkv": 864, "att": 288,
             "hid": int(self.params.filter_size)}[which]
    out = np.empty((tokens, width), np.uint16)
    self._check(self._lib.dcb_debug_operand(self._handle, stage, DEBUG_OPERANDS[which], _ptr(out), out.size))
    return out

  def debug_capture(self, tokens: int) -> Dict[str, object]:
    """Everything the debug capture kept of the last chunk's `tokens` valid tokens, by stage (include/dcb200_debug.h):
    emb; x, the residual of every stage; xb, the q/k/v or FFN operand by stage; and per layer qkv, att and hid."""
    nl = int(self.params.num_hidden_layers)
    return dict(emb=self.debug_operand(0, "embed", tokens),
                x=[self.debug_residual(s, tokens) for s in range(1 + 2 * nl)],
                xb={s: self.debug_operand(s, "xb", tokens) for s in range(2 * nl)},
                qkv=[self.debug_operand(1 + 2 * n, "qkv", tokens) for n in range(nl)],
                att=[self.debug_operand(1 + 2 * n, "att", tokens) for n in range(nl)],
                hid=[self.debug_operand(2 + 2 * n, "hid", tokens) for n in range(nl)])

  def debug_f32(self, stage: int, which: str, tokens: int) -> np.ndarray:
    """dcb_debug_f32: float32 image `which` (a DEBUG_F32 key) of the last float32 forward's last chunk, captured at
    `stage`, as float32 [tokens, width]."""
    width = {"emb": params_lib.embedded_width(self.params), "hid": int(self.params.filter_size)}.get(which, 280)
    out = np.empty((tokens, width), np.float32)
    self._check(self._lib.dcb_debug_f32(self._handle, stage, DEBUG_F32[which], _ptr(out), out.size))
    return out

  def debug_capture_f32(self, tokens: int) -> Dict[str, object]:
    """Everything the float32 capture kept of the last chunk's `tokens` tokens, shaped like debug_capture's: emb; x,
    the residual of every stage; y, the LayerNorm output by stage (pre-LN models; empty for ReZero); and per layer q,
    k, v, att and hid."""
    nl = int(self.params.num_hidden_layers)
    att_stages, ffn_stages = [1 + 2 * n for n in range(nl)], [2 + 2 * n for n in range(nl)]
    return dict(emb=self.debug_f32(0, "emb", tokens),
                x=[self.debug_f32(s, "x", tokens) for s in range(1 + 2 * nl)],
                y={} if self.params.rezero else {s: self.debug_f32(s, "y", tokens) for s in att_stages + ffn_stages},
                **{k: [self.debug_f32(s, k, tokens) for s in att_stages] for k in ("q", "k", "v", "att")},
                hid=[self.debug_f32(s, "hid", tokens) for s in ffn_stages])

  def debug_head_epilogue(self, logits: np.ndarray) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """dcb_debug_head_epilogue: the head's per-token epilogue (softmax .. ASCII, with this engine's calibration and
    max_base_quality) on final logits float32 [n, 5], no fc1 bias added.  Returns (bases uint8 [n], quals uint8 [n],
    probs float32 [n, 5])."""
    lg = np.ascontiguousarray(logits, dtype=np.float32)
    if lg.ndim != 2 or lg.shape[1] != 5:
      raise ValueError("debug_head_epilogue: logits must be [n, 5]")
    n = int(lg.shape[0])
    bases, quals, probs = np.empty(n, np.uint8), np.empty(n, np.uint8), np.empty((n, 5), np.float32)
    self._check(self._lib.dcb_debug_head_epilogue(self._handle, _ptr(lg), n, _ptr(bases), _ptr(quals), _ptr(probs)))
    return bases, quals, probs

  # -- raw device / pinned buffers (bench, multi-GPU driver) ----------------------------------
  def alloc_device(self, nbytes: int) -> int:
    p = ctypes.c_void_p()
    self._check(self._lib.dcb_alloc_device(self._handle, nbytes, ctypes.byref(p)))
    return p.value

  def free_device(self, ptr: int) -> None:
    self._check(self._lib.dcb_free_device(self._handle, _ptr(ptr)))

  def memcpy_h2d(self, dst: int, src: np.ndarray) -> None:
    src = np.ascontiguousarray(src)
    self._check(self._lib.dcb_memcpy_h2d(self._handle, _ptr(dst), _ptr(src), src.nbytes))

  def memcpy_d2h(self, dst: np.ndarray, src: int) -> None:
    self._check(self._lib.dcb_memcpy_d2h(self._handle, _ptr(dst), _ptr(src), dst.nbytes))

  def submit_raw(self, rows_ptr: int, batch: int, flags: int, bases_ptr: int, quals_ptr: int,
                 probs_ptr: int = 0, logits_ptr: int = 0) -> int:
    """dcb_submit on caller-managed pointers; returns the ticket for wait_raw()."""
    ticket = ctypes.c_int64(-1)
    self._check(self._lib.dcb_submit(self._handle, _ptr(rows_ptr), batch, flags, _ptr(bases_ptr), _ptr(quals_ptr),
                                     _ptr(probs_ptr), _ptr(logits_ptr), ctypes.byref(ticket)))
    return int(ticket.value)

  def wait_raw(self, ticket: int) -> None:
    self._check(self._lib.dcb_wait(self._handle, ticket))

  def forward_raw(self, rows_ptr: int, batch: int, flags: int, bases_ptr: int, quals_ptr: int,
                  probs_ptr: int = 0, logits_ptr: int = 0) -> None:
    """dcb_forward on caller-managed pointers (host or device per `flags`)."""
    self._check(self._lib.dcb_forward(self._handle, _ptr(rows_ptr), batch, flags, _ptr(bases_ptr), _ptr(quals_ptr),
                                      _ptr(probs_ptr), _ptr(logits_ptr)))

  def forward_packed_raw(self, packed_ptr: int, batch: int, flags: int, bases_ptr: int, quals_ptr: int,
                         probs_ptr: int = 0, logits_ptr: int = 0) -> None:
    """dcb_forward_packed on caller-managed pointers (host or device per `flags`)."""
    self._check(self._lib.dcb_forward_packed(self._handle, _ptr(packed_ptr), batch, flags, _ptr(bases_ptr),
                                             _ptr(quals_ptr), _ptr(probs_ptr), _ptr(logits_ptr)))

  def synchronize(self) -> None:
    self._check(self._lib.dcb_synchronize(self._handle))


def packed_window_bytes(params: params_lib.Params) -> int:
  """Bytes per window of the packed row format (include/dcb200.h "packed input rows")."""
  cfg = make_config(params, max_batch=1)
  return int(load_library().dcb_packed_window_bytes(ctypes.byref(cfg)))


def pack_rows(params: params_lib.Params, rows: np.ndarray, out: Optional[np.ndarray] = None,
              strict_input: bool = True) -> np.ndarray:
  """float32 rows [B, R, L(,1)] -> packed uint8 [B, packed_window_bytes] (dcb_pack_rows; host code, needs no GPU).
  Raises DcbError(-5) when a base / strand / ccs / ccs_bq value lies outside its vocabulary (TensorFlow's gather would
  raise) or an SN row is not constant, unless `strict_input` is False (values are clamped either way)."""
  rows = _rows3(params, rows)
  lib, cfg = load_library(), make_config(params, max_batch=1)
  stride = packed_window_bytes(params)
  B = rows.shape[0]
  if out is None:
    out = np.empty((B, stride), np.uint8)
  if out.shape != (B, stride) or out.dtype != np.uint8 or not out.flags.c_contiguous:
    raise ValueError("pack_rows(out=...): need C-contiguous uint8 [%d, %d]" % (B, stride))
  rc = lib.dcb_pack_rows(ctypes.byref(cfg), _ptr(rows), B, _ptr(out))
  if rc and not (rc == -5 and not strict_input):
    raise DcbError(rc, lib.dcb_last_error(None).decode())
  return out


def concat_records(zmws: List[Dict[str, Any]]) -> Dict[str, np.ndarray]:
  """The raw-record bundles of `preprocess.BamFeatureStream.next_zmw_records()` as one dcb_records batch: arrays
  concatenated, per-read offsets shifted, per-ZMW offsets added (and, with smart windows, the `wl` tags with wl_off)."""
  cig0 = np.cumsum([0] + [len(z["cigar"]) for z in zmws])
  q0 = np.cumsum([0] + [len(z["bases"]) for z in zmws])
  meta = []
  for k, z in enumerate(zmws):
    m = np.array(z["read_meta"], np.int32).reshape(-1, READ_META)
    m[:, 0] += cig0[k]
    m[:, 2] += q0[k]
    meta.append(m)
  cat = lambda key, dt, tail=(): (np.concatenate([np.asarray(z[key], dt).reshape((-1,) + tail) for z in zmws])
                                  if zmws else np.zeros((0,) + tail, dt))
  smart = dict(wl_off=np.cumsum([0] + [len(z["wl"]) for z in zmws]).astype(np.int32), wl=cat("wl", np.int32)) \
      if zmws and "wl" in zmws[0] else {}
  return dict(**smart, zmw_read_off=np.cumsum([0] + [len(m) for m in meta]).astype(np.int32),
              zmw_ccs_off=np.cumsum([0] + [len(z["ccs_bases"]) for z in zmws]).astype(np.int32),
              zmw_ccs_bq_any=np.array([int(z["ccs_bq_any"]) for z in zmws], np.int32),
              read_meta=np.concatenate(meta) if meta else np.zeros((0, READ_META), np.int32),
              read_sn=cat("read_sn", np.float32, (4,)), cigar=cat("cigar", np.uint32), bases=cat("bases", np.uint8),
              pw=cat("pw", np.uint8), ip=cat("ip", np.uint8), ccs_bases=cat("ccs_bases", np.uint8), ccs_bq=cat("ccs_bq", np.uint8))


def concat_labels(labels: List[Dict[str, Any]]) -> Dict[str, np.ndarray]:
  """Labels of `preprocess.BamFeatureStream.label()` (one per ZMW, in the order of the records batch) as dcb_labels
  arrays: cigar and bases concatenated, label_meta [n, LABEL_META] with offsets into them."""
  meta = np.zeros((len(labels), LABEL_META), np.int32)
  c0 = b0 = 0
  for i, lab in enumerate(labels):
    meta[i] = (c0, len(lab["cigar"]), b0, len(lab["bases"]), lab["pos"], lab["ccs0"])
    c0 += len(lab["cigar"])
    b0 += len(lab["bases"])
  cat = lambda k, dt: np.concatenate([np.asarray(lab[k], dt) for lab in labels]) if labels else np.zeros(0, dt)
  return dict(label_meta=meta, cigar=cat("cigar", np.uint32), bases=cat("bases", np.uint8))


def pipelined(items: Iterable[Any], submit: Callable[[Any], Any], wait: Callable[[Any], Any],
              retire: Callable[[Any], None]) -> Iterator[Tuple[Any, Any]]:
  """Two submissions in flight: yields (item, wait(submit(item))) in order, submitting item i + 1 before waiting for
  item i, so that the device works on one while the host prepares the next.  If a submit or a wait raises, or the
  consumer closes the generator, every submission not yet waited for is passed to `retire` (which must swallow
  DcbError) before the exception propagates, so the engines' slots are free again."""
  pending = []
  try:
    for item in items:
      pending.append((item, submit(item)))
      if len(pending) == 2:
        done, handle = pending.pop(0)
        yield done, wait(handle)
    while pending:
      done, handle = pending.pop(0)
      yield done, wait(handle)
  finally:
    for _, handle in pending:
      retire(handle)


def _empty_eval(n: int) -> Dict[str, np.ndarray]:
  """Zeroed per-window results of dcb_evaluate for n windows."""
  return dict(loss=np.zeros(n, np.float32), exact=np.zeros(n, np.uint8), pred_counts=np.zeros((n, 5), np.int32),
              ccs_counts=np.zeros((n, 5), np.int32))


def _concat_eval(parts: List[Dict[str, np.ndarray]], extra: Tuple[str, ...] = ()) -> Dict[str, np.ndarray]:
  """Per-chunk evaluate_windows() results, each with float32 [n] arrays `extra` added, concatenated over the chunks;
  empty arrays of the same dtypes when there is no chunk."""
  if not parts:
    parts = [dict(_empty_eval(0), **{k: np.zeros(0, np.float32) for k in extra})]
  return {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}


def unpack_rows(params: params_lib.Params, packed: np.ndarray) -> np.ndarray:
  """The float32 rows [B, R, L] a packed batch stands for (NumPy mirror of csrc/common.h packed_value; tests and
  debugging -- the engine never needs it)."""
  P, L, bq = int(params.max_passes), int(params.max_length), int(bool(params.use_ccs_bq))
  R = 4 * P + 5 + bq
  packed = np.asarray(packed, np.uint8)
  B = packed.shape[0]
  sn_off = ((3 * P + 1 + bq) * L + 15) & ~15
  planes = packed[:, :(3 * P + 1 + bq) * L].reshape(B, 3 * P + 1 + bq, L)
  rows = np.zeros((B, R, L), np.float32)
  rows[:, :P] = planes[:, :P] & 7
  rows[:, P:3 * P] = planes[:, P:3 * P]
  rows[:, 3 * P:4 * P] = (planes[:, :P] >> 3) & 3
  rows[:, 4 * P] = planes[:, 3 * P]
  if bq:
    rows[:, 4 * P + 1] = planes[:, 3 * P + 1].astype(np.float32) - 1
  sn = np.ascontiguousarray(packed[:, sn_off:sn_off + 16]).view(np.float32)
  rows[:, R - 4:] = sn[:, :, None]
  return rows


def ccs_ids_from_input(params: params_lib.Params, rows_or_packed: np.ndarray) -> np.ndarray:
  """The CCS row (row 4 * max_passes, data_providers.get_indices) of float32 rows [B, R, L(,1)] or packed rows
  [B, packed bytes] as uint8 ids [B, L]; values outside 0..4 become 0, the id their all-zero one-hot row decodes to."""
  x = np.asarray(rows_or_packed)
  P, L = int(params.max_passes), int(params.max_length)
  if x.dtype == np.uint8 and x.ndim == 2:
    return np.ascontiguousarray(x[:, 3 * P * L:(3 * P + 1) * L])   # dcb_pack_rows rejects ccs ids outside 0..4
  if x.ndim == 4:
    x = x[..., 0]
  c = x[:, 4 * P, :]
  ok = (c >= 0) & (c <= 4)
  return np.where(ok, np.trunc(np.where(ok, c, 0)), 0).astype(np.uint8)


def logit_loss_id(identifier: Any) -> int:
  """params.logit_loss_identifier (a tf.keras.losses.get identifier) -> DCB_LOGIT_LOSS_*; an int id passes through."""
  if isinstance(identifier, (int, np.integer)) and not isinstance(identifier, bool):
    return int(identifier)
  if identifier not in LOGIT_LOSS_IDS:
    raise ValueError("logit loss %r is not supported: use one of %s" % (identifier, ", ".join(LOGIT_LOSS_IDS)))
  return LOGIT_LOSS_IDS[identifier]


def alloc_pinned(nbytes: int) -> Tuple[int, np.ndarray]:
  """Pinned host buffer as (address, uint8 ndarray view). Free with free_pinned(address)."""
  lib = load_library()
  p = ctypes.c_void_p()
  rc = lib.dcb_alloc_host(nbytes, ctypes.byref(p))
  if rc:
    raise DcbError(rc, "cudaMallocHost failed")
  arr = np.ctypeslib.as_array(ctypes.cast(p, ctypes.POINTER(ctypes.c_uint8)), shape=(nbytes,))
  return p.value, arr


def free_pinned(addr: int) -> None:
  load_library().dcb_free_host(_ptr(addr))
