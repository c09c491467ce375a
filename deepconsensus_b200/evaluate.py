"""Evaluation of a checkpoint on labelled windows (mirror of the reference's models/model_inference.py): the reference's
training-mode tf.Examples in, `inference.csv` and `eval_metrics.json` out.

  python -m deepconsensus_b200.evaluate --checkpoint model_dir/checkpoint-50 --eval_path 'data/eval/*.tfrecord.gz' \\
         --out_dir OUT [--batch_size N --limit N --precision bf16|fp32|tf32x3 --random_weights SEED]
  python -m deepconsensus_b200.evaluate --checkpoint model_dir/checkpoint-50 --subreads_to_ccs S.bam --ccs_bam C.bam \\
         --truth_to_ccs T.bam --truth_bed B.bed --truth_split SPLIT.tsv --split eval [--split test] --out_dir OUT \\
         [--ins_trim 5 --cpus N and the options above]

The second form evaluates straight from BAMs: the labelled windows `preprocess` would write to the split's file are
built on the GPU (dcb_features_layout, then dcb_features_eval, which keeps the split's windows and leaves their packed,
label and CCS rows in device memory), scored there and measured there, with no tf.Example in between.  Window geometry
(max_passes, max_length, use_ccs_bq) comes from the checkpoint's params.json; `--ins_trim` and `--cpus` mean what they
mean in `preprocess`.  The dataset name of each split is the split itself, and its `eval_metrics.json` entry gains
"examples": preprocess's counters of the ZMWs read.  The results equal `preprocess` followed by `--eval_path` on the
split's file, window for window.

The forward writes its probabilities to device memory (submit path, two batches in flight) and dcb_evaluate reads them
there: AlignmentLoss, PerExampleAccuracy and the AlignmentMetric counts of the prediction and of the CCS row are
computed per window on the GPU; only those per-window values come back.  Params (del_cost, loss_reg, band_width,
batch_size, geometry) come from the params.json next to the checkpoint.  `--random_weights SEED` replaces the variables
by seeded ones (the reference's bundled test checkpoints ship without their data shard).

Aggregation follows what Keras reports (model.evaluate in model_utils.run_inference_and_write_results, and the metrics
of model_utils.get_deepconsensus_metrics):
  * loss: the mean over all windows (Keras weights its loss tracker by batch size, so the batch means average back to
    the window mean);
  * eval/per_example_accuracy: the fraction of windows whose left-shifted prediction matches the label exactly;
  * identity (batch identity): per_batch_identity per batch of `batch_size` windows, in file order, the last batch kept
    (drop_remainder=False), averaged over batches; identity_ccs the same for the CCS rows;
  * yield_over_ccs: divide_no_nan(#batches with identity >= 0.997, #batches with CCS identity >= 0.997).
`--limit N` takes the first N batches, as the reference's get_dataset applies ds.take(limit) after batching.

Distilled students (the reference's model_distillation.py): `--teacher_model_dir CKPT` (with `--teacher_random_weights
SEED` the counterpart of `--random_weights`) builds the teacher as a second engine on the same device and precision,
from its own params.json; its inputs (max_passes, max_length, use_ccs_bq, the embedding widths and the *_MAX clips) must
be the student's.  Both forwards leave their logits in device memory, dcb_distill_loss_grad compares them there, and
`eval_metrics.json` gains a "distillation" entry per dataset with what the distillation loop's eval step reports
(model_distillation.py:242-270,320-349): per example student_alpha * AlignmentLoss + distill_alpha * DistillationLoss,
per batch their sum / batch_size (tf.nn.compute_average_loss), `loss` (eval/loss) the mean over batches, the same for
`student_loss` and `distill_loss` alone, and the accuracy, identity and yield metrics -- all over FULL batches only, as
create_input_fn batches with drop_remainder=True and get_step_counts counts n // batch_size steps.  distill_alpha,
student_alpha, temperature and logit_loss_identifier come from the student's params.json (defaults: the
transformer_learn_values_distill config).  `inference.csv` and the other entries stay the student-only numbers.

`--calibration` also measures the base-quality calibration of the windows scored (every dataset, summed) and writes
`dc_calibration.csv` and `ccs_calibration.csv` (calculate_baseq_calibration's format) and `calibration.json` to
--out_dir.  dcb_evaluate_calibration walks the same AlignmentMetric traceback as the identity: each base of the argmax
prediction is a match or a mismatch (insertions count as mismatches) in the bin of its uncalibrated head quality, each
base of the CCS row in the bin of its raw CCS base quality, and label bases deleted are only counted.  From the counts
calibration.fit_calibration fits the `threshold,w,b` strings `run --dc_calibration` and `--ccs_calibration` take
(`--calibration_threshold`, `--calibration_min_bases`).  Without the flag every output is unchanged.
"""
from __future__ import annotations

import argparse
import collections
import contextlib
import json
import os
import re
import time
from typing import Any, Dict, Iterable, Iterator, List, Optional, Sequence, Tuple

import numpy as np

from deepconsensus_b200 import calculate_baseq_calibration
from deepconsensus_b200 import calibration as calibration_lib
from deepconsensus_b200 import engine as engine_lib
from deepconsensus_b200 import inference
from deepconsensus_b200 import params as params_lib
from deepconsensus_b200 import preprocess
from deepconsensus_b200 import tfrecord
from deepconsensus_b200 import weights as weights_lib

YIELD_THRESHOLD = 0.997        # YieldOverCCSMetric's default quality_threshold


def per_batch_identity(counts: np.ndarray) -> float:
  """losses_and_metrics.per_batch_identity on [n, 5] counts (EVAL_COUNT_KEYS columns)."""
  tot = int(counts[:, 4].sum())
  if tot == 0:
    return 1.0
  return float(np.float32(int(counts[:, 3].sum()) / tot))


def aggregate(loss: np.ndarray, exact: np.ndarray, pred_counts: np.ndarray, ccs_counts: np.ndarray,
              batch_size: int) -> Dict[str, Any]:
  """Per-window values -> the numbers model.evaluate and the training loop's metrics report (module docstring)."""
  n = int(loss.shape[0])
  ident, ident_ccs = [], []
  for b0 in range(0, n, batch_size):
    ident.append(per_batch_identity(pred_counts[b0:b0 + batch_size]))
    ident_ccs.append(per_batch_identity(ccs_counts[b0:b0 + batch_size]))
  dc = sum(1 for v in ident if np.float32(v) >= YIELD_THRESHOLD)
  cc = sum(1 for v in ident_ccs if np.float32(v) >= YIELD_THRESHOLD)
  return dict(loss=float(np.mean(loss.astype(np.float64))) if n else 0.0,
              per_example_accuracy=float(np.mean(exact.astype(np.float64))) if n else 0.0,
              identity=float(np.mean(ident)) if ident else 0.0,
              identity_ccs=float(np.mean(ident_ccs)) if ident_ccs else 0.0,
              yield_over_ccs=dc / cc if cc else 0.0,
              batch_identity_pred=ident, batch_identity_ccs=ident_ccs,
              n_windows=n, n_batches=len(ident), batch_size=int(batch_size))


# the inputs both models of a distillation pair must agree on: the rows they read and how they embed them
TEACHER_INPUT_KEYS = ("max_passes", "max_length", "use_ccs_bq", "per_base_hidden_size", "pw_hidden_size",
                      "ip_hidden_size", "strand_hidden_size", "ccs_bq_hidden_size", "sn_hidden_size", "PW_MAX",
                      "IP_MAX", "SN_MAX", "CCS_BQ_MAX", "STRAND_MAX")
DISTILL_KEYS = ("distill_alpha", "student_alpha", "temperature", "logit_loss_identifier")


def distill_settings(params: params_lib.Params) -> Dict[str, Any]:
  """The distillation loss parameters of a student's params.json, defaulting to the transformer_learn_values_distill
  config's (model_configs.py:155-190)."""
  defaults = params_lib.get_config("transformer_learn_values_distill+custom")
  return {k: params[k] if params.get(k) is not None else defaults[k] for k in DISTILL_KEYS}


def check_teacher_inputs(student: params_lib.Params, teacher: params_lib.Params) -> None:
  """Raises ValueError naming the first input key on which the teacher's params.json differs from the student's."""
  for k in TEACHER_INPUT_KEYS:
    if student.get(k) != teacher.get(k):
      raise ValueError("teacher params.%s=%r differs from the student's %r: both models must read the same windows" %
                       (k, teacher.get(k), student.get(k)))


def aggregate_distillation(student_loss: np.ndarray, distill_loss: np.ndarray, exact: np.ndarray,
                           pred_counts: np.ndarray, ccs_counts: np.ndarray, batch_size: int, student_alpha: float,
                           distill_alpha: float) -> Dict[str, Any]:
  """Per-window values -> what the distillation loop's eval step reports, over the full batches only (module
  docstring).  The losses are computed in float32, as the loop computes them, with sums taken left to right."""
  f32 = np.float32
  n_batches = int(student_loss.shape[0]) // batch_size
  n = n_batches * batch_size
  sl, dl = np.asarray(student_loss[:n], f32), np.asarray(distill_loss[:n], f32)
  per_example = ((f32(student_alpha) * sl).astype(f32) + (f32(distill_alpha) * dl).astype(f32)).astype(f32)
  out = dict(aggregate(sl, exact[:n], pred_counts[:n], ccs_counts[:n], batch_size))
  for key, v in (("loss", per_example), ("student_loss", sl), ("distill_loss", dl)):
    total = f32(0)                                     # tf.keras.metrics.Mean over the per-batch losses
    for b in range(n_batches):
      s = f32(0)
      for x in v[b * batch_size:(b + 1) * batch_size]:
        s = f32(s + x)
      total = f32(total + f32(s / f32(batch_size)))     # tf.nn.compute_average_loss
    out[key] = float(f32(total / f32(n_batches))) if n_batches else 0.0
  out.update(student_alpha=float(student_alpha), distill_alpha=float(distill_alpha))
  return out


def calibration_summary(counts: np.ndarray, deletions: np.ndarray, windows: int, threshold: float, min_bases: int,
                        params_dc_calibration: Optional[str]) -> Dict[str, Any]:
  """calibration.json: per sequence (dc: the prediction, ccs: the CCS row) its counts [q, match, mismatch], deletions,
  binned bases, the empirical quality [q, E] of the bins the fit uses, and the fitted "threshold,w,b" string, or null
  with the reason in fit_error."""
  out: Dict[str, Any] = dict(windows=int(windows), threshold=float(threshold), min_bases=int(min_bases))
  for which, key in enumerate(("dc", "ccs")):
    c = np.asarray(counts[which], np.int64)
    q, e, _ = calibration_lib.empirical_quality(c, threshold, min_bases)
    entry: Dict[str, Any] = dict(counts=[[i, int(m), int(x)] for i, (m, x) in enumerate(c)],
                                 deletions=int(deletions[which]), bases=int(c.sum()),
                                 empirical=[[int(a), float(b)] for a, b in zip(q, e)])
    try:
      entry["fit"] = calibration_lib.fit_calibration(c, threshold, min_bases)[1]
    except ValueError as err:
      entry["fit"], entry["fit_error"] = None, str(err)
    out[key] = entry
  out["params_dc_calibration"] = params_dc_calibration
  return out


def write_calibration(out_dir: str, counts: np.ndarray, summary: Dict[str, Any]) -> None:
  """dc_calibration.csv, ccs_calibration.csv (calculate_baseq_calibration's CSV) and calibration.json."""
  for which, key in enumerate(("dc", "ccs")):
    with open(os.path.join(out_dir, "%s_calibration.csv" % key), "w") as f:
      f.write(calculate_baseq_calibration.csv_text(counts[which]))
  with open(os.path.join(out_dir, "calibration.json"), "w") as f:
    json.dump(summary, f, indent=1)


def write_inference_csv(path: str, rows: Sequence[Tuple[str, float, float]]) -> None:
  """inference.csv in model_utils.run_inference_and_write_results' layout: header, one line per dataset, blank line."""
  lines = ["dataset,loss,eval/per_example_accuracy\n"] + ["%s,%s,%s\n" % (p, l, a) for p, l, a in rows]
  with open(path, "w") as f:
    f.write("".join(lines))
    f.write("\n")


class HostRowsChunk:
  """One chunk of host float32 rows (the tf.Example path): staged into the pipeline slot's pinned rows and submitted
  with dcb_submit; dcb_evaluate gets its label and CCS rows (and dcb_evaluate_calibration the CCS qualities, uint8
  [n, L] or None) as host arrays."""
  packed, rows_flag, labels_on_device = False, 0, False

  def __init__(self, model: engine_lib.B200Model, rows: np.ndarray, labels: np.ndarray, ccs: np.ndarray,
               ccs_bq: Optional[np.ndarray] = None):
    self.model, self.rows, self.labels, self.ccs_ids, self.ccs_bq = model, rows, labels, ccs, ccs_bq
    self.n = int(rows.shape[0])

  def stage(self, slot: int) -> int:
    staging = self.model.staging_rows(slot)
    staging[:self.n] = self.rows
    return staging.ctypes.data


def host_row_chunks(model: engine_lib.B200Model, rows: np.ndarray, labels: np.ndarray, chunk: int,
                    ccs_bq: Optional[np.ndarray] = None) -> Iterator[HostRowsChunk]:
  """The chunk source of float32 rows [N, R, L] and uint8 labels [N, L] in host memory; ccs_bq (the tf.Examples'
  ccs_base_quality_scores [N, L]) is needed for the calibration counts only."""
  ccs = model.ccs_ids(rows)
  bq = None if ccs_bq is None else engine_lib.ccs_bq_bytes(ccs_bq)
  for b0 in range(0, rows.shape[0], chunk):
    b1 = min(rows.shape[0], b0 + chunk)
    yield HostRowsChunk(model, rows[b0:b1], labels[b0:b1], ccs[b0:b1], None if bq is None else bq[b0:b1])


def evaluate_chunks(model: engine_lib.B200Model, chunks: Iterable[Any], chunk: int, strict: Optional[bool] = None,
                    teacher: Optional[engine_lib.B200Model] = None, temperature: float = 1.0,
                    logit_loss: Any = "kl_divergence", calibration: bool = False) -> Dict[str, Any]:
  """Per-window evaluation of a chunk source: per chunk of at most `chunk` windows the forward runs through the submit
  path (device outputs, two chunks in flight) and dcb_evaluate reads its probabilities on the device.  A chunk has `n`
  windows and `stage(slot)`, which returns the address of its rows: pinned host float32 rows (packed False), or
  device packed rows (packed True, rows_flag DCB_ROWS_ON_DEVICE); its `labels` / `ccs_ids` are host arrays, or device
  addresses with labels_on_device.  Returns evaluate_windows()'s arrays over all windows and forward_ms / eval_ms, the
  summed device times.

  With the `teacher` of a distilled student, the teacher's forward runs from the same rows, and once both are done
  dcb_distill_loss_grad compares the two engines' logits on the device.  This adds distill_loss float32 [N] and the
  teacher's forward and the distillation kernel's device times (teacher_forward_ms, distill_ms).

  With `calibration`, every chunk also has `ccs_bq` beside its CCS rows, and dcb_evaluate_calibration reads the same
  probabilities: this adds calibration_counts int64 [2, CALIB_BINS, 2] and calibration_deletions int64 [2], summed over
  the chunks, and calibration_ms.  Its per-window counts must equal dcb_evaluate's and its binned totals their sums; a
  CCS quality outside 0..99 raises ValueError naming the window (its index among the windows of `chunks`)."""
  L = model.max_length
  flag = engine_lib.DCB_OUT_ON_DEVICE | model._precision_flag(strict)
  engines = [model] if teacher is None else [model, teacher]
  out_bytes = chunk * L * 5 * 4
  owned = []                                            # (engine, device address) of every buffer allocated here
  parts: List[Dict[str, np.ndarray]] = []
  if teacher is None:
    times = dict(forward_ms=0.0, eval_ms=0.0)
  else:
    times = dict(forward_ms=0.0, teacher_forward_ms=0.0, eval_ms=0.0, distill_ms=0.0)
  cal = dict(counts=np.zeros((2, engine_lib.CALIB_BINS, 2), np.int64), deletions=np.zeros(2, np.int64), ms=0.0, w0=0)

  def alloc(m, nbytes):
    owned.append((m, m.alloc_device(nbytes)))
    return owned[-1][1]

  def retire(handle):
    for m, ticket in handle:
      try:
        m.wait_raw(ticket)
      except engine_lib.DcbError:
        pass

  def submit(item):
    """Both engines' forwards of one chunk; if the teacher's submit fails, the student's ticket is retired."""
    slot, c = item
    ptr = c.stage(slot)
    handle = []
    try:
      for m, buf in zip(engines, bufs[slot]):
        fn = m.submit_packed_raw if c.packed else m.submit_raw
        handle.append((m, fn(ptr, c.n, flag | c.rows_flag, buf["bq"], buf["bq"] + chunk * L,
                             probs_ptr=buf.get("probs", 0), logits_ptr=buf.get("logits", 0))))
    except BaseException:
      retire(handle)
      raise
    return handle

  def wait(handle):
    """Waits for the chunk's ticket on every engine (the teacher's also when the student's wait fails)."""
    for i, (m, ticket) in enumerate(handle):
      try:
        m.wait_raw(ticket)
      except BaseException:
        retire(handle[i + 1:])
        raise
    times["forward_ms"] += model.last_forward_ms()
    if teacher is not None:
      times["teacher_forward_ms"] += teacher.last_forward_ms()

  try:
    # per slot and engine: bases and quals, the student's probabilities, and with a teacher both engines' logits
    bufs = [[dict(bq=alloc(m, 2 * chunk * L)) for m in engines] for _ in range(2)]
    for slot in bufs:
      slot[0]["probs"] = alloc(model, out_bytes)
      if teacher is not None:
        slot[0]["logits"], slot[1]["logits"] = alloc(model, out_bytes), alloc(teacher, out_bytes)
    items = ((i % 2, c) for i, c in enumerate(chunks))
    with contextlib.closing(engine_lib.pipelined(items, submit, wait, retire)) as done:   # retired before the frees
      for (slot, c), _ in done:
        r = model.evaluate_windows(bufs[slot][0]["probs"], c.labels, c.ccs_ids, on_device=True, batch=c.n,
                                   labels_on_device=c.labels_on_device)
        times["eval_ms"] += r.pop("ms")
        if calibration:
          add_calibration(model, cal, bufs[slot][0]["probs"], c, r)
        if teacher is not None:
          d = model.distill_loss(bufs[slot][1]["logits"], bufs[slot][0]["logits"], temperature, logit_loss,
                                 on_device=True, batch=c.n, length=L)
          times["distill_ms"] += d["ms"]
          r["distill_loss"] = d["loss"]
        parts.append(r)
  finally:
    for m, addr in owned:
      m.free_device(addr)
  out = engine_lib._concat_eval(parts, () if teacher is None else ("distill_loss",))
  out.update(times)
  if calibration:
    out.update(calibration_counts=cal["counts"], calibration_deletions=cal["deletions"], calibration_ms=cal["ms"])
  return out


def add_calibration(model: engine_lib.B200Model, cal: Dict[str, Any], probs: int, c: Any, r: Dict[str, Any]) -> None:
  """dcb_evaluate_calibration of one chunk whose probabilities are at device address `probs`, added to `cal`; `r` is
  dcb_evaluate's result for the same chunk, which the calibration's per-window counts and totals must agree with."""
  try:
    k = model.evaluate_calibration(probs, c.labels, c.ccs_ids, c.ccs_bq, on_device=True, batch=c.n,
                                   labels_on_device=c.labels_on_device)
  except engine_lib.DcbError as err:
    m = re.search(r"window (\d+) of the batch", str(err))
    if m is None:
      raise
    raise ValueError("window %d: %s" % (cal["w0"] + int(m.group(1)), err)) from err
  for which, key in enumerate(("pred_counts", "ccs_counts")):
    if not np.array_equal(k[key], r[key]):
      raise RuntimeError("dcb_evaluate_calibration's %s differ from dcb_evaluate's" % key)
    nm, ni, nd, nc = (int(v) for v in r[key][:, :4].sum(0))
    got = k["counts"][which].sum(0)
    if (int(got[0]), int(got[1]), int(k["deletions"][which])) != (nc, nm - nc + ni, nd):
      raise RuntimeError("calibration totals (%d, %d, %d) do not match the alignment counts (%d, %d, %d)" %
                         (int(got[0]), int(got[1]), int(k["deletions"][which]), nc, nm - nc + ni, nd))
  cal["counts"] += k["counts"]
  cal["deletions"] += k["deletions"]
  cal["ms"] += k["ms"]
  cal["w0"] += c.n


def evaluate_rows(model: engine_lib.B200Model, rows: np.ndarray, labels: np.ndarray, chunk: int,
                  strict: Optional[bool] = None, teacher: Optional[engine_lib.B200Model] = None,
                  temperature: float = 1.0, logit_loss: Any = "kl_divergence",
                  ccs_bq: Optional[np.ndarray] = None) -> Dict[str, Any]:
  """evaluate_chunks() of float32 rows [N, R, L] and uint8 labels [N, L] in host memory: per chunk the rows go
  through the pipeline slot's pinned staging and dcb_submit.  With ccs_bq (int16 [N, L], the tf.Examples'
  ccs_base_quality_scores) the calibration counts are added."""
  return evaluate_chunks(model, host_row_chunks(model, rows, labels, chunk, ccs_bq), chunk, strict, teacher,
                         temperature, logit_loss, calibration=ccs_bq is not None)


class DevicePackedChunk:
  """One chunk of the BAM path: packed rows, label rows and CCS rows that dcb_features_eval left in device memory, and
  with the calibration counts the CCS qualities beside them (ccs_bq, a device address, else 0)."""
  packed, rows_flag, labels_on_device = True, engine_lib.DCB_ROWS_ON_DEVICE, True

  def __init__(self, packed: int, labels: int, ccs: int, n: int, ccs_bq: int = 0):
    self.packed_ptr, self.labels, self.ccs_ids, self.n, self.ccs_bq = packed, labels, ccs, int(n), ccs_bq

  def stage(self, slot: int) -> int:
    return self.packed_ptr


class BamWindows:
  """The chunk source of the BAM path: the labelled windows of one split, built on the GPU from the subreads and CCS
  BAMs and the truth alignment, in the order `preprocess` writes that split's file.

  ZMWs are decoded (preprocess.BamFeatureStream with `cpus` worker threads), selected by preprocess.select_zmw and laid
  out `batch_zmws` at a time (dcb_features_layout); dcb_features_eval then builds every window's label, keeps the
  windows of the split's ZMWs whose label fits, and writes their packed, label and CCS rows to one of two device
  buffer sets.  Chunks of at most `chunk` windows are slices of that set, so nothing goes through the host.  The sets
  alternate between ZMW batches that keep a window: when a batch is laid out, every chunk of the batch before the
  previous one has been waited for, on both engines.  `counter` receives preprocess's counters of every ZMW read;
  `limit_windows` > 0 stops after that many windows.  With `calibration`, the CCS qualities of the kept windows (the
  layout's ccs_bq, compacted in dcb_features_eval's window order) are copied beside their CCS rows, L bytes each."""

  def __init__(self, model: engine_lib.B200Model, subreads_to_ccs: str, ccs_bam: str, truth_to_ccs: str,
               bed: Dict[str, Dict[str, Any]], contig_split: Dict[str, str], split: str, chunk: int,
               ins_trim: int = 5, cpus: int = 0, batch_zmws: int = 64, limit_windows: int = 0,
               calibration: bool = False):
    self.model, self.split, self.chunk, self.ins_trim = model, split, int(chunk), int(ins_trim)
    self.bed, self.contig_split = bed, contig_split
    self.batch_zmws, self.limit_windows = max(int(batch_zmws), 1), int(limit_windows)
    self.calibration = bool(calibration)
    self.paths = (subreads_to_ccs, ccs_bam, truth_to_ccs)
    self.cpus = max(int(cpus), 0)
    self.counter: collections.Counter = collections.Counter()
    self.features_ms = 0.0
    self.n_windows = 0
    self._sets: List[Optional[Dict[str, int]]] = [None, None]

  def _buffers(self, which: int, n: int) -> Dict[str, int]:
    """Device buffer set `which` with room for n windows (grown, never shrunk)."""
    cur = self._sets[which]
    if cur is not None and cur["cap"] >= n:
      return cur
    self._free(which)
    m, L, cap = self.model, self.model.max_length, max(n, self.chunk)
    self._sets[which] = dict(cap=cap, packed=m.alloc_device(cap * m.packed_window_bytes), labels=m.alloc_device(cap * L),
                             ccs=m.alloc_device(cap * L))
    if self.calibration:
      self._sets[which]["bq"] = m.alloc_device(cap * L)
    return self._sets[which]

  def _free(self, which: int) -> None:
    cur, self._sets[which] = self._sets[which], None
    if cur is not None:
      for k in ("packed", "labels", "ccs", "bq"):
        if k in cur:
          self.model.free_device(cur[k])

  def close(self) -> None:
    for which in (0, 1):
      self._free(which)

  def _batch_chunks(self, batch: List[Tuple[Dict[str, Any], Dict[str, Any], str]], which: int):
    """Lays out one ZMW batch into buffer set `which`; returns its chunks."""
    m, L = self.model, self.model.max_length
    zmws, labels, splits = zip(*batch)
    lay = m.features_layout(engine_lib.concat_records(list(zmws)), self.ins_trim)
    n = len(lay["window_pos"])
    buf = self._buffers(which, n)
    keep = np.array([s == self.split for s in splits], np.uint8)
    r = m.features_eval(engine_lib.concat_labels(list(labels)), keep, buf["cap"], buf["packed"], buf["labels"],
                        buf["ccs"])
    self.features_ms += lay["ms"] + r["ms"]
    w = 0
    for z, s in enumerate(splits):
      n_win = int(lay["zmw_windows"][z])
      preprocess.count_zmw_windows(self.counter, L, n_win, int(r["ccs_width"][z]), r["status"][w:w + n_win], s)
      w += n_win
    k = r["k"]
    if self.limit_windows:
      k = min(k, self.limit_windows - self.n_windows)
    self.n_windows += k
    if self.calibration and k:
      m.memcpy_h2d(buf["bq"], engine_lib.ccs_bq_bytes(lay["ccs_bq"][r["windows"][:k]]))
    stride = m.packed_window_bytes
    return [DevicePackedChunk(buf["packed"] + j0 * stride, buf["labels"] + j0 * L, buf["ccs"] + j0 * L,
                              min(k, j0 + self.chunk) - j0, buf["bq"] + j0 * L if self.calibration else 0)
            for j0 in range(0, k, self.chunk)]

  def __iter__(self) -> Iterator[DevicePackedChunk]:
    stream = preprocess.BamFeatureStream(self.paths[0], self.paths[1], self.model.params.max_passes,
                                         self.model.max_length, bool(self.model.params.use_ccs_bq), self.ins_trim,
                                         threads=self.cpus, records=True, truth_to_ccs=self.paths[2])
    which, batch = 0, []
    try:
      while not (self.limit_windows and self.n_windows >= self.limit_windows):
        z = stream.next_zmw_records()
        if z is not None:
          picked = preprocess.select_zmw(stream, z, self.ins_trim, self.counter, self.bed, self.contig_split)
          if picked is not None:
            batch.append((z,) + picked)
          if len(batch) < self.batch_zmws:
            continue
        if batch:
          chunks = self._batch_chunks(batch, which)
          batch = []
          if chunks:
            which ^= 1
          yield from chunks
        if z is None:
          break
    finally:
      stream.close()


def _load_teacher(teacher_model_dir: str, options: inference.InferenceOptions, random_weights: Optional[int],
                  device: int, precision: str) -> engine_lib.B200Model:
  """The teacher engine: its own params.json (layer count and filter size may differ), the student's options."""
  tparams = params_lib.read_params_from_json(teacher_model_dir)
  weights = None
  if random_weights is not None:
    params_lib.modify_params(tparams, max_length=options.max_length)
    weights = weights_lib.init_weights(tparams, seed=random_weights)
  model, _ = inference.initialize_model(teacher_model_dir, tparams, options, weights=weights, device=device,
                                        precision=precision)
  return model


def check_bam_source(eval_path: Optional[Sequence[str]], subreads_to_ccs: Optional[str], ccs_bam: Optional[str],
                     truth_to_ccs: Optional[str], truth_bed: Optional[str], truth_split: Optional[str],
                     split: Optional[Sequence[str]], use_ccs_smart_windows: bool = False) -> Optional[Dict[str, Any]]:
  """Checks the input form before any decoding starts: tf.Example files (`eval_path`, returns None) or the BAM source
  (returns dict(bed, contig_split)), never both.  The BAM source needs all five inputs and at least one --split, every
  one a split truth_split gives some contig; smart windows are refused, as in training-mode preprocess."""
  bam = dict(subreads_to_ccs=subreads_to_ccs, ccs_bam=ccs_bam, truth_to_ccs=truth_to_ccs, truth_bed=truth_bed,
             truth_split=truth_split)
  given = [k for k, v in bam.items() if v]
  if eval_path and (given or split):
    raise ValueError("--eval_path and the BAM inputs (%s) are exclusive: evaluate either tf.Examples or BAMs" %
                     ", ".join("--" + k for k in given + (["split"] if split else [])))
  if eval_path:
    if use_ccs_smart_windows:
      raise ValueError("--use_ccs_smart_windows applies to the BAM inputs only")
    return None
  if not given and not split:
    raise ValueError("give either --eval_path or the BAM inputs (--subreads_to_ccs --ccs_bam --truth_to_ccs "
                     "--truth_bed --truth_split --split)")
  missing = [k for k in bam if not bam[k]]
  if missing:
    raise ValueError("the BAM inputs also need %s" % ", ".join("--" + k for k in missing))
  if use_ccs_smart_windows:
    raise ValueError("--use_ccs_smart_windows is not supported with the truth inputs (labelled windows are cut every "
                     "max_length columns, as training-mode preprocess cuts them)")
  if not split:
    raise ValueError("the BAM inputs need at least one --split")
  contig_split = preprocess.read_truth_split(truth_split)
  produced = sorted(set(contig_split.values()))
  for sp in split:
    if sp not in produced:
      raise ValueError("--split %s: %s assigns its contigs only to %s" % (sp, truth_split, ", ".join(produced) or "no split"))
  return dict(bed=preprocess.read_truth_bed(truth_bed), contig_split=contig_split)


def run(checkpoint: str, eval_path: Optional[Sequence[str]] = None, out_dir: str = ".", limit: int = -1,
        batch_size: Optional[int] = None, precision: str = "bf16", random_weights: Optional[int] = None,
        device: int = 0, chunk: int = 1024, teacher_model_dir: Optional[str] = None,
        teacher_random_weights: Optional[int] = None, subreads_to_ccs: Optional[str] = None,
        ccs_bam: Optional[str] = None, truth_to_ccs: Optional[str] = None, truth_bed: Optional[str] = None,
        truth_split: Optional[str] = None, split: Optional[Sequence[str]] = None, ins_trim: int = 5, cpus: int = 0,
        batch_zmws: int = 64, use_ccs_smart_windows: bool = False, calibration: bool = False,
        calibration_threshold: float = 0.0, calibration_min_bases: int = 1000) -> Dict[str, Any]:
  truth = check_bam_source(eval_path, subreads_to_ccs, ccs_bam, truth_to_ccs, truth_bed, truth_split, split,
                           use_ccs_smart_windows)
  if truth is not None and cpus == 1:
    raise ValueError("Must set cpus to 0 or >=2 for parallel processing.")
  params = params_lib.read_params_from_json(checkpoint)
  if params.get("band_width") is not None:
    raise ValueError("params.band_width=%s: the banded alignment loss is not supported" % params.band_width)
  distill = None
  if teacher_random_weights is not None and teacher_model_dir is None:
    raise ValueError("--teacher_random_weights needs --teacher_model_dir")
  if teacher_model_dir is not None:
    distill = distill_settings(params)
    engine_lib.logit_loss_id(distill["logit_loss_identifier"])      # an unsupported identifier fails before any work
    check_teacher_inputs(params, params_lib.read_params_from_json(teacher_model_dir))
  bs = int(batch_size or params.get("batch_size", 1))
  options = inference.InferenceOptions(
      max_length=int(params.max_length), example_height=params_lib.get_total_rows(params.max_passes, params.use_ccs_bq),
      max_passes=int(params.max_passes), min_quality=0, min_length=0, batch_size=int(chunk),
      use_ccs_bq=bool(params.use_ccs_bq), cpus=0, skip_windows_above=0, use_saved_model=False, max_base_quality=93,
      dc_calibration_values=None, ccs_calibration_values=None)
  weights = None
  if random_weights is not None:
    params_lib.modify_params(params, max_length=options.max_length)
    weights = weights_lib.init_weights(params, seed=random_weights)
  model, params = inference.initialize_model(checkpoint, params, options, weights=weights, device=device,
                                             precision=precision)
  teacher = None
  if distill is not None:
    try:
      teacher = _load_teacher(teacher_model_dir, options, teacher_random_weights, device, precision)
    except BaseException:
      model.close()
      raise
  os.makedirs(out_dir, exist_ok=True)
  csv_rows, metrics = [], {}
  cal_counts, cal_deletions, cal_windows = np.zeros((2, engine_lib.CALIB_BINS, 2), np.int64), np.zeros(2, np.int64), 0
  kw = {} if teacher is None else dict(teacher=teacher, temperature=float(distill["temperature"]),
                                       logit_loss=distill["logit_loss_identifier"])
  try:
    for path in (eval_path if truth is None else split):
      t0 = time.time()
      if truth is None:
        d = tfrecord.read_examples(path, limit=-1 if limit < 0 else limit * bs)
        rows, labels = d["rows"], d["labels"]
        if rows.shape[0] and rows.shape[1:] != (model.total_rows, model.max_length):
          raise ValueError("%s: windows of shape %s, the checkpoint's params expect [%d, %d]" %
                           (path, rows.shape[1:], model.total_rows, model.max_length))
        t1 = time.time()
        per = evaluate_rows(model, rows, labels, chunk, ccs_bq=d["ccs_base_quality_scores"] if calibration else None,
                            **kw)
        timing = dict(seconds_read=t1 - t0, seconds_model_and_eval=time.time() - t1)
      else:
        source = BamWindows(model, subreads_to_ccs, ccs_bam, truth_to_ccs, truth["bed"], truth["contig_split"], path,
                            chunk, ins_trim=ins_trim, cpus=cpus, batch_zmws=batch_zmws,
                            limit_windows=0 if limit < 0 else limit * bs, calibration=calibration)
        try:
          per = evaluate_chunks(model, source, chunk, calibration=calibration, **kw)
        finally:
          source.close()
        timing = dict(features_ms=source.features_ms, seconds=time.time() - t0)
      agg = aggregate(per["loss"], per["exact"], per["pred_counts"], per["ccs_counts"], bs)
      agg.update(precision=precision, forward_ms=per["forward_ms"], eval_ms=per["eval_ms"], **timing)
      if truth is not None:
        agg["examples"] = dict(source.counter.items())
      if teacher is not None:
        dist = aggregate_distillation(per["loss"], per["distill_loss"], per["exact"], per["pred_counts"],
                                      per["ccs_counts"], bs, float(distill["student_alpha"]),
                                      float(distill["distill_alpha"]))
        dist.update(temperature=float(distill["temperature"]), logit_loss=distill["logit_loss_identifier"],
                    student_forward_ms=per["forward_ms"], teacher_forward_ms=per["teacher_forward_ms"],
                    eval_ms=per["eval_ms"], distill_ms=per["distill_ms"])
        agg["distillation"] = dist
      csv_rows.append((path, agg["loss"], agg["per_example_accuracy"]))
      metrics[path] = agg
      if calibration:
        cal_counts += per["calibration_counts"]
        cal_deletions += per["calibration_deletions"]
        cal_windows += int(per["loss"].shape[0])
  finally:
    model.close()
    if teacher is not None:
      teacher.close()
  write_inference_csv(os.path.join(out_dir, "inference.csv"), csv_rows)
  with open(os.path.join(out_dir, "eval_metrics.json"), "w") as f:
    json.dump(metrics, f, indent=1)
  if calibration:
    write_calibration(out_dir, cal_counts, calibration_summary(cal_counts, cal_deletions, cal_windows,
                                                               calibration_threshold, calibration_min_bases,
                                                               params.get("dc_calibration")))
  return metrics


def main(argv: Optional[List[str]] = None) -> None:
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument("--checkpoint", required=True)
  ap.add_argument("--eval_path", nargs="+", help="glob(s) of labelled *.tfrecord.gz; one csv line each")
  bam = ap.add_argument_group("BAM inputs", "labelled windows built on the GPU, as training-mode preprocess builds them "
                              "(exclusive with --eval_path)")
  bam.add_argument("--subreads_to_ccs")
  bam.add_argument("--ccs_bam")
  bam.add_argument("--truth_to_ccs", help="truth alignment to the CCS reads, indexed (path + .bai)")
  bam.add_argument("--truth_bed")
  bam.add_argument("--truth_split")
  bam.add_argument("--split", action="append", help="split to evaluate (train / eval / test); repeat for one csv line "
                                                    "each")
  bam.add_argument("--ins_trim", type=int, default=5)
  bam.add_argument("--cpus", type=int, default=0, help="host threads that decode and validate the BAMs (0: none)")
  bam.add_argument("--use_ccs_smart_windows", action="store_true", help="not supported: refused")
  ap.add_argument("--out_dir", required=True)
  ap.add_argument("--limit", type=int, default=-1, help="batches per dataset (-1: all)")
  ap.add_argument("--batch_size", type=int, default=None, help="windows per metric batch (default: params.batch_size)")
  ap.add_argument("--precision", default="bf16", choices=["bf16", "fp32", "tf32x3"])
  ap.add_argument("--random_weights", type=int, default=None)
  ap.add_argument("--device", type=int, default=0)
  ap.add_argument("--teacher_model_dir", default=None,
                  help="checkpoint of the teacher of a distilled student: adds the distillation losses")
  ap.add_argument("--teacher_random_weights", type=int, default=None)
  ap.add_argument("--calibration", action="store_true",
                  help="also write dc_calibration.csv, ccs_calibration.csv and calibration.json (fitted threshold,w,b)")
  ap.add_argument("--calibration_threshold", type=float, default=0.0,
                  help="fit only bins above this quality, the threshold of the fitted string (0: every bin)")
  ap.add_argument("--calibration_min_bases", type=int, default=1000, help="fit only bins with at least this many bases")
  a = ap.parse_args(argv)
  try:
    check_bam_source(a.eval_path, a.subreads_to_ccs, a.ccs_bam, a.truth_to_ccs, a.truth_bed, a.truth_split, a.split,
                     a.use_ccs_smart_windows)
  except ValueError as e:
    ap.error(str(e))
  if a.eval_path is None and a.cpus == 1:
    ap.error("Must set cpus to 0 or >=2 for parallel processing.")
  m = run(**vars(a))
  print(json.dumps({p: {k: v for k, v in r.items() if not k.startswith("batch_identity")} for p, r in m.items()}))


if __name__ == "__main__":
  main()
