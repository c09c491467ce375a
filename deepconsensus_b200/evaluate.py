"""Evaluation of a checkpoint on labelled windows (mirror of the reference's models/model_inference.py): the reference's
training-mode tf.Examples in, `inference.csv` and `eval_metrics.json` out.

  python -m deepconsensus_b200.evaluate --checkpoint model_dir/checkpoint-50 --eval_path 'data/eval/*.tfrecord.gz' \\
         --out_dir OUT [--batch_size N --limit N --precision bf16|fp32 --random_weights SEED]

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
"""
from __future__ import annotations

import argparse
import contextlib
import json
import os
import time
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np

from deepconsensus_b200 import engine as engine_lib
from deepconsensus_b200 import inference
from deepconsensus_b200 import params as params_lib
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


def write_inference_csv(path: str, rows: Sequence[Tuple[str, float, float]]) -> None:
  """inference.csv in model_utils.run_inference_and_write_results' layout: header, one line per dataset, blank line."""
  lines = ["dataset,loss,eval/per_example_accuracy\n"] + ["%s,%s,%s\n" % (p, l, a) for p, l, a in rows]
  with open(path, "w") as f:
    f.write("".join(lines))
    f.write("\n")


def evaluate_rows(model: engine_lib.B200Model, rows: np.ndarray, labels: np.ndarray, chunk: int,
                  strict: Optional[bool] = None, teacher: Optional[engine_lib.B200Model] = None,
                  temperature: float = 1.0, logit_loss: Any = "kl_divergence") -> Dict[str, Any]:
  """Per-window evaluation of float32 rows [N, R, L]: per chunk of the rows the forward runs through dcb_submit from the
  pipeline slot's pinned staging (device outputs, two chunks in flight) and dcb_evaluate reads its probabilities on the
  device.  Returns evaluate_windows()'s arrays over all N windows and forward_ms / eval_ms, the summed device times.

  With the `teacher` of a distilled student, the teacher's forward runs from the same pinned rows, and once both are
  done dcb_distill_loss_grad compares the two engines' logits on the device.  This adds distill_loss float32 [N] and
  the teacher's forward and the distillation kernel's device times (teacher_forward_ms, distill_ms)."""
  N, L = rows.shape[0], model.max_length
  ccs = model.ccs_ids(rows)
  flag = engine_lib.DCB_OUT_ON_DEVICE | model._precision_flag(strict)
  engines = [model] if teacher is None else [model, teacher]
  out_bytes = chunk * L * 5 * 4
  owned = []                                            # (engine, device address) of every buffer allocated here
  parts: List[Dict[str, np.ndarray]] = []
  if teacher is None:
    times = dict(forward_ms=0.0, eval_ms=0.0)
  else:
    times = dict(forward_ms=0.0, teacher_forward_ms=0.0, eval_ms=0.0, distill_ms=0.0)

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
    slot, b0, b1 = item
    staging = model.staging_rows(slot)
    staging[:b1 - b0] = rows[b0:b1]
    handle = []
    try:
      for m, buf in zip(engines, bufs[slot]):
        handle.append((m, m.submit_raw(staging.ctypes.data, b1 - b0, flag, buf["bq"], buf["bq"] + chunk * L,
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
    chunks = [(i % 2, b0, min(N, b0 + chunk)) for i, b0 in enumerate(range(0, N, chunk))]
    with contextlib.closing(engine_lib.pipelined(chunks, submit, wait, retire)) as done:   # retired before the frees
      for (slot, b0, b1), _ in done:
        r = model.evaluate_windows(bufs[slot][0]["probs"], labels[b0:b1], ccs[b0:b1], on_device=True, batch=b1 - b0)
        times["eval_ms"] += r.pop("ms")
        if teacher is not None:
          d = model.distill_loss(bufs[slot][1]["logits"], bufs[slot][0]["logits"], temperature, logit_loss,
                                 on_device=True, batch=b1 - b0, length=L)
          times["distill_ms"] += d["ms"]
          r["distill_loss"] = d["loss"]
        parts.append(r)
  finally:
    for m, addr in owned:
      m.free_device(addr)
  out = engine_lib._concat_eval(parts, () if teacher is None else ("distill_loss",))
  out.update(times)
  return out


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


def run(checkpoint: str, eval_path: Sequence[str], out_dir: str, limit: int = -1, batch_size: Optional[int] = None,
        precision: str = "bf16", random_weights: Optional[int] = None, device: int = 0,
        chunk: int = 1024, teacher_model_dir: Optional[str] = None,
        teacher_random_weights: Optional[int] = None) -> Dict[str, Any]:
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
  try:
    for path in eval_path:
      t0 = time.time()
      d = tfrecord.read_examples(path, limit=-1 if limit < 0 else limit * bs)
      rows, labels = d["rows"], d["labels"]
      if rows.shape[0] and rows.shape[1:] != (model.total_rows, model.max_length):
        raise ValueError("%s: windows of shape %s, the checkpoint's params expect [%d, %d]" %
                         (path, rows.shape[1:], model.total_rows, model.max_length))
      t1 = time.time()
      if teacher is None:
        per = evaluate_rows(model, rows, labels, chunk)
      else:
        per = evaluate_rows(model, rows, labels, chunk, teacher=teacher, temperature=float(distill["temperature"]),
                            logit_loss=distill["logit_loss_identifier"])
      agg = aggregate(per["loss"], per["exact"], per["pred_counts"], per["ccs_counts"], bs)
      agg.update(precision=precision, forward_ms=per["forward_ms"], eval_ms=per["eval_ms"],
                 seconds_read=t1 - t0, seconds_model_and_eval=time.time() - t1)
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
  finally:
    model.close()
    if teacher is not None:
      teacher.close()
  write_inference_csv(os.path.join(out_dir, "inference.csv"), csv_rows)
  with open(os.path.join(out_dir, "eval_metrics.json"), "w") as f:
    json.dump(metrics, f, indent=1)
  return metrics


def main(argv: Optional[List[str]] = None) -> None:
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument("--checkpoint", required=True)
  ap.add_argument("--eval_path", required=True, nargs="+", help="glob(s) of labelled *.tfrecord.gz; one csv line each")
  ap.add_argument("--out_dir", required=True)
  ap.add_argument("--limit", type=int, default=-1, help="batches per dataset (-1: all)")
  ap.add_argument("--batch_size", type=int, default=None, help="windows per metric batch (default: params.batch_size)")
  ap.add_argument("--precision", default="bf16", choices=["bf16", "fp32"])
  ap.add_argument("--random_weights", type=int, default=None)
  ap.add_argument("--device", type=int, default=0)
  ap.add_argument("--teacher_model_dir", default=None,
                  help="checkpoint of the teacher of a distilled student: adds the distillation losses")
  ap.add_argument("--teacher_random_weights", type=int, default=None)
  a = ap.parse_args(argv)
  m = run(**vars(a))
  print(json.dumps({p: {k: v for k, v in r.items() if not k.startswith("batch_identity")} for p, r in m.items()}))


if __name__ == "__main__":
  main()
