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
"""
from __future__ import annotations

import argparse
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


def write_inference_csv(path: str, rows: Sequence[Tuple[str, float, float]]) -> None:
  """inference.csv in model_utils.run_inference_and_write_results' layout: header, one line per dataset, blank line."""
  lines = ["dataset,loss,eval/per_example_accuracy\n"] + ["%s,%s,%s\n" % (p, l, a) for p, l, a in rows]
  with open(path, "w") as f:
    f.write("".join(lines))
    f.write("\n")


def evaluate_rows(model: engine_lib.B200Model, rows: np.ndarray, labels: np.ndarray, chunk: int,
                  strict: Optional[bool] = None) -> Dict[str, Any]:
  """Per-window evaluation of float32 rows [N, R, L] through dcb_submit (device outputs, two batches in flight) and
  dcb_evaluate on the device probabilities."""
  N, L = rows.shape[0], model.max_length
  ccs = model.ccs_ids(rows)
  flag = engine_lib.DCB_OUT_ON_DEVICE | model._precision_flag(strict)
  d_probs = [model.alloc_device(chunk * L * 5 * 4) for _ in range(2)]
  d_bq = [model.alloc_device(2 * chunk * L) for _ in range(2)]
  parts: List[Dict[str, np.ndarray]] = []
  times = dict(forward_ms=0.0, eval_ms=0.0)

  def finish(p):
    ticket, slot, b0, b1 = p
    model.wait_raw(ticket)
    times["forward_ms"] += model.last_forward_ms()
    r = model.evaluate_windows(d_probs[slot], labels[b0:b1], ccs[b0:b1], on_device=True, batch=b1 - b0)
    times["eval_ms"] += r.pop("ms")
    parts.append(r)

  pending = None
  try:
    for i, b0 in enumerate(range(0, N, chunk)):
      b1, slot = min(N, b0 + chunk), i % 2
      staging = model.staging_rows(slot)
      staging[:b1 - b0] = rows[b0:b1]
      ticket = model.submit_raw(staging.ctypes.data, b1 - b0, flag, d_bq[slot], d_bq[slot] + chunk * L,
                                probs_ptr=d_probs[slot])
      prev, pending = pending, (ticket, slot, b0, b1)
      if prev is not None:
        finish(prev)
    if pending is not None:
      prev, pending = pending, None
      finish(prev)
  finally:
    if pending is not None:
      try:
        model.wait_raw(pending[0])
      except engine_lib.DcbError:
        pass
    for p in d_probs + d_bq:
      model.free_device(p)
  if not parts:
    parts = [dict(loss=np.zeros(0, np.float32), exact=np.zeros(0, np.uint8), pred_counts=np.zeros((0, 5), np.int32),
                  ccs_counts=np.zeros((0, 5), np.int32))]
  out = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
  out.update(times)
  return out


def run(checkpoint: str, eval_path: Sequence[str], out_dir: str, limit: int = -1, batch_size: Optional[int] = None,
        precision: str = "bf16", random_weights: Optional[int] = None, device: int = 0,
        chunk: int = 1024) -> Dict[str, Any]:
  params = params_lib.read_params_from_json(checkpoint)
  if params.get("band_width") is not None:
    raise ValueError("params.band_width=%s: the banded alignment loss is not supported" % params.band_width)
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
      per = evaluate_rows(model, rows, labels, chunk)
      agg = aggregate(per["loss"], per["exact"], per["pred_counts"], per["ccs_counts"], bs)
      agg.update(precision=precision, forward_ms=per["forward_ms"], eval_ms=per["eval_ms"],
                 seconds_read=t1 - t0, seconds_model_and_eval=time.time() - t1)
      csv_rows.append((path, agg["loss"], agg["per_example_accuracy"]))
      metrics[path] = agg
  finally:
    model.close()
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
  a = ap.parse_args(argv)
  m = run(**vars(a))
  print(json.dumps({p: {k: v for k, v in r.items() if not k.startswith("batch_identity")} for p, r in m.items()}))


if __name__ == "__main__":
  main()
