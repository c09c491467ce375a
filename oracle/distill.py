"""NumPy restatement of the reference's distillation loss and of how its distillation loop aggregates it (test
infrastructure only), pinned against vectors produced by running the reference's own `DistillationLoss`
(scripts/make_distill_golden.py, tests/golden/ref_distill.npz):

  distillation_loss       DistillationLoss.call (losses_and_metrics.py:1170-1213) with the Keras logit losses
                          mean_squared_error and kl_divergence.  Keras is not part of the reference tree, so those two
                          are restated from their documented semantics (keras/losses.py of Keras 2.x):
                          mean_squared_error(y_true, y_pred) = mean(square(y_pred - y_true), axis=-1); kl_divergence
                          clips both arguments to [epsilon(), 1] = [1e-7, 1] and returns
                          sum(y_true * log(y_true / y_pred), axis=-1).  The teacher is y_true.
  distillation_aggregate  the eval step of model_distillation.py (:242-270,320-349): per example
                          student_alpha * student_loss + distill_alpha * distill_loss, per batch
                          tf.nn.compute_average_loss (sum / batch_size), eval/loss the Mean over batches; full batches
                          only (drop_remainder=True)
float32 throughout, with sums over small axes taken in order, left to right.  The student term itself is
oracle/losses.alignment_loss.
"""
from __future__ import annotations

from typing import Dict

import numpy as np

F32 = np.float32
KERAS_EPSILON = F32(1e-7)                    # keras.backend.epsilon()
LOGIT_LOSSES = {"mean_squared_error": "mse", "mse": "mse", "MSE": "mse", "kl_divergence": "kl",
                "kullback_leibler_divergence": "kl", "kld": "kl", "KLD": "kl"}


def _fold_last(x: np.ndarray) -> np.ndarray:
  """Sum over the last axis in order, left to right, in float32."""
  acc = x[..., 0]
  for t in range(1, x.shape[-1]):
    acc = (acc + x[..., t]).astype(F32)
  return acc


def softmax_scaled(logits: np.ndarray, temperature: float) -> np.ndarray:
  """tf.nn.softmax(logits / T, axis=-1) in float32: divide by T, subtract the max, exp, sum in order, divide."""
  x = (np.asarray(logits, F32) / F32(temperature)).astype(F32)
  e = np.exp((x - x.max(-1, keepdims=True)).astype(F32)).astype(F32)
  return (e / _fold_last(e)[..., None]).astype(F32)


def distillation_loss(teacher_logits: np.ndarray, student_logits: np.ndarray, temperature: float = 1.0,
                      logit_loss: str = "kl_divergence") -> np.ndarray:
  """DistillationLoss(temperature, tf.keras.losses.get(logit_loss)).call(teacher, student): float32 [B]."""
  if logit_loss not in LOGIT_LOSSES:
    raise ValueError("unsupported logit loss %r" % (logit_loss,))
  t = softmax_scaled(teacher_logits, temperature)        # y_true
  s = softmax_scaled(student_logits, temperature)        # y_pred
  if LOGIT_LOSSES[logit_loss] == "mse":
    d = (s - t).astype(F32)
    per_pos = (_fold_last((d * d).astype(F32)) / F32(t.shape[-1])).astype(F32)
  else:
    tc = np.clip(t, KERAS_EPSILON, F32(1))
    sc = np.clip(s, KERAS_EPSILON, F32(1))
    per_pos = _fold_last((tc * np.log((tc / sc).astype(F32))).astype(F32))
  return (_fold_last(per_pos) / F32(per_pos.shape[-1])).astype(F32)


def distillation_aggregate(student_loss: np.ndarray, distill_loss: np.ndarray, batch_size: int,
                           student_alpha: float = 1.0, distill_alpha: float = 1.0e5) -> Dict[str, float]:
  """The distillation loop's eval losses over the full batches of per-window values (a ragged tail is dropped):
  loss (eval/loss) = Mean over batches of sum(student_alpha * sl + distill_alpha * dl) / batch_size, and the same for
  each term alone."""
  sl, dl = np.asarray(student_loss, F32), np.asarray(distill_loss, F32)
  n_batches = sl.shape[0] // batch_size
  bs = F32(batch_size)
  sums = {"loss": F32(0), "student_loss": F32(0), "distill_loss": F32(0)}
  for i in range(n_batches):
    s, d = sl[i * batch_size:(i + 1) * batch_size], dl[i * batch_size:(i + 1) * batch_size]
    per_example = ((F32(student_alpha) * s).astype(F32) + (F32(distill_alpha) * d).astype(F32)).astype(F32)
    for k, v in (("loss", per_example), ("student_loss", s), ("distill_loss", d)):
      sums[k] = F32(sums[k] + F32(_fold_last(v) / bs))
  out: Dict[str, float] = {k: float(F32(v / F32(n_batches))) if n_batches else 0.0 for k, v in sums.items()}
  out["n_batches"] = n_batches
  return out
