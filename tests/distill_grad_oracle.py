"""The gradient of the reference's DistillationLoss with respect to the student's logits, in NumPy (test helper):

  distillation_loss_grad(teacher, student, T, logit_loss, dtype)
      float32: the op order of distill_loss_kernel's gradient variant (deepconsensus_b200/csrc/eval_kernels.cu), built
               on oracle/distill.py's float32 softmax;
      float64: the same formulas in float64 from the float32 logits, the reference for error bounds.
  Per position, t = softmax(teacher / T), s = softmax(student / T); the logit loss's gradient with respect to s is
  2 (s - t) / 5 (mean squared error) or -t' / s' (KL divergence, t' and s' clipped to [1e-7, 1]; 0 where s lies outside
  [1e-7, 1], as clip_by_value's gradient), times 1 / L (the mean over the window), then the softmax backward
  (g - sum_c g_c s_c) s and the division by T.  The teacher is a constant.
"""
from __future__ import annotations

from typing import Dict

import numpy as np

from oracle import distill as od

F32 = np.float32


def _softmax64(logits: np.ndarray, temperature: float) -> np.ndarray:
  x = np.asarray(logits, np.float64) / float(F32(temperature))
  e = np.exp(x - x.max(-1, keepdims=True))
  return e / e.sum(-1, keepdims=True)


def distillation_loss64(teacher: np.ndarray, student: np.ndarray, temperature: float, logit_loss: str) -> np.ndarray:
  """DistillationLoss.call in float64: [B]."""
  t, s = _softmax64(teacher, temperature), _softmax64(student, temperature)
  if od.LOGIT_LOSSES[logit_loss] == "mse":
    per_pos = ((s - t) ** 2).mean(-1)
  else:
    eps = float(od.KERAS_EPSILON)
    tc, sc = np.clip(t, eps, 1.0), np.clip(s, eps, 1.0)
    per_pos = (tc * np.log(tc / sc)).sum(-1)
  return per_pos.mean(-1)


def distillation_loss_grad(teacher: np.ndarray, student: np.ndarray, temperature: float = 1.0,
                           logit_loss: str = "kl_divergence", dtype=np.float32) -> Dict[str, np.ndarray]:
  """loss [B] and grad = d loss[b] / d student[b] [B, L, 5], in `dtype` (module docstring); also dlds, the gradient
  with respect to the student's probabilities s (softmax(student / T), returned as s), before the softmax backward."""
  if logit_loss not in od.LOGIT_LOSSES:
    raise ValueError("unsupported logit loss %r" % (logit_loss,))
  kl = od.LOGIT_LOSSES[logit_loss] == "kl"
  L = np.shape(student)[1]
  if dtype == np.float64:
    t, s = _softmax64(teacher, temperature), _softmax64(student, temperature)
    eps = float(od.KERAS_EPSILON)
    if kl:
      g = np.where((s >= eps) & (s <= 1.0), -np.clip(t, eps, 1.0) / np.clip(s, eps, 1.0), 0.0) / L
    else:
      g = 2.0 * (s - t) / 5.0 / L
    grad = (g - (g * s).sum(-1, keepdims=True)) * s / float(F32(temperature))
    return dict(loss=distillation_loss64(teacher, student, temperature, logit_loss), grad=grad, dlds=g, s=s)
  t, s = od.softmax_scaled(teacher, temperature), od.softmax_scaled(student, temperature)
  inv_L = F32(F32(1) / F32(L))
  if kl:
    tc, sc = np.clip(t, od.KERAS_EPSILON, F32(1)), np.clip(s, od.KERAS_EPSILON, F32(1))
    g = np.where((s >= od.KERAS_EPSILON) & (s <= F32(1)), ((-(tc / sc).astype(F32)) * inv_L).astype(F32), F32(0))
  else:
    d = (s - t).astype(F32)
    g = ((((F32(2) * d).astype(F32) / F32(5)).astype(F32)) * inv_L).astype(F32)
  g = g.astype(F32)
  gs = (g * s).astype(F32)
  dot = gs[..., 0]
  for c in range(1, 5):
    dot = (dot + gs[..., c]).astype(F32)
  grad = ((((g - dot[..., None]).astype(F32) * s).astype(F32)) / F32(temperature)).astype(F32)
  return dict(loss=od.distillation_loss(teacher, student, temperature, logit_loss), grad=grad, dlds=g, s=s)
