"""ORACLE -- test infrastructure.  Post-model arithmetic of `run_model_on_examples`.

Restates quick_inference.py:377-389 (argmax / error prob / Phred / calibration /
clip / round / int / floor) and :390-414 (string building) with NumPy, keeping the
reference's dtypes: softmax output float32, `1 - max` and `-10*log10` in float32,
calibration float32 when threshold == 0 and float64 otherwise
(calibration_lib.py:89-99), np.round half-to-even.
"""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np

SEQ_VOCAB = " ATCG"   # dc_constants.py:39-41


def quality_from_probs(probs: np.ndarray, max_base_quality: int = 93,
                       calibration: Optional[Tuple[float, float, float]] = None,
                       log10: str = "libm") -> Tuple[np.ndarray, np.ndarray]:
  """probs [B,L,5] float32 -> (y_preds int64 [B,L], quality int32 [B,L]).

  log10="libm": `np.log10` on the float32 array, as the reference writes it -- the platform's float32 log10 (glibc /
  SVML: <= 1 ulp, not always correctly rounded, so the value is platform-dependent in its last bit).
  log10="exact": the correctly rounded float32 log10 (float64 log10 rounded once) -- the platform-independent
  definition the device epilogue implements (csrc/head_finish.cuh); differs from "libm" only where the platform's
  float32 log10 is off by an ulp AND that ulp crosses a rounding boundary of the final integer.
  """
  probs = np.asarray(probs, dtype=np.float32)
  y_preds = np.argmax(probs, -1)                         # :377
  error_prob = 1 - np.max(probs, axis=-1)                # :378 (float32)
  with np.errstate(divide="ignore"):
    if log10 == "exact":
      q = np.float32(-10) * np.log10(error_prob.astype(np.float64)).astype(np.float32)
    else:
      q = -10 * np.log10(error_prob)                     # :379 (float32; inf when p == 1)
  return y_preds, quality_from_phred(q, max_base_quality, calibration)


def quality_from_phred(q: np.ndarray, max_base_quality: int = 93,
                       calibration: Optional[Tuple[float, float, float]] = None) -> np.ndarray:
  """float32 Phred scores -> integer qualities: calibration, cap, round, clamp at 0 (quick_inference.py:380-389)."""
  q = np.asarray(q, dtype=np.float32)
  if calibration is not None:                            # :380-383
    thr, w, b = calibration
    if thr == 0:
      q = q * w + b
    else:
      q = q * np.where(q > thr, w, 1.0) + np.where(q > thr, b, 0.0)
  q = np.minimum(q, max_base_quality)                    # :385
  q = np.round(q, decimals=0)                            # :386
  q = q.astype(dtype=np.int32)                           # :387
  return np.maximum(q, 0)                                # :389


def fused_calibration_disagreements(w: float, b: float, max_base_quality: int = 93) -> Tuple[np.ndarray, np.ndarray]:
  """Where a threshold-0 calibration of the head depends on its rounding: every float32 pmax in [0.2, 1) whose integer
  quality differs between NumPy's `q * w + b` (float32 product, rounded, then float32 sum) and a fused multiply-add
  (one rounding of the exact q * w + b).  Returns (pmax, q) float32 arrays.

  The exact value is formed in long double: q * w is exact in 48 bits, and q * w + b spans < 64 bits for |q| < 100
  and |b| < 64, so rounding it to float32 once is the fused result.
  """
  if np.finfo(np.longdouble).nmant < 63:
    raise RuntimeError("needs an 80-bit long double")
  lo, hi = np.float32(0.2).view(np.uint32), np.float32(1.0).view(np.uint32)
  p = np.arange(lo, hi, dtype=np.uint32).view(np.float32)
  q = np.float32(-10) * np.log10((np.float32(1) - p).astype(np.float64)).astype(np.float32)
  w32, b32 = np.float32(w), np.float32(b)
  unfused = q * w32 + b32
  fused = (q.astype(np.longdouble) * np.longdouble(w32) + np.longdouble(b32)).astype(np.float32)
  cap = np.float32(max_base_quality)
  final = lambda v: np.maximum(np.rint(np.minimum(v, cap)), 0)         # cap, round half to even, clamp at 0
  diff = final(unfused) != final(fused)
  return p[diff], q[diff]


# Windows whose avg_phred (deepconsensus_b200.utils) sits on a decision threshold, found by search; the skip decision
# and the read quality filter are tested at them.  Each entry (t, a, na, b, nb) is the multiset [a] * na + [b] * nb.
# On an integer t: |avg_phred - t| < 1e-8.
AVG_PHRED_ON_INTEGER = [(16, 6, 16, 26, 160), (24, 14, 19, 34, 190), (31, 11, 2, 41, 220), (31, 11, 2, 51, 200),
                        (46, 36, 19, 56, 190), (47, 37, 11, 67, 100), (51, 41, 2, 61, 20), (65, 55, 19, 75, 190),
                        (79, 69, 10, 89, 100), (80, 70, 23, 90, 230)]
# Within 5e-6 of t - 5e-6, the boundary of round(avg_phred, 5) >= t, on both sides, and inside and outside 1e-7 of it.
AVG_PHRED_AT_ROUNDING_EDGE = [(10, 0, 1, 69, 9), (30, 10, 1, 89, 99), (20, 0, 1, 79, 99), (10, 0, 1, 70, 9)]


def to_strings(y_pred: np.ndarray, quality: np.ndarray) -> Tuple[str, str]:
  """One window: ids -> ' ATCG' string, scores -> Phred+33 string (:408-411, utils.py:60-62)."""
  seq = "".join(SEQ_VOCAB[int(i)] for i in y_pred)
  qual = "".join(chr(int(s) + 33) for s in quality)
  return seq, qual


def to_ascii(y_preds: np.ndarray, quality: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
  """Batch form of to_strings: uint8 [B,L] base characters and Phred+33 characters."""
  vocab = np.frombuffer(SEQ_VOCAB.encode(), dtype=np.uint8)
  return vocab[y_preds], (quality + 33).astype(np.uint8)
