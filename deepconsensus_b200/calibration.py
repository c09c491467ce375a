"""Base-quality calibration (mirror of `quality_calibration/calibration_lib.py:35-99`).

The device epilogue applies the same linear map (csrc/head_finish.cuh, csrc/post_kernels.cu); this module
is the host-side parser plus a NumPy implementation for skipped windows and tests, and fit_calibration, which fits
the map's w and b to calibration counts.
"""
from __future__ import annotations

import dataclasses
from typing import Tuple

import numpy as np


@dataclasses.dataclass
class QualityCalibrationValues:
  """enabled / threshold / w / b, as in calibration_lib.py:35-50."""
  enabled: bool
  threshold: float
  w: float
  b: float


def parse_calibration_string(calibration: str) -> QualityCalibrationValues:
  """'skip' or 'threshold,w,b' (calibration_lib.py:52-75)."""
  if calibration == "skip":
    return QualityCalibrationValues(enabled=False, threshold=0.0, w=1.0, b=0.0)
  fields = calibration.split(",")
  if len(fields) != 3:
    raise ValueError(
        ("Malformed calibration string. Expected 3 values (or set "
         'to "skip" to perform no quality calibration).'), calibration)
  t, w, b = (float(x) for x in fields)
  return QualityCalibrationValues(enabled=True, threshold=t, w=w, b=b)


def calibrate_quality_scores(quality_scores: np.ndarray,
                             calibration_values: QualityCalibrationValues) -> np.ndarray:
  """q*w+b for every score (threshold==0) or only where q > threshold (calibration_lib.py:77-99).

  dtype behaviour is the reference's: with threshold==0 a float32 input stays
  float32 (python-scalar multiply); otherwise np.where yields float64 factors.
  """
  cv = calibration_values
  if cv.threshold == 0:
    return quality_scores * cv.w + cv.b
  above = quality_scores > cv.threshold
  return quality_scores * np.where(above, cv.w, 1.0) + np.where(above, cv.b, 0.0)


def empirical_quality(counts: np.ndarray, threshold: float = 0.0,
                      min_bases: int = 1000) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
  """The bins fit_calibration uses, from int64 [100, 2] (match, mismatch) counts per quality (calculate_baseq_calibration
  or `evaluate --calibration`): bins q with match + mismatch >= min_bases, mismatch >= 1 and, when threshold > 0,
  q > threshold (the bins calibrate_quality_scores would change).  Returns q int64 [k], the empirical quality
  E(q) = -10 log10(mismatch / total) float64 [k] and the mismatches int64 [k]."""
  c = np.asarray(counts)
  if c.ndim != 2 or c.shape[1] != 2:
    raise ValueError("counts must be [bins, 2] (match, mismatch), got shape %s" % (c.shape,))
  c = c.astype(np.int64)
  q = np.arange(c.shape[0], dtype=np.int64)
  total, mismatch = c[:, 0] + c[:, 1], c[:, 1]
  use = (total >= min_bases) & (mismatch >= 1)
  if threshold > 0:
    use &= q > threshold
  q, total, mismatch = q[use], total[use], mismatch[use]
  return q, -10.0 * np.log10(mismatch / total), mismatch


def fit_calibration(counts: np.ndarray, threshold: float = 0.0,
                    min_bases: int = 1000) -> Tuple[QualityCalibrationValues, str]:
  """The linear map `run` applies (calibrate_quality_scores) fitted to calibration counts: w, b of the weighted least
  squares line E(q) ~ w q + b over empirical_quality's bins, each weighted by its mismatch count (about the inverse
  variance of a log binomial proportion).  Returns the values and their "threshold,w,b" string, which
  parse_calibration_string reads back to the same doubles.  ValueError when fewer than two bins are usable."""
  q, e, wt = empirical_quality(counts, threshold, min_bases)
  if len(q) < 2:
    c = np.asarray(counts).astype(np.int64)
    raise ValueError("calibration fit needs at least two quality bins with >= %d bases and a mismatch%s; usable bins: "
                     "%s (of %d bins with bases, %d bases, %d mismatches)" %
                     (min_bases, " above threshold %g" % threshold if threshold > 0 else "", q.tolist(),
                      int((c.sum(1) > 0).sum()), int(c.sum()), int(c[:, 1].sum())))
  x, wt = q.astype(np.float64), wt.astype(np.float64)
  mx, my = np.sum(wt * x) / np.sum(wt), np.sum(wt * e) / np.sum(wt)
  w = float(np.sum(wt * (x - mx) * (e - my)) / np.sum(wt * (x - mx) ** 2))
  b = float(my - w * mx)
  values = QualityCalibrationValues(enabled=True, threshold=float(threshold), w=w, b=b)
  return values, "%r,%r,%r" % (float(threshold), w, b)
