"""Agreement statistics between two scorings of the same windows (e.g. the engine's default bf16 path against its
strict-fp32 path, or either against reference vectors).

The reference's bar for this path is "identical argmax bases" with per-base qualities computed from the same
probabilities (quick_inference.py:377-389).  `compare` reports how far two outputs are from that: the share of
identical base calls over ALL positions and over the positions whose reference top-2 logit margin exceeds a
threshold, the share of identical quality characters, the largest quality difference, and logit errors.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import numpy as np


def top2_margin(logits: np.ndarray) -> np.ndarray:
  """Difference between the largest and second largest logit per position ([..., 5] -> [...])."""
  srt = np.sort(np.asarray(logits, np.float32), axis=-1)
  return srt[..., -1] - srt[..., -2]


def compare(test: Dict[str, np.ndarray], ref: Dict[str, np.ndarray], margin: float = 1e-3) -> Dict[str, float]:
  """`test` / `ref`: dicts with uint8 `bases`, `quals` [B, L] and optionally float32 `logits` [B, L, 5]
  (margins and logit errors need `ref["logits"]`; logit errors also `test["logits"]`)."""
  tb, rb = np.asarray(test["bases"]), np.asarray(ref["bases"])
  tq, rq = np.asarray(test["quals"]).astype(np.int32), np.asarray(ref["quals"]).astype(np.int32)
  same = tb == rb
  out: Dict[str, float] = dict(
      positions=int(same.size),
      bases_identical_pct=100.0 * float(same.mean()) if same.size else 100.0,
      base_mismatches=int((~same).sum()),
      qv_exact_pct=100.0 * float((tq == rq).mean()) if same.size else 100.0,
      max_dq=int(np.abs(tq - rq).max()) if same.size else 0,
      qv_within_1_pct=100.0 * float((np.abs(tq - rq) <= 1).mean()) if same.size else 100.0)
  if "logits" in ref:
    m = top2_margin(ref["logits"])
    safe = m > margin
    out["margin"] = float(margin)
    out["safe_positions"] = int(safe.sum())
    out["base_mismatches_outside_margin"] = int((~same & safe).sum())
    out["largest_margin_of_a_mismatch"] = float(m[~same].max()) if (~same).any() else 0.0
    out["max_dq_outside_margin"] = int(np.abs(tq - rq)[safe].max()) if safe.any() else 0
    if "logits" in test:
      d = np.asarray(test["logits"], np.float64) - np.asarray(ref["logits"], np.float64)
      out["max_logit_err"] = float(np.abs(d).max()) if d.size else 0.0
      out["rms_logit_err"] = float(np.sqrt((d * d).mean())) if d.size else 0.0
      # How many argmax flips the measured logit error predicts: a position flips when the error of the difference of
      # its two leading logits (sd = sqrt(2) * rms for independent errors) exceeds the reference margin.  Near-ties
      # are a property of the model's margins, not of the arithmetic; this puts the mismatch count on that scale.
      sd = math.sqrt(2.0) * out["rms_logit_err"]
      out["expected_flips"] = float(sum(0.5 * math.erfc(x / (sd * math.sqrt(2.0))) for x in m.ravel().tolist())) if sd > 0 else 0.0
  return out


def summary(stats: Dict[str, float], digits: int = 4) -> Dict[str, float]:
  """The four parity numbers that travel with every throughput number (+ their context)."""
  keys = ("bases_identical_pct", "qv_exact_pct", "max_dq", "max_logit_err", "rms_logit_err", "positions",
          "base_mismatches", "base_mismatches_outside_margin", "largest_margin_of_a_mismatch", "margin", "expected_flips")
  return {k: (round(v, digits) if isinstance(v, float) else v) for k, v in stats.items() if k in keys}
