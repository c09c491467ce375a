"""Base-quality calibration counts of labelled windows, restated literally (what dcb_evaluate_calibration computes).

The alignment is oracle/losses.py's alignment_metric: the same forward recursion over anti-diagonals (affine gaps,
first-max tie-breaking in the order [match, ins, del]) and the same traceback.  Here the traceback also records each
step's cell and edge, so every base of the left-shifted aligned sequence is classified as
calculate_baseq_calibration classifies a read's M / I / D operations:
  edge 1 at (i, j), label base i - 1 equal to base j - 1   match
  edge 1 with a different label base, edges 2 and 3        mismatch
  edges 4 and 5                                            a deletion of label base i - 1 (no quality)
Each base keeps the quality of the position it came from through the left shift.  The prediction's quality is the
head's uncalibrated epilogue (csrc/head_finish.cuh): -10 log10(1 - p_max) in float32 from a float64 log10, capped at 93
with fminf (so NaN, from rows that sum above 1, caps too), rounded half to even, clamped at 0."""
from typing import Dict, List, Tuple

import numpy as np

from oracle import losses as ol

BINS = 100
MAX_Q = 93
F32 = np.float32


def pred_quality(probs: np.ndarray) -> np.ndarray:
  """int [..., L] head quality of every probability row [..., L, 5], without calibration."""
  p = np.asarray(probs, F32)
  err = (F32(1.0) - p.max(-1)).astype(F32)
  with np.errstate(divide="ignore", invalid="ignore"):     # p_max = 1 gives +inf, p_max > 1 NaN: both cap (fminf)
    qf = (F32(-10.0) * np.log10(err.astype(np.float64)).astype(F32)).astype(F32)
  return np.maximum(np.rint(np.fmin(qf, F32(MAX_Q))), 0).astype(np.int64)


def _shift_with_source(ids: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
  """left_shift of one row, and the original position of every non-gap id in order."""
  src = np.flatnonzero(ids != ol.GAP)
  out = np.zeros_like(ids)
  out[:len(src)] = ids[src]
  return out, src


def traceback_steps(y_true: np.ndarray, x_ids: np.ndarray) -> List[List[Tuple[int, int, int]]]:
  """Per window the (i, j, edge) of every traceback step of AlignmentMetric.alignment on label ids [B, m] and decoded ids
  [B, n], in the order the walk takes them (from the end).  The recursion is alignment_metric's, step for step."""
  y = ol.left_shift(np.asarray(y_true).astype(np.int32))
  x = ol.left_shift(np.asarray(x_ids).astype(np.int32))
  B, m = y.shape
  n = x.shape[1]
  tl, pl = (y != ol.GAP).sum(-1), (x != ol.GAP).sum(-1)
  NEG = -ol.INF
  go, ge = F32(5.0 + 4.0), F32(4.0)
  gap_pens = np.array([go, go, ge], F32)[:, None, None]
  subs = np.where(y[:, :, None] == x[:, None, :], F32(2.0), F32(-5.0)).astype(F32)

  def wf(k):
    i = np.arange(m)
    j = k - i
    ok = (j >= 0) & (j < n)
    return np.where(ok[:, None], subs[:, i, np.clip(j, 0, n - 1)].T, F32(0)).astype(F32)

  v_p2 = np.full((3, m, B), NEG, F32)
  v_p2[0, 0] = 0
  v_p1 = np.full((3, m + 1, B), NEG, F32)
  v_p1[1, 0] = -go
  v_p1[2, 1] = -go
  dirs = np.full((m + n + 1, 3, m + 1, B), -2, np.int32)
  dirs[0, 0, 0] = -1
  dirs[1, 1, 0] = 0
  dirs[1, 2, 1] = 0
  m_opt = np.full(B, -1, np.int32)
  i_range = np.arange(m + 1)
  k_end = tl + pl
  bidx = np.arange(B)
  m_opt = np.where(k_end == 1, v_p1[:, tl, bidx].argmax(0), m_opt)
  for k in range(2, m + n + 1):
    valid = (((k - i_range) >= 0) & ((k - i_range) <= n))[None, :, None]
    o_match = (v_p2 + wf(k - 2)[None]).astype(F32)
    o_ins = (v_p1[:2] - gap_pens[1:]).astype(F32)
    v_p2 = v_p1[:, :-1]
    o_del = (v_p2 - gap_pens).astype(F32)
    vm, dm = o_match.max(0), o_match.argmax(0)
    vi, di = o_ins.max(0), o_ins.argmax(0)
    vd, dd = o_del.max(0), o_del.argmax(0)
    vm = np.concatenate([np.full((1, B), NEG, F32), vm])
    vd = np.concatenate([np.full((1, B), NEG, F32), vd])
    dm = np.concatenate([np.full((1, B), -2), dm])
    dd = np.concatenate([np.full((1, B), -2), dd])
    v_p1 = np.where(valid, np.stack([vm, vi, vd]), NEG).astype(F32)
    dirs[k] = np.stack([dm, di, dd])
    m_opt = np.where(k_end == k, v_p1[:, tl, bidx].argmax(0), m_opt).astype(np.int32)

  steps_k, steps_i = (-2, -1, -1), (-1, 0, -1)
  trans_enc = ((1, 1, 1), (2, 3, 2), (4, 4, 5))
  out = []
  for b in range(B):
    k_opt, i_opt, s = int(k_end[b]), int(tl[b]), int(m_opt[b])
    steps = []
    for k in range(m + n, -1, -1):
      if k_opt != k:
        continue
      ss = max(s, 0)
      s_n = int(dirs[k, ss, max(i_opt, 0), b])
      if s_n == -1:
        break
      steps.append((i_opt, k_opt - i_opt, trans_enc[ss][max(s_n, 0)]))
      k_opt, i_opt, s = k_opt + steps_k[ss], i_opt + steps_i[ss], s_n
    out.append(steps)
  return out


def classify(y_true: np.ndarray, x_ids: np.ndarray) -> Tuple[List[np.ndarray], List[np.ndarray], np.ndarray]:
  """Per window: class int8 [pl] of every base of the left-shifted sequence x (0 match, 1 mismatch, -1 never on the
  path), the original position of each of those bases, and deletions int64 [B]."""
  y = ol.left_shift(np.asarray(y_true).astype(np.int32))
  classes, sources = [], []
  dels = np.zeros(len(y), np.int64)
  for b, steps in enumerate(traceback_steps(y_true, x_ids)):
    xs, src = _shift_with_source(np.asarray(x_ids[b]).astype(np.int32))
    cls = np.full(len(src), -1, np.int8)
    for i, j, edge in steps:
      if edge == 1:
        cls[j - 1] = 0 if y[b, i - 1] == xs[j - 1] else 1
      elif edge in (2, 3):
        cls[j - 1] = 1
      else:
        dels[b] += 1
    classes.append(cls)
    sources.append(src)
  return classes, sources, dels


def calibration_counts(y_true: np.ndarray, x_ids: np.ndarray, quals: np.ndarray) -> Dict[str, np.ndarray]:
  """counts int64 [BINS, 2] (match, mismatch) over the windows, per-window totals int64 [B, 3] (match, mismatch,
  deletions), and deletions.  quals [B, L] is the quality of every original position; a binned value outside 0..99
  raises ValueError naming the window."""
  classes, sources, dels = classify(y_true, x_ids)
  counts = np.zeros((BINS, 2), np.int64)
  per = np.zeros((len(classes), 3), np.int64)
  for b, (cls, src) in enumerate(zip(classes, sources)):
    on = cls >= 0
    q = np.asarray(quals[b]).astype(np.int64)[src[on]]
    if q.size and (q.min() < 0 or q.max() >= BINS):
      raise ValueError("window %d: quality outside 0..%d" % (b, BINS - 1))
    np.add.at(counts, (q, cls[on].astype(np.int64)), 1)
    per[b] = ((cls == 0).sum(), (cls == 1).sum(), dels[b])
  return dict(counts=counts, per_window=per, deletions=int(dels.sum()))


def cross_check(per_window: np.ndarray, counts5: np.ndarray) -> bool:
  """Per window: match = num_correct_matches, mismatch = num_matches - num_correct_matches + num_insertions,
  deletions = num_deletions (counts5 in EVAL_COUNT_KEYS columns)."""
  c = np.asarray(counts5).astype(np.int64)
  want = np.stack([c[:, 3], c[:, 0] - c[:, 3] + c[:, 1], c[:, 2]], -1)
  return bool(np.array_equal(per_window, want))


def window_counts(probs: np.ndarray, labels: np.ndarray, ccs_ids: np.ndarray, ccs_bq: np.ndarray,
                  pred_quals: np.ndarray = None) -> Dict[str, np.ndarray]:
  """What dcb_evaluate_calibration returns for windows: counts int64 [2, BINS, 2], deletions int64 [2], and per-window
  totals [2, B, 3].  pred_quals (default pred_quality(probs)) are the prediction's qualities per position."""
  pq = pred_quality(probs) if pred_quals is None else pred_quals
  d = calibration_counts(labels, np.asarray(probs).argmax(-1), pq)
  c = calibration_counts(labels, ol.decode_ccs_ids(ccs_ids), ccs_bq)
  return dict(counts=np.stack([d["counts"], c["counts"]]), deletions=np.array([d["deletions"], c["deletions"]]),
              per_window=np.stack([d["per_window"], c["per_window"]]))


def classes_from_paths(paths: np.ndarray, y_true: np.ndarray, x_ids: np.ndarray) -> Tuple[List[np.ndarray], np.ndarray]:
  """The same classification read off the reference's `paths` [B, m + 1, n + 1] (the edge of the step taken from each
  cell of the optimal path): class int8 [pl] per window and deletions int64 [B]."""
  y = ol.left_shift(np.asarray(y_true).astype(np.int32))
  x = ol.left_shift(np.asarray(x_ids).astype(np.int32))
  classes = []
  dels = np.zeros(len(y), np.int64)
  for b in range(len(y)):
    pl = int((x[b] != ol.GAP).sum())
    cls = np.full(pl, -1, np.int8)
    for i, j in zip(*np.nonzero(paths[b])):
      edge = int(paths[b, i, j])
      if edge == 1:
        cls[j - 1] = 0 if y[b, i - 1] == x[b, j - 1] else 1
      elif edge in (2, 3):
        cls[j - 1] = 1
      else:
        dels[b] += 1
    classes.append(cls)
  return classes, dels
