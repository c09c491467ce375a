"""NumPy restatement of the reference's evaluation losses and metrics (test infrastructure only), pinned against vectors
produced by running the reference's own `losses_and_metrics.py` (scripts/make_loss_golden.py,
tests/golden/ref_losses.npz):

  left_shift              losses_and_metrics.left_shift_sequence (:92-115)
  alignment_loss          AlignmentLoss.eval with width=None (:306-411,549-595): float32, the same op order
                          (normalise, clip, xentropy costs, soft-min = -reg * logsumexp(-t / reg) with the max subtracted
                          as tf.reduce_logsumexp does, or the hard min)
  alignment_metric        AlignmentMetric.alignment (:704-1043): affine-gap Needleman-Wunsch, first-max tie-breaking in
                          the stacking order [match, ins, del], the traceback and its edge codes 1-5
  per_example_accuracy    PerExampleAccuracy.update_state (:43-65), one flag per window
  per_batch_identity, yield_over_ccs   :1101-1166
Everything is vectorised over the batch; the dynamic programs loop over anti-diagonals as the reference does.
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np

F32 = np.float32
GAP = 0            # dc_constants.SEQ_VOCAB.find(dc_constants.GAP): ' ATCG'
INF = F32(1e9)
EPS = 1e-7
COUNT_KEYS = ("num_matches", "num_insertions", "num_deletions", "num_correct_matches", "alignment_length")


def left_shift(y: np.ndarray) -> np.ndarray:
  """Non-gap tokens first, in order, then the gaps (a stable sort on [non-gap, gap])."""
  y = np.asarray(y)
  order = np.argsort(y == GAP, axis=-1, kind="stable")
  return np.take_along_axis(y, order, axis=-1)


def _reduce_logsumexp0(x: np.ndarray) -> np.ndarray:
  """tf.reduce_logsumexp over axis 0: log(sum(exp(x - max))) + max, max replaced by 0 where it is not finite."""
  raw = x.max(0)
  m = np.where(np.isfinite(raw), raw, F32(0)).astype(F32)
  s = np.exp((x - m).astype(F32)).astype(F32)
  acc = s[0]
  for t in range(1, s.shape[0]):           # three terms, summed in order
    acc = (acc + s[t]).astype(F32)
  return (np.log(acc).astype(F32) + m).astype(F32)


def alignment_loss(probs: np.ndarray, labels: np.ndarray, del_cost: float = 10.0,
                   loss_reg: Optional[float] = 0.1) -> np.ndarray:
  """AlignmentLoss.eval(labels, probs) for width=None: float32 [B]."""
  y = left_shift(np.asarray(labels).astype(np.int32))
  B, m = y.shape
  seq_lens = (y != GAP).sum(-1).astype(np.int32)
  p = np.asarray(probs, F32)
  n = p.shape[1]
  tot = p[..., 0]
  for t in range(1, p.shape[-1]):
    tot = (tot + p[..., t]).astype(F32)
  p = (p / tot[..., None]).astype(F32)
  lp = (-np.log(np.clip(p, F32(EPS), F32(1 - EPS)))).astype(F32)      # [B, n, 5]
  bidx = np.arange(B)[:, None, None]
  subs = lp[bidx, np.arange(n)[None, None, :], y[:, :, None]]          # [B, m, n]: subs[b, i, j] = lp[b, j, y[b, i]]
  ins = lp[..., GAP]                                                     # [B, n]
  dc = F32(del_cost)
  if loss_reg is None:
    minop = lambda t: t.min(0)
  else:
    reg = F32(loss_reg)
    minop = lambda t: ((-reg) * _reduce_logsumexp0((-t / reg).astype(F32))).astype(F32)

  def wf(k, i):                                    # subs[b, i, k - i] (0 outside), i: array of rows
    j = k - i
    ok = (j >= 0) & (j < n)
    return np.where(ok[None, :], subs[:, i, np.clip(j, 0, n - 1)], F32(0)).astype(F32)

  def wfv(k, i):                                   # ins[b, k - i] (0 outside)
    j = k - i
    ok = (j >= 0) & (j < n)
    return np.where(ok[None, :], ins[:, np.clip(j, 0, n - 1)], F32(0)).astype(F32)

  v_opt = np.full(B, INF, F32)
  v_p2 = np.full((B, m), INF, F32)
  v_p2[:, 0] = 0
  v_p1 = np.full((B, m + 1), INF, F32)
  v_p1[:, 0] = ins[:, 0]
  v_p1[:, 1] = dc
  i_range = np.arange(m + 1)
  k_end = seq_lens + n
  for k in range(2, m + n + 1):
    j_range = k - i_range
    valid = (j_range >= 0) & (j_range <= n)
    o_m = (v_p2 + wf(k - 2, np.arange(m))).astype(F32)
    o_i = (v_p1 + wfv(k - 1, i_range)).astype(F32)
    v_p2 = v_p1[:, :-1]
    o_d = (v_p2 + dc).astype(F32)
    new = np.concatenate([o_i[:, :1], minop(np.stack([o_m, o_i[:, 1:], o_d]))], axis=1)
    v_p1 = np.where(valid[None, :], new, INF).astype(F32)
    hit = k_end == k
    v_opt = np.where(hit, v_p1[np.arange(B), seq_lens], v_opt)
  return v_opt


def alignment_metric(y_true: np.ndarray, y_pred_ids: np.ndarray) -> Dict[str, np.ndarray]:
  """AlignmentMetric.alignment on label ids [B, m] and ARGMAX-DECODED prediction ids [B, n] (the reference's one-hot
  CCS input decodes to its ids).  Returns the five counts, int32 [B] each, and pid."""
  y = left_shift(np.asarray(y_true).astype(np.int32))
  x = left_shift(np.asarray(y_pred_ids).astype(np.int32))
  B, m = y.shape
  n = x.shape[1]
  tl = (y != GAP).sum(-1)
  pl = (x != GAP).sum(-1)
  NEG = -INF
  go, ge = F32(5.0 + 4.0), F32(4.0)
  gap_pens = np.array([go, go, ge], F32)[:, None, None]
  subs = np.where(y[:, :, None] == x[:, None, :], F32(2.0), F32(-5.0)).astype(F32)     # [B, m, n]

  def wf(k):                                       # [m, B]: subs[b, i, k - i]
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
  v_opt = np.zeros(B, F32)
  m_opt = np.full(B, -1, np.int32)
  i_range = np.arange(m + 1)
  k_end = tl + pl
  bidx = np.arange(B)

  def update(k, v_opt, m_opt, v_p1):
    hit = k_end == k
    col = v_p1[:, tl, bidx]                        # [3, B]
    return np.where(hit, col.max(0), v_opt), np.where(hit, col.argmax(0), m_opt).astype(np.int32)

  v_opt, m_opt = update(1, v_opt, m_opt, v_p1)
  for k in range(2, m + n + 1):
    j_range = k - i_range
    valid = ((j_range >= 0) & (j_range <= n))[None, :, None]
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
    v_opt, m_opt = update(k, v_opt, m_opt, v_p1)

  steps_k, steps_i = np.array([-2, -1, -1]), np.array([-1, 0, -1])
  trans_enc = np.array([[1, 1, 1], [2, 3, 2], [4, 4, 5]])
  counts = {k: np.zeros(B, np.int32) for k in COUNT_KEYS}
  for b in range(B):
    k_opt, i_opt, s = int(k_end[b]), int(tl[b]), int(m_opt[b])
    nm = ni = nd = nc = 0
    for k in range(m + n, -1, -1):
      if k_opt != k:
        continue
      ss = max(s, 0)
      s_n = int(dirs[k, ss, max(i_opt, 0), b])
      if s_n == -1:
        break
      edge = trans_enc[ss, max(s_n, 0)]
      j_opt = k_opt - i_opt
      if edge == 1:
        nm += 1
        if i_opt >= 1 and j_opt >= 1 and y[b, i_opt - 1] == x[b, j_opt - 1]:
          nc += 1
      elif edge in (2, 3):
        ni += 1
      else:
        nd += 1
      k_opt, i_opt, s = k_opt + steps_k[ss], i_opt + steps_i[ss], s_n
    counts["num_matches"][b], counts["num_insertions"][b], counts["num_deletions"][b] = nm, ni, nd
    counts["num_correct_matches"][b] = nc
  counts["alignment_length"] = (counts["num_matches"] + counts["num_insertions"] + counts["num_deletions"]).astype(np.int32)
  al = counts["alignment_length"]
  counts["pid"] = np.where(al > 0, counts["num_correct_matches"] / np.maximum(al, 1), 1.0).astype(F32)
  counts["v_opt"] = v_opt
  return counts


def per_example_accuracy(probs: np.ndarray, labels: np.ndarray) -> np.ndarray:
  """1 where the left-shifted argmax prediction equals the left-shifted label at all L positions (uint8 [B])."""
  y = left_shift(np.asarray(labels).astype(np.int32))
  x = left_shift(np.asarray(probs).argmax(-1).astype(np.int32))
  return (y == x).all(-1).astype(np.uint8)


def decode_ccs_ids(ccs: np.ndarray) -> np.ndarray:
  """get_batch_identity_ccs_pred's one_hot(ccs, 5) followed by AlignmentMetric's argmax: ids outside 0..4 give an
  all-zero row, whose argmax is 0, the gap."""
  ccs = np.asarray(ccs).astype(np.int32)
  return np.where((ccs >= 0) & (ccs <= 4), ccs, 0).astype(np.uint8)


def ccs_ids_from_rows(rows: np.ndarray, max_passes: int) -> np.ndarray:
  """model_utils.get_ccs_from_example + one_hot/argmax decoding: row 4P of every window (data_providers.get_indices),
  ids outside 0..4 decode to 0 (an all-zero one-hot row)."""
  return decode_ccs_ids(np.asarray(rows)[:, 4 * max_passes, :])


def evaluate_windows(probs: np.ndarray, labels: np.ndarray, ccs_ids: np.ndarray, del_cost: float = 10.0,
                     loss_reg: Optional[float] = 0.1) -> Dict[str, np.ndarray]:
  """Per-window values the engine's dcb_evaluate computes: loss, exact-match flag, counts for prediction and CCS.
  `ccs_ids` are the stored CCS ids (uint8 [B, L]); ids above 4 decode as gaps (decode_ccs_ids)."""
  pred = alignment_metric(labels, np.asarray(probs).argmax(-1))
  ccs = alignment_metric(labels, decode_ccs_ids(ccs_ids))
  return dict(loss=alignment_loss(probs, labels, del_cost, loss_reg), exact=per_example_accuracy(probs, labels),
              pred_counts=np.stack([pred[k] for k in COUNT_KEYS], -1).astype(np.int32),
              ccs_counts=np.stack([ccs[k] for k in COUNT_KEYS], -1).astype(np.int32))


def per_batch_identity(num_correct_matches: np.ndarray, alignment_length: np.ndarray) -> float:
  tot = int(np.sum(alignment_length))
  if tot == 0:
    return 1.0
  return float(np.float32(np.sum(num_correct_matches) / tot))


def yield_over_ccs(identity_pred, identity_ccs, quality_threshold: float = 0.997) -> float:
  """YieldOverCCSMetric over a sequence of batch identities: divide_no_nan(#dc >= thr, #ccs >= thr)."""
  dc = float(np.sum(np.asarray(identity_pred, np.float32) >= quality_threshold))
  cc = float(np.sum(np.asarray(identity_ccs, np.float32) >= quality_threshold))
  return dc / cc if cc else 0.0
