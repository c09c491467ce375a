"""NumPy backward of the reference's AlignmentLoss (test infrastructure only): the gradient of each window's loss with
respect to the probabilities, and the soft alignment matches of AlignmentLoss.eval(return_matches=True), as
TensorFlow's tape computes them.  The forward is oracle/losses.py's alignment_loss, cell for cell.  Pinned against
finite differences and against the reference's own loss code run on torch autograd (scripts/make_loss_grad_golden.py,
tests/golden/ref_loss_grad.npz) by tests/test_loss_grad_host.py; the yardstick of tests/test_gpu_loss_grad.py.
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np

from oracle.losses import EPS, GAP, left_shift


def _softmin3_weights(om, oi, od, reg, dt):
  """d softmin3 / d (om, oi, od) as TensorFlow differentiates the minop: softmax(-t / reg) with the max held constant,
  or for the hard min (reg None) tf.reduce_min's indicator / count over exactly tied minima."""
  if reg is None:
    mn = np.minimum(np.minimum(om, oi), od)
    ind = [(o == mn).astype(dt) for o in (om, oi, od)]
    cnt = ((ind[0] + ind[1]).astype(dt) + ind[2]).astype(dt)
    return [(x / cnt).astype(dt) for x in ind]
  xs = [(-o / reg).astype(dt) for o in (om, oi, od)]
  mx = np.maximum(np.maximum(xs[0], xs[1]), xs[2])
  mx = np.where(np.isfinite(mx), mx, dt(0)).astype(dt)
  es = [np.exp((x - mx).astype(dt)).astype(dt) for x in xs]
  s = ((es[0] + es[1]).astype(dt) + es[2]).astype(dt)
  return [(e / s).astype(dt) for e in es]


def _softmin3(om, oi, od, reg, dt):
  if reg is None:
    return np.minimum(np.minimum(om, oi), od)
  xs = [(-o / reg).astype(dt) for o in (om, oi, od)]
  mx = np.maximum(np.maximum(xs[0], xs[1]), xs[2])
  mx = np.where(np.isfinite(mx), mx, dt(0)).astype(dt)
  s = np.exp((xs[0] - mx).astype(dt)).astype(dt)
  s = (s + np.exp((xs[1] - mx).astype(dt))).astype(dt)
  s = (s + np.exp((xs[2] - mx).astype(dt))).astype(dt)
  return ((-reg) * (np.log(s).astype(dt) + mx).astype(dt)).astype(dt)


def alignment_loss_grad(probs: np.ndarray, labels: np.ndarray, del_cost: float = 10.0,
                        loss_reg: Optional[float] = 0.1, dtype=np.float32) -> Dict[str, np.ndarray]:
  """AlignmentLoss.eval(labels, probs, return_matches=True) for width=None and the gradient of each window's loss with
  respect to probs, as TensorFlow's tape computes them; the backward of alignment_loss over the full DP table.

  dtype float32 follows the engine kernel's op order (align_loss_grad_kernel): the forward of alignment_loss, the
  adjoint of a cell summed as (from the match successor + from the insertion successor) + from the deletion successor,
  the cost gradients accumulated per column in decreasing anti-diagonal order.  dtype float64 is the same algorithm in
  double precision, the yardstick for both.  Returns loss [B], grad [B, n, 5], matches [B, m, n] (d loss / d
  substitution cost), ins [B, n] (the probability that prediction position j is an insertion) and dels [B, m] (that
  label position i is deleted).  A window whose last anti-diagonal seq_len + n is below 2 keeps the recursion's initial
  loss 1e9 and has zero gradient, as in the reference."""
  dt = np.dtype(dtype).type
  y = left_shift(np.asarray(labels).astype(np.int32))
  B, m = y.shape
  seq_lens = (y != GAP).sum(-1).astype(np.int64)
  p = np.asarray(probs, dt)
  n = p.shape[1]
  tot = p[..., 0]
  for t in range(1, p.shape[-1]):
    tot = (tot + p[..., t]).astype(dt)
  q = (p / tot[..., None]).astype(dt)
  lo, hi = dt(EPS), dt(1 - EPS)
  lp = (-np.log(np.clip(q, lo, hi))).astype(dt)                  # [B, n, 5]
  dc = dt(del_cost)
  reg = None if loss_reg is None else dt(loss_reg)
  inf = dt(1e9)
  bidx = np.arange(B)[:, None]
  V = np.full((B, m + 1, n + 1), inf, dt)
  V[:, 0, 0] = 0

  def diag(k):
    i = np.arange(max(0, k - n), min(m, k) + 1)
    return i, k - i

  def candidates(i, j):                            # interior cells, i >= 1, j >= 1
    lab = y[:, i - 1]                              # [B, c]
    lp_sub = lp[bidx, j[None, :] - 1, lab]
    lp_ins = lp[:, j - 1, GAP]
    om = (V[:, i - 1, j - 1] + lp_sub).astype(dt)
    oi = (V[:, i, j - 1] + lp_ins).astype(dt)
    od = (V[:, i - 1, j] + dc).astype(dt)
    return om, oi, od, lab

  for k in range(1, m + n + 1):
    i, j = diag(k)
    for ii, jj in zip(i, j):
      if ii == 0:
        V[:, 0, jj] = (V[:, 0, jj - 1] + lp[:, jj - 1, GAP]).astype(dt)
      elif k == 1:
        V[:, 1, 0] = dc
      elif jj == 0:
        V[:, ii, 0] = _softmin3(np.full(B, inf, dt), np.full(B, inf, dt), (V[:, ii - 1, 0] + dc).astype(dt), reg, dt)
    sel = (i >= 1) & (j >= 1)
    if sel.any():
      om, oi, od, _ = candidates(i[sel], j[sel])
      V[:, i[sel], j[sel]] = _softmin3(om, oi, od, reg, dt)
  k_end = seq_lens + n
  live = k_end >= 2
  loss = np.where(live, V[np.arange(B), seq_lens, n], inf).astype(dt)

  E = np.zeros((B, m + 1, n + 1), dt)
  E[np.arange(B), seq_lens, n] = np.where(live, dt(1), dt(0))
  g = np.zeros((B, n, 5), dt)                                      # d loss / d lp
  matches = np.zeros((B, m, n), dt)
  ins = np.zeros((B, n), dt)
  dels = np.zeros((B, m), dt)
  for k in range(m + n, 0, -1):
    i, j = diag(k)
    keep = i <= seq_lens[:, None]                                  # rows past seq_len are never reached
    e = np.where(keep, E[:, i, j], dt(0)).astype(dt)
    wm = np.zeros_like(e)
    wi = np.zeros_like(e)
    wd = np.zeros_like(e)
    r0 = i == 0
    wi[:, r0] = e[:, r0]                                           # row 0: the insertion chain
    c0 = (j == 0) & (i >= 1)
    if c0.any():                                                   # column 0: deletions only
      i0 = i[c0]
      if k == 1:
        wd[:, c0] = e[:, c0]
      else:
        w = _softmin3_weights(np.full((B, len(i0)), inf, dt), np.full((B, len(i0)), inf, dt),
                              (V[:, i0 - 1, 0] + dc).astype(dt), reg, dt)
        wd[:, c0] = (e[:, c0] * w[2]).astype(dt)
    sel = (i >= 1) & (j >= 1)
    if sel.any():
      om, oi, od, lab = candidates(i[sel], j[sel])
      w = _softmin3_weights(om, oi, od, reg, dt)
      wm[:, sel] = (e[:, sel] * w[0]).astype(dt)
      wi[:, sel] = (e[:, sel] * w[1]).astype(dt)
      wd[:, sel] = (e[:, sel] * w[2]).astype(dt)
      isel, jsel = i[sel], j[sel]
      matches[:, isel - 1, jsel - 1] = wm[:, sel]
      g[bidx, jsel[None, :] - 1, lab] = (g[bidx, jsel[None, :] - 1, lab] + wm[:, sel]).astype(dt)
    jin = j >= 1
    g[:, j[jin] - 1, GAP] = (g[:, j[jin] - 1, GAP] + wi[:, jin]).astype(dt)
    ins[:, j[jin] - 1] = (ins[:, j[jin] - 1] + wi[:, jin]).astype(dt)
    iin = i >= 1
    dels[:, i[iin] - 1] = (dels[:, i[iin] - 1] + wd[:, iin]).astype(dt)
    # push to the predecessors in the kernel's summation order: match, then insertion, then deletion messages
    s = sel
    E[:, i[s] - 1, j[s] - 1] = (E[:, i[s] - 1, j[s] - 1] + wm[:, s]).astype(dt)
    E[:, i[jin], j[jin] - 1] = (E[:, i[jin], j[jin] - 1] + wi[:, jin]).astype(dt)
    E[:, i[iin] - 1, j[iin]] = (E[:, i[iin] - 1, j[iin]] + wd[:, iin]).astype(dt)

  inside = (q >= lo) & (q <= hi)
  with np.errstate(divide="ignore", invalid="ignore"):
    gq = np.where(inside, -(g / q), dt(0)).astype(dt)
  dot = (gq[..., 0] * q[..., 0]).astype(dt)
  for t in range(1, 5):
    dot = (dot + (gq[..., t] * q[..., t]).astype(dt)).astype(dt)
  grad = ((gq - dot[..., None]).astype(dt) / tot[..., None]).astype(dt)
  return dict(loss=loss, grad=grad, matches=matches, ins=ins, dels=dels)
