"""Generates tests/golden/ref_loss_grad.npz by EXECUTING the reference's own losses_and_metrics.py
(deepconsensus/models/losses_and_metrics.py, unmodified, from the checkout at REF) with its tensors on torch (CPU,
float32): scripts/tf_shim.py's stand-in for TensorFlow, with the ops AlignmentLoss uses re-bound to torch functions and
tf.GradientTape implemented on torch.autograd.

For every loss case of tests/golden/ref_losses.npz -- the hand tables (hand_loss_*), rand_L{100,120,200} under the
soft min (loss_reg 0.1) and the hard min (None), and the 65 real windows -- it stores
  <case>_loss      AlignmentLoss.eval(y_true, y_pred, return_matches=True)[0]    [B]
  <case>_matches   its matches: the tape gradient with respect to subs_costs       [B, m, n]
  <case>_grad      the gradient of sum(loss) with respect to y_pred                [B, n, 5]
Inputs are not repeated: they are the ones in ref_losses.npz (keys <case>_labels / _probs, del_cost / loss_reg of the
hand tables; the rand cases use del_cost 10, real del_cost 10 and loss_reg 0.1).

Why torch: its gradients have TensorFlow's semantics where AlignmentLoss depends on them -- torch.amin splits the
gradient equally among tied minima as tf.reduce_min does, clamp passes the gradient at its bounds as clip_by_value,
xlogy's gradient is 0 where x is 0, where() passes no gradient to the masked branch -- and reduce_logsumexp is restated
as TensorFlow writes it (the max is a constant).  Reductions over the 5-token axis are summed in order, as in the NumPy
shim.  What is NOT pinned: TensorFlow's own kernels.
Needs a checkout of google/deepconsensus v1.2 at REF and no GPU; the output is committed.
"""
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "scripts"))
REF = "/root/reference"
IN = os.path.join(REPO, "tests", "golden", "ref_losses.npz")
OUT = os.path.join(REPO, "tests", "golden", "ref_loss_grad.npz")

import tf_shim  # noqa: E402

_DT = {"float32": torch.float32, "float64": torch.float64, "int32": torch.int64, "int64": torch.int64,
       "bool": torch.bool}


def _dtype(d):
  if d is None or isinstance(d, torch.dtype):
    return d
  return _DT[getattr(d, "name", None) or str(d)]


def _tt(x, dtype=None):
  if isinstance(x, torch.Tensor):
    return x if dtype is None else x.to(_dtype(dtype))
  a = np.asarray(x)
  t = torch.from_numpy(a.copy()) if a.dtype.kind in "fiub" else torch.tensor(a)
  if t.dtype in (torch.int32, torch.int16, torch.uint8):
    t = t.to(torch.int64)
  return t if dtype is None else t.to(_dtype(dtype))


def _fold_sum(x, axis):
  x = torch.movedim(x, axis, 0)
  acc = x[0]
  for t in range(1, x.shape[0]):
    acc = acc + x[t]
  return acc


def _reduce_sum(x, axis=None, keepdims=False):
  x = _tt(x)
  if x.dtype in (torch.bool,):
    x = x.to(torch.int64)
  if not x.is_floating_point():
    return x.sum(dim=axis, keepdim=keepdims) if axis is not None else x.sum()
  out = _fold_sum(x.reshape(-1), 0) if axis is None else _fold_sum(x, axis % x.dim())
  if keepdims and axis is not None:
    out = out.unsqueeze(axis % x.dim())
  return out


def _reduce_logsumexp(x, axis):
  """tf.math.reduce_logsumexp: log(sum(exp(x - m))) + m, m = max (0 where not finite) under stop_gradient."""
  raw = torch.amax(x, dim=axis, keepdim=True)
  m = torch.where(torch.isfinite(raw), raw, torch.zeros_like(raw)).detach()
  return torch.log(_fold_sum(torch.exp(x - m), axis % x.dim())) + m.squeeze(axis)


class _TensorArray:
  def __init__(self, dtype, size=0, clear_after_read=True, **kw):
    self._items = {}

  def write(self, i, v):
    self._items[int(i)] = v
    return self

  def stack(self):
    return torch.stack([self._items[i] for i in sorted(self._items)])


class _GradientTape:
  """tf.GradientTape on torch.autograd: the watched tensors are already in the graph (y_pred requires grad)."""

  def __enter__(self):
    return self

  def __exit__(self, *a):
    return False

  def watch(self, x):
    if not x.requires_grad:
      raise ValueError("watched tensor is not connected to a leaf that requires grad")

  def gradient(self, target, source):
    g, = torch.autograd.grad(target.sum(), source, retain_graph=True, allow_unused=True)
    return torch.zeros_like(source) if g is None else g


def _slice(x, begin, size):
  idx = tuple(slice(int(b), None if int(s) == -1 else int(b) + int(s)) for b, s in zip(begin, size))
  return x[idx]


def _pad(x, paddings, constant_values=0):
  flat = []
  for a, b in reversed([(int(a), int(b)) for a, b in paddings]):
    flat += [a, b]
  return torch.nn.functional.pad(x, flat, value=float(constant_values))


def install_torch_losses_ops(tf):
  """Re-binds, on the stand-in module, every op AlignmentLoss.eval reaches to a torch implementation."""
  tf.float32, tf.int32 = torch.float32, torch.int32
  tf.cast = lambda x, dtype: _tt(x).to(_dtype(dtype))
  tf.shape = lambda x: torch.tensor(list(_tt(x).shape), dtype=torch.int64)
  tf.range = lambda *a, dtype=None: torch.arange(*[int(v) for v in a], dtype=torch.int64)
  tf.broadcast_to = lambda x, shape: torch.broadcast_to(_tt(x), [int(s) for s in shape])
  tf.sort = lambda x, axis=-1: torch.sort(_tt(x), dim=axis).values
  tf.where = lambda c, a, b: torch.where(_tt(c), _tt(a), _tt(b))
  tf.gather = lambda params, indices, axis=None, batch_dims=0: torch.gather(_tt(params), axis, _tt(indices))
  tf.gather_nd = lambda params, indices: params[tuple(_tt(indices).unbind(-1))]
  tf.reduce_sum = _reduce_sum
  tf.reduce_min = lambda x, axis=None: torch.amin(x, dim=axis)
  tf.reduce_logsumexp = _reduce_logsumexp
  tf.one_hot = lambda indices, depth, dtype=None: torch.nn.functional.one_hot(_tt(indices).long(), depth).to(
      _dtype(dtype) or torch.float32)
  tf.convert_to_tensor = lambda x, dtype=None, **kw: _tt(x, dtype)
  tf.clip_by_value = lambda x, lo, hi: torch.clamp(x, float(lo), float(hi))
  tf.expand_dims = lambda x, axis: _tt(x).unsqueeze(axis)
  tf.squeeze = lambda x, axis=None: _tt(x).squeeze(axis)
  tf.slice = _slice
  tf.pad = _pad
  tf.transpose = lambda x, perm=None: _tt(x).permute(*perm)
  tf.fill = lambda dims, value: torch.full([int(d) for d in dims], float(value), dtype=torch.float32)
  tf.concat = lambda xs, axis: torch.cat([_tt(x) for x in xs], dim=axis)
  tf.stack = lambda xs, axis=0: torch.stack([_tt(x) for x in xs], dim=axis)
  tf.logical_and = lambda a, b: torch.logical_and(a, b)
  tf.equal = lambda a, b: torch.eq(_tt(a), _tt(b))
  tf.TensorArray = _TensorArray
  tf.GradientTape = _GradientTape
  tf.math.log = torch.log
  tf.math.xlogy = torch.xlogy
  sys.modules["tensorflow.compat.v2"].__dict__.update(tf.__dict__)
  return tf


def import_reference():
  tf = tf_shim.install()
  tf_shim.install_losses_ops(tf)
  install_torch_losses_ops(tf)
  sys.path.insert(0, REF)
  from deepconsensus.models import losses_and_metrics
  return losses_and_metrics


def run(lm, labels, probs, del_cost, loss_reg):
  y = torch.from_numpy(np.asarray(labels, np.float32))
  p = torch.from_numpy(np.asarray(probs, np.float32).copy()).requires_grad_(True)
  loss, matches = lm.AlignmentLoss(del_cost=del_cost, loss_reg=loss_reg, width=None).eval(y, p, return_matches=True)
  grad, = torch.autograd.grad(loss.sum(), p)
  return loss.detach().numpy(), matches.detach().numpy(), grad.numpy()


def cases(gold):
  """(name, labels, probs, del_cost, loss_reg) for every loss case of ref_losses.npz."""
  i = 0
  while "hand_loss_%d_labels" % i in gold:
    k = "hand_loss_%d_" % i
    reg = float(gold[k + "loss_reg"])
    yield ("hand_loss_%d" % i, gold[k + "labels"], gold[k + "probs"], float(gold[k + "del_cost"]),
           None if np.isnan(reg) else reg)
    i += 1
  for L in (100, 120, 200):
    k = "rand_L%d" % L
    yield k + "_reg01", gold[k + "_labels"], gold[k + "_probs"], 10.0, 0.1
    yield k + "_hard", gold[k + "_labels"], gold[k + "_probs"], 10.0, None
  yield "real", gold["real_labels"], gold["real_probs"], 10.0, 0.1


def main():
  torch.set_num_threads(1)
  lm = import_reference()
  gold = dict(np.load(IN))
  out = {}
  for name, lab, probs, dc, reg in cases(gold):
    loss, matches, grad = run(lm, lab, probs, dc, reg)
    out[name + "_loss"], out[name + "_matches"], out[name + "_grad"] = loss, matches, grad
    print(name, "loss", loss[:4], "sum|grad|", float(np.abs(grad).sum()))
  np.savez_compressed(OUT, **out)
  print("->", OUT)


if __name__ == "__main__":
  main()
