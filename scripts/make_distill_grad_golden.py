"""Generates tests/golden/ref_distill_grad.npz by EXECUTING the reference's own DistillationLoss.call
(deepconsensus/models/losses_and_metrics.py, unmodified, from the checkout at REF) with its tensors on torch (CPU,
float32) and tf.GradientTape on torch.autograd, as scripts/make_loss_grad_golden.py does for the alignment loss.

The ops DistillationLoss.call reaches are re-bound to torch with TensorFlow's gradients:
  tf.nn.softmax          forward as tf_shim (subtract the max, exp, sum in order, divide); backward TF's SoftmaxGrad,
                         (g - sum(g * s)) * s
  tf.math.reduce_mean    the in-order sum divided by the count (gradient g / n)
  the Keras logit losses mean_squared_error and kl_divergence, restated from keras/losses.py (Keras 2.x) as in
                         tf_shim.py; clip_by_value is torch.clamp, whose gradient passes at the bounds and is 0 outside
                         them, as TensorFlow's
The teacher's logits are constants (the distillation loop computes them outside its tape).  For every case it stores
  <case>_<mse|kl>_T<T>_loss   DistillationLoss(T, logit_loss).call(teacher, student)      float32 [B]
  <case>_<mse|kl>_T<T>_grad   d sum(loss) / d student_logits                              float32 [B, L, 5]
Cases: rand_L100 / rand_L120 of tests/golden/ref_distill.npz (inputs not repeated) at T = 0.5, 1.0, 2.5, and new
logit pairs stored as <case>_logits_teacher / _logits_student:
  edge_L1     6 windows of one position
  edge_L256   3 windows of 256 positions
  clip        4 windows, L = 100, whose softmax puts some classes below 1e-7 (student, teacher or both), so that
              kl_divergence's clip is active
What is NOT pinned: TensorFlow's and Keras's own kernels.
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
IN = os.path.join(REPO, "tests", "golden", "ref_distill.npz")
OUT = os.path.join(REPO, "tests", "golden", "ref_distill_grad.npz")

import tf_shim  # noqa: E402

IDS = {"mse": "mean_squared_error", "kl": "kl_divergence"}
TEMPERATURES = (0.5, 1.0, 2.5)
KERAS_EPSILON = 1e-7


def _fold_sum(x, axis=-1):
  x = torch.movedim(x, axis, 0)
  acc = x[0]
  for t in range(1, x.shape[0]):
    acc = acc + x[t]
  return acc


class _Softmax(torch.autograd.Function):
  @staticmethod
  def forward(ctx, x):
    e = torch.exp(x - x.amax(-1, keepdim=True))
    s = e / _fold_sum(e).unsqueeze(-1)
    ctx.save_for_backward(s)
    return s

  @staticmethod
  def backward(ctx, g):
    (s,) = ctx.saved_tensors
    return (g - _fold_sum(g * s).unsqueeze(-1)) * s


def _softmax(x, axis=-1, name=None):
  assert axis == -1
  return _Softmax.apply(x)


def _reduce_mean(x, axis=-1):
  return _fold_sum(x, axis) / x.shape[axis]


def _mean_squared_error(y_true, y_pred):
  return _reduce_mean(torch.square(y_pred - y_true), -1)


def _kl_divergence(y_true, y_pred):
  y_true = torch.clamp(y_true, KERAS_EPSILON, 1.0)
  y_pred = torch.clamp(y_pred, KERAS_EPSILON, 1.0)
  return _fold_sum(y_true * torch.log(y_true / y_pred), -1)


def import_reference():
  tf = tf_shim.install()
  tf_shim.install_losses_ops(tf)
  tf.nn.softmax = _softmax
  tf.math.reduce_mean = _reduce_mean
  sys.modules["tensorflow.compat.v2"].__dict__.update(tf.__dict__)
  sys.path.insert(0, REF)
  from deepconsensus.models import losses_and_metrics
  return losses_and_metrics


def new_cases(rng):
  out = {}
  t = (rng.normal(size=(6, 1, 5)) * 3.0).astype(np.float32)
  s = (t + rng.normal(size=t.shape) * np.array([0.05, 0.5, 2.0, 3.0, 0.0, 1.0])[:, None, None]).astype(np.float32)
  out["edge_L1"] = (t, s)
  t = (rng.normal(size=(3, 256, 5)) * 3.0).astype(np.float32)
  s = (t + rng.normal(size=t.shape) * np.array([0.1, 1.0, 3.0])[:, None, None]).astype(np.float32)
  out["edge_L256"] = (t, s)
  # classes 25..40 logits below the window's largest: probabilities of 1e-11..1e-18 at T = 1, below the clip
  t = (rng.normal(size=(4, 100, 5)) * 2.0).astype(np.float32)
  s = (t + rng.normal(size=t.shape) * 0.5).astype(np.float32)
  low = rng.random(size=t.shape) < 0.3
  s[0][low[0]] -= rng.uniform(25, 40, size=int(low[0].sum())).astype(np.float32)       # student clipped
  t[1][low[1]] -= rng.uniform(25, 40, size=int(low[1].sum())).astype(np.float32)       # teacher clipped
  s[2][low[2]] -= rng.uniform(25, 40, size=int(low[2].sum())).astype(np.float32)       # both, same classes
  t[2][low[2]] -= rng.uniform(25, 40, size=int(low[2].sum())).astype(np.float32)
  s[3] = (t[3] * 12.0).astype(np.float32)                                             # sharp student
  out["clip"] = (t.astype(np.float32), s.astype(np.float32))
  return out


def run(lm, teacher, student, T, ident):
  s = torch.from_numpy(np.array(student, np.float32)).requires_grad_(True)
  t = torch.from_numpy(np.array(teacher, np.float32))
  loss = lm.DistillationLoss(temperature=T, logit_loss=_mean_squared_error if ident == "mse" else _kl_divergence,
                             reduction="none").call(t, s)
  grad, = torch.autograd.grad(loss.sum(), s)
  return loss.detach().numpy().astype(np.float32), grad.numpy().astype(np.float32)


def main():
  torch.set_num_threads(1)
  lm = import_reference()
  gold = dict(np.load(IN))
  cases = {k: (gold[k + "_logits_teacher"], gold[k + "_logits_student"]) for k in ("rand_L100", "rand_L120")}
  added = new_cases(np.random.default_rng(1213))
  cases.update(added)
  out = {}
  for name, (t, s) in added.items():
    out[name + "_logits_teacher"], out[name + "_logits_student"] = t, s
  for name, (t, s) in cases.items():
    for short in IDS:
      for T in TEMPERATURES:
        loss, grad = run(lm, t, s, T, short)
        key = "%s_%s_T%s" % (name, short, T)
        out[key + "_loss"], out[key + "_grad"] = loss, grad
        if key in gold:   # the same loss as the NumPy stand-in's run of the reference
          np.testing.assert_allclose(loss, gold[key], rtol=1e-5, atol=2e-8)
        print(key, "loss", loss[:3], "max|grad|", float(np.abs(grad).max()))
  np.savez_compressed(OUT, **out)
  print("->", OUT)


if __name__ == "__main__":
  main()
