"""The alignment-loss gradient on the GPU (dcb_alignment_loss_grad through B200Model.alignment_loss_grad and the torch
op of deepconsensus_b200/torch_loss.py) against dcb_evaluate, the float64 oracle (tests/loss_grad_oracle.py) and the vectors the
reference's own AlignmentLoss produced on torch autograd (tests/golden/ref_loss_grad.npz).  -m gpu.

Tolerances:
  * loss: bitwise equal to dcb_evaluate's (the same per-cell arithmetic).
  * gradient: max |g - g64| <= GRAD_GATE * max(max |g64|, 1) per case; matches: max |m - m64| <= MATCH_GATE.  The gates
    are 8x the float32 oracle's measured deviation from float64 on the same cases (tests/test_loss_grad_host.py says
    why); the largest ratio of error to gate is printed per case.  Those cases reach L = 200; at L = 256 the float32
    oracle itself deviates further (1.1e-4 of max |g64| on test_window_length_extremes' soft-min input), so there each
    gate is at least twice the float32 oracle's own deviation on the same input.
  * repeated calls, host vs device pointers, one big batch vs its windows alone: bitwise identical.
"""
import ctypes
import os
import sys

import numpy as np
import pytest

from deepconsensus_b200 import params as params_lib, synthetic, weights as weights_lib
from oracle import losses as ol

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import loss_grad_oracle as lgo  # noqa: E402

pytestmark = pytest.mark.gpu

GRAD_GATE = 8 * 1.3e-5
MATCH_GATE = 8 * 3e-5
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")


@pytest.fixture(scope="module")
def gold():
  return dict(np.load(os.path.join(GOLD, "ref_losses.npz")))


@pytest.fixture(scope="module")
def grad_gold():
  return dict(np.load(os.path.join(GOLD, "ref_loss_grad.npz")))


def _model(max_length=100, max_batch=16):
  from deepconsensus_b200 import engine
  p = params_lib.synthetic_params(max_passes=20, max_length=max_length)
  return engine.B200Model(p, weights_lib.init_weights(p, seed=3), max_batch=max_batch)


@pytest.fixture(scope="module")
def model():
  m = _model()
  yield m
  m.close()


def _cases(gold):
  out = []
  i = 0
  while "hand_loss_%d_labels" % i in gold:
    k = "hand_loss_%d_" % i
    reg = float(gold[k + "loss_reg"])
    out.append(("hand_loss_%d" % i, gold[k + "labels"], gold[k + "probs"], float(gold[k + "del_cost"]),
                None if np.isnan(reg) else reg))
    i += 1
  for L in (100, 120, 200):
    k = "rand_L%d" % L
    out.append((k + "_reg01", gold[k + "_labels"], gold[k + "_probs"], 10.0, 0.1))
    out.append((k + "_hard", gold[k + "_labels"], gold[k + "_probs"], 10.0, None))
  out.append(("real", gold["real_labels"], gold["real_probs"], 10.0, 0.1))
  return out


def _gate_check(name, r, want, f32=None):
  """Error / gate against `want`.  With `f32` (the float32 oracle on the same input, for inputs outside the golden
  cases the gates were measured on) each gate is at least twice the float32 oracle's own deviation from `want`."""
  scale = max(float(np.abs(want["grad"]).max()), 1.0)
  g_gate, m_gate = GRAD_GATE * scale, MATCH_GATE
  if f32 is not None:
    g_gate = max(g_gate, 2 * float(np.abs(f32["grad"] - want["grad"]).max()))
    m_gate = max(m_gate, 2 * float(np.abs(f32["matches"] - want["matches"]).max()))
  eg = float(np.abs(r["grad"] - want["grad"]).max()) / g_gate
  em = float(np.abs(r["matches"] - want["matches"]).max()) / m_gate
  print("%-16s error / gate: grad %.3f matches %.3f" % (name, eg, em))
  assert eg <= 1 and em <= 1, name


def test_golden_cases(model, gold, grad_gold):
  for name, lab, probs, dc, reg in _cases(gold):
    m, n = lab.shape[1], probs.shape[1]
    if m > n:
      continue
    lab_sq = np.pad(lab, [(0, 0), (0, n - m)])          # square windows: gap padding does not change the loss
    r = model.alignment_loss_grad(probs, lab_sq, del_cost=dc, loss_reg=reg, want_matches=True)
    ev = model.evaluate_windows(probs, lab_sq, lab_sq, del_cost=dc, loss_reg=reg)
    assert r["loss"].tobytes() == ev["loss"].tobytes(), name
    assert not r["matches"][:, m:].any(), name
    r["matches"] = r["matches"][:, :m]
    np.testing.assert_allclose(r["loss"], grad_gold[name + "_loss"], rtol=2e-6, atol=1e-5, err_msg=name)
    _gate_check(name + " ref", r, dict(grad=grad_gold[name + "_grad"], matches=grad_gold[name + "_matches"]))
    _gate_check(name + " f64", r, lgo.alignment_loss_grad(probs, lab, dc, reg, np.float64))


def test_deterministic_and_device_pointer_path(model, gold):
  lab, probs = gold["real_labels"], gold["real_probs"]
  a = model.alignment_loss_grad(probs, lab, want_matches=True)
  b = model.alignment_loss_grad(probs, lab, want_matches=True)
  B, L = lab.shape
  dp, dl = model.alloc_device(probs.nbytes), model.alloc_device(lab.nbytes)
  dout = [model.alloc_device(n) for n in (B * 4, B * L * 5 * 4, B * L * L * 4)]
  try:
    model.memcpy_h2d(dp, probs)
    model.memcpy_h2d(dl, lab)
    c = model.alignment_loss_grad(dp, dl, want_matches=True, on_device=True, batch=B)
    d = model.alignment_loss_grad(dp, dl, want_matches=True, on_device=True, batch=B,
                                  out=dict(loss=dout[0], grad=dout[1], matches=dout[2]))
    assert d["loss"] is None
    d = dict(loss=np.zeros(B, np.float32), grad=np.zeros((B, L, 5), np.float32), matches=np.zeros((B, L, L), np.float32))
    for k, ptr in zip(("loss", "grad", "matches"), dout):
      model.memcpy_d2h(d[k], ptr)
  finally:
    for ptr in [dp, dl] + dout:
      model.free_device(ptr)
  for k in ("loss", "grad", "matches"):
    assert a[k].tobytes() == b[k].tobytes() == c[k].tobytes() == d[k].tobytes(), k
  only_loss = model.alignment_loss_grad(probs, lab, want_grad=False)
  assert only_loss["grad"] is None and only_loss["loss"].tobytes() == a["loss"].tobytes()


@pytest.mark.parametrize("L", [1, 256])
def test_window_length_extremes(L):
  rng = np.random.default_rng(L)
  m = _model(max_length=100, max_batch=4)
  try:
    B = 4
    lab = rng.integers(1, 5, (B, L)).astype(np.uint8)      # window 0: full label
    lab[1] = 0                                               # all gaps
    lab[2, rng.random(L) < 0.3] = 0
    z = rng.normal(size=(B, L, 5)).astype(np.float32)
    probs = (np.exp(z) / np.exp(z).sum(-1, keepdims=True)).astype(np.float32)
    for reg in (0.1, None):
      r = m.alignment_loss_grad(probs, lab, del_cost=10.0, loss_reg=reg, want_matches=True)
      ev = m.evaluate_windows(probs, lab, lab, del_cost=10.0, loss_reg=reg)
      assert r["loss"].tobytes() == ev["loss"].tobytes()
      _gate_check("L%d reg %s" % (L, reg), r, lgo.alignment_loss_grad(probs, lab, 10.0, reg, np.float64),
                  f32=lgo.alignment_loss_grad(probs, lab, 10.0, reg, np.float32))
      assert not r["matches"][1].any()
      if L == 1:
        assert r["loss"][1] == np.float32(1e9) and not r["grad"][1].any()
  finally:
    m.close()


def test_batch_zero_and_persistent_grid_reuse(model, gold):
  import torch
  r = model.alignment_loss_grad(np.zeros((0, 100, 5), np.float32), np.zeros((0, 100), np.uint8), want_matches=True)
  assert r["loss"].shape == (0,) and r["grad"].shape == (0, 100, 5)
  sms = torch.cuda.get_device_properties(model.device).multi_processor_count
  B = 4 * sms + 3                                            # more windows than resident CTAs: every CTA loops
  lab, probs = gold["real_labels"], gold["real_probs"]
  idx = np.arange(B) % lab.shape[0]
  big = model.alignment_loss_grad(probs[idx], lab[idx], want_matches=True)
  one = model.alignment_loss_grad(probs, lab, want_matches=True)
  for k in ("loss", "grad", "matches"):
    assert big[k].tobytes() == one[k][idx].tobytes(), k


def test_fresh_engine_and_after_forward(gold):
  lab, probs = gold["rand_L100_labels"], gold["rand_L100_probs"]
  fresh = _model(max_batch=4)
  try:
    a = fresh.alignment_loss_grad(probs, lab, want_matches=True)
  finally:
    fresh.close()
  used = _model(max_batch=4)
  try:
    rows = synthetic.make_rows(used.params, 4, seed=2)
    used.forward(rows, want_probs=True)
    used.evaluate_windows(probs, lab, lab)
    b = used.alignment_loss_grad(probs, lab, want_matches=True)
  finally:
    used.close()
  for k in ("loss", "grad", "matches"):
    assert a[k].tobytes() == b[k].tobytes(), k


def test_invalid_arguments(model, gold):
  from deepconsensus_b200 import engine
  lab, probs = gold["real_labels"][:2], gold["real_probs"][:2]
  bad = lab.copy()
  bad[1, 3] = 5
  with pytest.raises(engine.DcbError) as ei:
    model.alignment_loss_grad(probs, bad)
  assert ei.value.code == -1 and "label" in str(ei.value)
  with pytest.raises(engine.DcbError) as ei:
    model.alignment_loss_grad(probs, lab, band_width=2)
  assert ei.value.code == -1 and "band" in str(ei.value)
  lib, h = model._lib, model._handle
  vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
  loss = np.zeros(2, np.float32)
  call = lambda p, l, B, L, out: lib.dcb_alignment_loss_grad(h, p, l, B, L, 10.0, 0.1, -1, 0, out, None, None, None)
  assert call(vp(probs), vp(lab), -1, 100, vp(loss)) == -1
  assert call(vp(probs), vp(lab), 2, 0, vp(loss)) == -1
  assert call(vp(probs), vp(lab), 2, 257, vp(loss)) == -1
  assert call(None, vp(lab), 2, 100, vp(loss)) == -1
  assert call(vp(probs), None, 2, 100, vp(loss)) == -1
  assert call(vp(probs), vp(lab), 2, 100, None) == -1
  assert call(None, None, 0, 100, None) == 0                  # batch 0 does nothing
  assert lib.dcb_alignment_loss_grad(None, vp(probs), vp(lab), 2, 100, 10.0, 0.1, -1, 0, vp(loss), None, None,
                                     None) == -1


# ---------------------------------------------------------------------------------------------------- torch op
def test_torch_backward_scales_by_weights(model, gold):
  import torch
  from deepconsensus_b200 import torch_loss
  lab, probs = gold["real_labels"], gold["real_probs"]
  dev = torch.device("cuda", model.device)
  p = torch.tensor(probs, device=dev, requires_grad=True)
  y = torch.tensor(lab, device=dev)
  loss = torch_loss.alignment_loss(model, p, y)
  w = torch.linspace(0.5, 2.0, lab.shape[0], device=dev)
  loss.mul(w).sum().backward()
  k = model.alignment_loss_grad(probs, lab)
  assert loss.detach().cpu().numpy().tobytes() == k["loss"].tobytes()
  want = torch.tensor(k["grad"], device=dev) * w[:, None, None]
  assert torch.equal(p.grad, want)
  m = torch_loss.soft_alignments(model, p, y)
  assert not m.requires_grad
  assert m.cpu().numpy().tobytes() == model.alignment_loss_grad(probs, lab, want_matches=True)["matches"].tobytes()


def test_torch_gradient_through_softmax(model, gold):
  import torch
  from deepconsensus_b200 import torch_loss
  lab = gold["rand_L120_labels"]
  rng = np.random.default_rng(5)
  logits = rng.normal(size=(lab.shape[0], lab.shape[1], 5)).astype(np.float32) * 2
  dev = torch.device("cuda", model.device)
  z = torch.tensor(logits, device=dev, requires_grad=True)
  torch_loss.alignment_loss(model, torch.softmax(z, -1), torch.tensor(lab, device=dev)).sum().backward()
  s = torch.softmax(torch.tensor(logits, dtype=torch.float64), -1).numpy()
  g = lgo.alignment_loss_grad(s, lab, 10.0, 0.1, np.float64)["grad"]
  want = s * (g - (g * s).sum(-1, keepdims=True))           # softmax's Jacobian, by hand
  err = float(np.abs(z.grad.cpu().numpy() - want).max()) / (GRAD_GATE * max(float(np.abs(want).max()), 1.0))
  print("softmax chain error / gate: %.3f" % err)
  assert err <= 1


def test_torch_sgd_lowers_the_loss(model, gold):
  import torch
  from deepconsensus_b200 import torch_loss
  lab, probs = gold["real_labels"], gold["real_probs"]
  dev = torch.device("cuda", model.device)
  z = torch.tensor(np.log(np.maximum(probs, 1e-6)), device=dev, requires_grad=True)
  y = torch.tensor(lab, device=dev, dtype=torch.int64)
  opt = torch.optim.SGD([z], lr=0.02)
  losses = []
  for _ in range(4):
    opt.zero_grad()
    loss = torch_loss.alignment_loss(model, torch.softmax(z, -1), y).mean()
    losses.append(float(loss))
    loss.backward()
    opt.step()
  print("SGD mean loss:", losses)
  assert all(b < a for a, b in zip(losses, losses[1:])), losses


def test_torch_takes_forward_device_probs_and_rejects_bad_inputs(model, gold):
  import torch
  from deepconsensus_b200 import engine, torch_loss
  B, L = 5, model.max_length
  rows = synthetic.make_rows(model.params, B, seed=9)
  dev = torch.device("cuda", model.device)
  probs = torch.empty((B, L, 5), dtype=torch.float32, device=dev)
  bq = torch.empty((2, B, L), dtype=torch.uint8, device=dev)
  torch.cuda.synchronize(dev)
  rows = np.ascontiguousarray(rows, np.float32)
  model.forward_raw(rows.ctypes.data, B, engine.DCB_OUT_ON_DEVICE, bq[0].data_ptr(), bq[1].data_ptr(), probs.data_ptr())
  lab = gold["real_labels"][:B]
  loss = torch_loss.alignment_loss(model, probs, torch.tensor(lab, device=dev))
  host = model.forward(rows, want_probs=True)["probs"]
  assert loss.cpu().numpy().tobytes() == model.alignment_loss_grad(host, lab)["loss"].tobytes()
  y = torch.tensor(lab, device=dev)
  for p_, y_ in ((probs.cpu(), y), (probs, y.cpu()), (probs.double(), y), (probs, y.float()), (probs[:, :, :4], y),
                 (probs, y[:, :-1])):
    with pytest.raises(ValueError):
      torch_loss.alignment_loss(model, p_, y_)
