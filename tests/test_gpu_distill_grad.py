"""The distillation gradient on the GPU (dcb_distill_loss_grad through B200Model.distill_loss_grad), the teacher's logits
as a CUDA tensor, and the torch ops of deepconsensus_b200/torch_loss.py, against dcb_distill_loss, the float64 oracle
(tests/distill_grad_oracle.py) and the reference's own DistillationLoss differentiated by torch autograd
(tests/golden/ref_distill_grad.npz).  -m gpu.

Tolerances:
  * loss: bitwise equal to dcb_distill_loss's (one code path).  Against the golden: relative 2e-6 with the absolute
    floor LOSS_ATOL = 2e-7 of tests/test_distill_grad_host.py.
  * gradient against the float64 oracle, per element: |g - g64| <= K u kappa scale, with u = 2^-24 and
      kappa = 1 + max_c |student_c / T|  (rounding x = logits / T moves exp(x - max) by up to kappa u relatively)
      scale = (a_c + sum_c' a_c' s_c') s_c / T, a_c = |dl/ds_c| (+ 2 (s_c + t_c) / (5 L) for the MSE, whose s - t
              carries the absolute error of both probabilities)
    and K = 32 roundings along the longest chain: the softmax (divide, subtract, expf at 2 ulp, four adds, divide), the
    logit loss's factor (subtract or divide, multiply, divide, multiply), five products and four adds of the dot
    product, and subtract, multiply and divide at the end, each counted twice for the error it inherits.  The largest
    ratio of error to bound is printed.  Against the golden: GOLDEN_GRAD_TOL = 4e-6 of max |grad| per case.
  * repeated calls, host vs device pointers in and out: bitwise identical.
  * teacher_logits: bitwise equal to dcb_forward's logits_out on the same rows.
"""
import ctypes
import math
import os
import sys

import numpy as np
import pytest

from deepconsensus_b200 import params as params_lib, synthetic, tfrecord, weights as weights_lib

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import distill_grad_oracle as dgo  # noqa: E402

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
EVAL = os.path.join(GOLD, "human_1m", "tf_examples", "eval", "*.tfrecord.gz")
CKPT = os.path.join(GOLD, "ckpt", "model", "checkpoint-1")
LOSSES = {"mse": "mean_squared_error", "kl": "kl_divergence"}
LOSS_ATOL = 2e-7
GOLDEN_GRAD_TOL = 4e-6
K_OPS = 32
U = 2.0 ** -24


@pytest.fixture(scope="module")
def gold():
  return dict(np.load(os.path.join(GOLD, "ref_distill.npz")))


@pytest.fixture(scope="module")
def grad_gold():
  return dict(np.load(os.path.join(GOLD, "ref_distill_grad.npz")))


def _distill_params(max_length=100, **over):
  p = params_lib.get_config("transformer_learn_values_distill+test")
  for k, v in over.items():
    p[k] = v
  params_lib.modify_params(p, max_length=max_length)
  return p


@pytest.fixture(scope="module")
def model():
  from deepconsensus_b200 import engine
  p = _distill_params(batch_size=3)
  m = engine.B200Model(p, weights_lib.init_weights(p, seed=3), max_batch=16)
  yield m
  m.close()


def _random_logits(L, B=9, seed=0):
  rng = np.random.default_rng(seed + L)
  t = (rng.normal(size=(B, L, 5)) * 3.0).astype(np.float32)
  s = (t + rng.normal(size=t.shape) * np.linspace(0.05, 3.0, B)[:, None, None]).astype(np.float32)
  s[-1] = (rng.normal(size=(L, 5)) * 3.0 - np.where(rng.random((L, 5)) < 0.3, 30.0, 0.0)).astype(np.float32)
  return t, s


def _bound_ratio(got, t, s, T, ident):
  r = dgo.distillation_loss_grad(t, s, T, ident, np.float64)
  sp, L = r["s"], s.shape[1]
  a = np.abs(r["dlds"])
  if ident == "mean_squared_error":
    a = a + 2.0 * (sp + dgo._softmax64(t, T)) / (5.0 * L)
  kappa = 1.0 + np.abs(s.astype(np.float64) / T).max(-1, keepdims=True)
  scale = (a + (a * sp).sum(-1, keepdims=True)) * sp / float(np.float32(T))
  bound = K_OPS * U * kappa * scale + 1e-38
  return float((np.abs(got.astype(np.float64) - r["grad"]) / bound).max())


def _abi_losses(model, t, s, T, lid):
  """The loss of dcb_distill_loss, of dcb_distill_loss_grad with a gradient and of dcb_distill_loss_grad with a NULL
  gradient, each called directly with host arrays."""
  vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
  lib, h, (B, L) = model._lib, model._handle, t.shape[:2]
  loss = [np.full(B, np.nan, np.float32) for _ in range(3)]
  grad = np.empty_like(t)
  assert lib.dcb_distill_loss(h, vp(t), vp(s), B, L, T, lid, 0, vp(loss[0]), None) == 0
  assert lib.dcb_distill_loss_grad(h, vp(t), vp(s), B, L, T, lid, 0, vp(loss[1]), vp(grad), None) == 0
  assert lib.dcb_distill_loss_grad(h, vp(t), vp(s), B, L, T, lid, 0, vp(loss[2]), None, None) == 0
  return loss


@pytest.mark.parametrize("L", [1, 31, 32, 33, 100, 120, 256])
def test_loss_bits_equal_dcb_distill_loss_and_gradient_within_bound(model, L):
  from deepconsensus_b200 import engine
  t, s = _random_logits(L)
  worst = 0.0
  for ident in LOSSES.values():
    for T in (0.5, 1.0, 2.5):
      r = model.distill_loss_grad(t, s, T, ident)
      plain, with_grad, null_grad = _abi_losses(model, t, s, T, engine.logit_loss_id(ident))
      assert plain.tobytes() == with_grad.tobytes() == null_grad.tobytes() == r["loss"].tobytes(), (ident, T)
      assert r["loss"].tobytes() == model.distill_loss(t, s, T, ident)["loss"].tobytes(), (ident, T)
      worst = max(worst, _bound_ratio(r["grad"], t, s, T, ident))
  print("L = %d: largest gradient error / bound %.3g" % (L, worst))
  assert worst <= 1


def test_gradient_matches_reference_code_golden(model, gold, grad_gold):
  worst = 0.0
  for name in ("rand_L100", "rand_L120", "edge_L1", "edge_L256", "clip"):
    src = gold if name.startswith("rand") else grad_gold
    t, s = src[name + "_logits_teacher"], src[name + "_logits_student"]
    for short, ident in LOSSES.items():
      for T in (0.5, 1.0, 2.5):
        key = "%s_%s_T%s" % (name, short, T)
        r = model.distill_loss_grad(t, s, T, ident)
        np.testing.assert_allclose(r["loss"], grad_gold[key + "_loss"], rtol=2e-6, atol=LOSS_ATOL, err_msg=key)
        want = grad_gold[key + "_grad"]
        err = float(np.abs(r["grad"] - want).max()) / float(np.abs(want).max())
        ratio = _bound_ratio(r["grad"], t, s, T, ident)
        worst = max(worst, err)
        assert err <= GOLDEN_GRAD_TOL and ratio <= 1, (key, err, ratio)
  print("largest deviation from the golden gradient, relative to max |grad|: %.3g" % worst)


def test_clip_and_identical_logits(model, grad_gold):
  t, s = grad_gold["clip_logits_teacher"], grad_gold["clip_logits_student"]
  for T in (0.5, 1.0, 2.5):
    got = model.distill_loss_grad(t, s, T, "kl_divergence")["grad"]
    r = dgo.distillation_loss_grad(t, s, T, "kl_divergence", np.float64)
    clipped = r["s"] < 0.5e-7
    assert clipped.sum() > 50
    # dl/ds is 0 on a clipped class: what reaches its logit is the softmax backward's -sum_c g_c s_c * s_c / T alone
    only_softmax = np.broadcast_to(-(r["dlds"] * r["s"]).sum(-1, keepdims=True) * r["s"] / T, r["s"].shape)
    np.testing.assert_allclose(got[clipped], only_softmax[clipped], rtol=1e-5, atol=1e-38)
  same = model.distill_loss_grad(t, t, 1.0, "mean_squared_error")
  assert (same["loss"] == 0).all() and (same["grad"] == 0).all()


def test_deterministic_host_and_device_pointers(model, gold):
  t, s = gold["rand_L120_logits_teacher"], gold["rand_L120_logits_student"]
  B, L = t.shape[:2]
  for ident in LOSSES.values():
    a = model.distill_loss_grad(t, s, 2.5, ident)
    b = model.distill_loss_grad(t, s, 2.5, ident)
    bufs = [model.alloc_device(n) for n in (t.nbytes, s.nbytes, B * 4, t.nbytes)]
    try:
      model.memcpy_h2d(bufs[0], t)
      model.memcpy_h2d(bufs[1], s)
      model.distill_loss_grad(bufs[0], bufs[1], 2.5, ident, on_device=True, batch=B, length=L,
                              out=dict(loss=bufs[2], grad=bufs[3]))
      loss, grad = np.empty(B, np.float32), np.empty_like(t)
      model.memcpy_d2h(loss, bufs[2])
      model.memcpy_d2h(grad, bufs[3])
      c = model.distill_loss_grad(bufs[0], bufs[1], 2.5, ident, on_device=True, batch=B, length=L)
    finally:
      for p in bufs:
        model.free_device(p)
    assert a["loss"].tobytes() == b["loss"].tobytes() == loss.tobytes() == c["loss"].tobytes(), ident
    assert a["grad"].tobytes() == b["grad"].tobytes() == grad.tobytes() == c["grad"].tobytes(), ident
    assert a["ms"] > 0
    assert model.distill_loss_grad(t, s, 2.5, ident, want_grad=False)["loss"].tobytes() == a["loss"].tobytes()


def test_invalid_arguments_and_empty_batch(model, gold):
  t = np.ascontiguousarray(gold["rand_L100_logits_teacher"])
  s = np.ascontiguousarray(gold["rand_L100_logits_student"])
  out, grad = np.zeros(t.shape[0], np.float32), np.zeros_like(t)
  vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
  lib, h = model._lib, model._handle

  def call(tp=vp(t), sp=vp(s), batch=6, L=100, T=1.0, lid=0, op=vp(out), gp=vp(grad)):
    return lib.dcb_distill_loss_grad(h, tp, sp, batch, L, T, lid, 0, op, gp, None)

  cases = dict(negative_batch=dict(batch=-1), zero_L=dict(L=0), long_L=dict(L=257), zero_T=dict(T=0.0),
               negative_T=dict(T=-1.0), nan_T=dict(T=math.nan), inf_T=dict(T=math.inf),
               T_below_float32=dict(T=1e-50), T_above_float32=dict(T=1e39), unknown_id=dict(lid=2),
               negative_id=dict(lid=-1), null_teacher=dict(tp=None), null_student=dict(sp=None),
               null_out=dict(op=None))
  for name, kw in cases.items():
    assert call(**kw) == -1, name
    assert lib.dcb_last_error(h).decode().startswith("dcb_distill_loss_grad"), name
  grad[:] = 7.0
  assert call(batch=0, tp=None, sp=None, op=None, gp=None) == 0     # batch 0: nothing to do
  assert (grad == 7.0).all()
  assert call(gp=None) == 0                                          # the gradient is optional
  assert call() == 0
  assert lib.dcb_distill_loss_grad(None, vp(t), vp(s), 6, 100, 1.0, 0, 0, vp(out), None, None) == -1


# ---------------------------------------------------------------------------------------------------- teacher logits
def _teacher(precision="bf16", max_batch=16):
  from deepconsensus_b200 import engine
  p = params_lib.synthetic_params(max_passes=20, max_length=100)
  return engine.B200Model(p, weights_lib.init_weights(p, seed=21), max_batch=max_batch, precision=precision)


@pytest.mark.parametrize("strict", [False, True])
def test_teacher_logits_equal_forward_logits(strict):
  import torch
  from deepconsensus_b200 import torch_loss
  m = _teacher(max_batch=8)
  try:
    dev = torch.device("cuda", m.device)
    B = 19                                                         # > max_batch: three chunks
    rows = np.ascontiguousarray(synthetic.make_rows(m.params, B, seed=22))
    want = m.forward(rows, want_logits=True, strict=strict)["logits"]
    for x in (rows, rows[..., 0]):
      got = torch_loss.teacher_logits(m, torch.tensor(x, device=dev), strict=strict)
      assert got.dtype == torch.float32 and got.device == dev and not got.requires_grad
      assert got.cpu().numpy().tobytes() == want.tobytes()
    packed = m.pack_rows(rows)
    got = torch_loss.teacher_logits(m, torch.tensor(packed, device=dev), strict=strict)
    assert got.cpu().numpy().tobytes() == want.tobytes()
    # an unaligned view (offset by one float) and a non-contiguous one
    big = torch.zeros(B * rows[0].size + 1, dtype=torch.float32, device=dev)
    view = big[1:].view(rows[..., 0].shape)
    view.copy_(torch.tensor(rows[..., 0], device=dev))
    assert view.data_ptr() % 16 != 0
    assert torch_loss.teacher_logits(m, view, strict=strict).cpu().numpy().tobytes() == want.tobytes()
    nc = torch.tensor(rows[..., 0], device=dev).transpose(1, 2).contiguous().transpose(1, 2)
    assert not nc.is_contiguous()
    assert torch_loss.teacher_logits(m, nc, strict=strict).cpu().numpy().tobytes() == want.tobytes()
  finally:
    m.close()


def test_teacher_logits_rejects_bad_inputs():
  import torch
  from deepconsensus_b200 import engine, torch_loss
  m = _teacher()
  try:
    dev = torch.device("cuda", m.device)
    rows = torch.tensor(synthetic.make_rows(m.params, 2, seed=3)[..., 0], device=dev)
    for bad in (rows.cpu(), rows.double(), rows[:, :-1], rows[:, :, :-1], rows.unsqueeze(-1).expand(-1, -1, -1, 2),
                rows.to(torch.int32), torch.zeros((2, 7), dtype=torch.uint8, device=dev), 5):
      with pytest.raises(ValueError):
        torch_loss.teacher_logits(m, bad)
    assert torch_loss.teacher_logits(m, rows[:0]).shape == (0, 100, 5)
    out_of_range = rows.clone()
    out_of_range[0, 0, :] = 99.0                                     # a base id outside the vocabulary
    with pytest.raises(engine.DcbError) as ei:
      torch_loss.teacher_logits(m, out_of_range)
    assert ei.value.code == -5
  finally:
    m.close()


# ---------------------------------------------------------------------------------------------------- torch ops
def test_torch_backward_scales_by_weights(model, gold):
  import torch
  from deepconsensus_b200 import torch_loss
  t, s = gold["rand_L100_logits_teacher"], gold["rand_L100_logits_student"]
  dev = torch.device("cuda", model.device)
  tt = torch.tensor(t, device=dev, requires_grad=True)
  st = torch.tensor(s, device=dev, requires_grad=True)
  loss = torch_loss.distillation_loss(model, tt, st, 2.5, "kl_divergence")
  w = torch.linspace(0.5, 2.0, t.shape[0], device=dev)
  loss.mul(w).sum().backward()
  k = model.distill_loss_grad(t, s, 2.5, "kl_divergence")
  assert loss.detach().cpu().numpy().tobytes() == k["loss"].tobytes()
  assert torch.equal(st.grad, torch.tensor(k["grad"], device=dev) * w[:, None, None])
  assert tt.grad is None                                              # the teacher is a constant
  # defaults: the student's params.json (mean squared error, T = 1)
  d = torch_loss.distillation_loss(model, tt, st)
  assert d.detach().cpu().numpy().tobytes() == model.distill_loss(t, s, 1.0, "mean_squared_error")["loss"].tobytes()
  for bad in ((tt.cpu(), st), (tt, st.double()), (tt[:, :, :4], st[:, :, :4]), (tt, st[:, :-1])):
    with pytest.raises(ValueError):
      torch_loss.distillation_loss(model, *bad)


def test_torch_gradient_through_softmax(model, gold):
  import torch
  from deepconsensus_b200 import torch_loss
  t = gold["rand_L120_logits_teacher"]
  rng = np.random.default_rng(6)
  z0 = rng.normal(size=t.shape).astype(np.float32) * 2
  dev = torch.device("cuda", model.device)
  z = torch.tensor(z0, device=dev, requires_grad=True)
  student = torch.log_softmax(z, -1)                                  # a student head: log-probabilities as logits
  torch_loss.distillation_loss(model, torch.tensor(t, device=dev), student, 1.0, "kl_divergence").sum().backward()
  ls = torch.log_softmax(torch.tensor(z0, dtype=torch.float64), -1)
  g = dgo.distillation_loss_grad(t, ls.numpy().astype(np.float32), 1.0, "kl_divergence", np.float64)["grad"]
  p = ls.exp().numpy()
  want = g - p * g.sum(-1, keepdims=True)                            # log_softmax's Jacobian, by hand
  err = float(np.abs(z.grad.cpu().numpy() - want).max()) / float(np.abs(want).max())
  print("log_softmax chain error relative to max |grad|: %.3g" % err)
  assert err <= 1e-5


def test_distillation_objective_matches_oracle_and_golden(model, gold):
  import torch
  from deepconsensus_b200 import torch_loss
  from oracle import distill as od, losses as ol
  lab, t, s = gold["rand_L100_labels"], gold["rand_L100_logits_teacher"], gold["rand_L100_logits_student"]
  dev = torch.device("cuda", model.device)
  assert model.params.batch_size == 3 == int(gold["batch_size"])
  sa, da = float(gold["student_alpha"]), float(gold["distill_alpha"])
  for b0 in (0, 3):
    z = torch.tensor(s[b0:b0 + 3], device=dev, requires_grad=True)
    y = torch.tensor(lab[b0:b0 + 3], device=dev)
    out = torch_loss.distillation_objective(model, y, z, torch.tensor(t[b0:b0 + 3], device=dev))
    assert set(out) == {"total_loss", "student_loss", "distill_loss"}
    sl = ol.alignment_loss(od.softmax_scaled(s[b0:b0 + 3], 1.0), lab[b0:b0 + 3], 10.0, 0.1)
    dl = od.distillation_loss(t[b0:b0 + 3], s[b0:b0 + 3], 1.0, "mean_squared_error")
    agg = od.distillation_aggregate(sl, dl, 3, sa, da)
    for k, ok in (("total_loss", "loss"), ("student_loss", "student_loss"), ("distill_loss", "distill_loss")):
      assert float(out[k]) == pytest.approx(agg[ok], rel=1e-5), k
    assert float(out["total_loss"]) == pytest.approx(float(gold["rand_L100_batch_total"][b0 // 3]), rel=1e-5)
    out["total_loss"].backward()
    # student_alpha * alignment-term gradient (through the softmax) + distill_alpha * distillation gradient, / batch
    p = torch.softmax(z.detach(), -1)
    ga = model.alignment_loss_grad(p.cpu().numpy(), lab[b0:b0 + 3])["grad"].astype(np.float64)
    pn = p.cpu().numpy().astype(np.float64)
    ga = pn * (ga - (ga * pn).sum(-1, keepdims=True))
    gd = model.distill_loss_grad(t[b0:b0 + 3], s[b0:b0 + 3], 1.0, "mean_squared_error")["grad"]
    want = (sa * ga + da * gd) / 3.0
    err = float(np.abs(z.grad.cpu().numpy() - want).max()) / float(np.abs(want).max())
    assert err <= 1e-5, err
  # a ragged batch is still divided by the global batch size
  z = torch.tensor(s[:2], device=dev)
  out = torch_loss.distillation_objective(model, torch.tensor(lab[:2], device=dev), z, torch.tensor(t[:2], device=dev))
  dl = od.distillation_loss(t[:2], s[:2], 1.0, "mean_squared_error")
  assert float(out["distill_loss"]) == pytest.approx(float(dl.astype(np.float64).sum() / 3), rel=1e-5)


# ---------------------------------------------------------------------------------------------------- end to end
def test_student_from_teacher_engine_and_sgd_on_the_objective():
  """A 6-layer teacher and a 5-layer student initialised from it (layers [1..5] onto [0..4], embeddings, condenser and
  fc1) build and run; then SGD on a free student-logits tensor against the teacher's logits and the eval fixture's
  labels lowers total_loss at every step."""
  import torch
  from deepconsensus_b200 import engine, torch_loss
  d = tfrecord.read_examples(EVAL)
  pt = params_lib.read_params_from_json(CKPT)
  params_lib.modify_params(pt, max_length=100)
  ps = params_lib.Params(dict(pt))
  ps.update(num_hidden_layers=5, init_encoder_stack=True, init_nonencoder_layers=True,
            teacher_encoder_layers=[1, 2, 3, 4, 5], student_encoder_layers=[0, 1, 2, 3, 4], distill_alpha=1.0e5,
            student_alpha=1.0, temperature=1.0, logit_loss_identifier="mean_squared_error")
  B = d["rows"].shape[0]
  ps.batch_size = B
  tw = weights_lib.init_weights(pt, seed=41)
  sw = weights_lib.student_from_teacher(tw, pt, ps, weights_lib.init_weights(ps, seed=42))
  teacher = engine.B200Model(pt, tw, max_batch=32)
  student = engine.B200Model(ps, sw, max_batch=32)
  try:
    dev = torch.device("cuda", teacher.device)
    rows = torch.tensor(d["rows"], device=dev)
    tl = torch_loss.teacher_logits(teacher, rows)
    sl0 = torch_loss.teacher_logits(student, rows)                   # the student engine runs its forward
    assert torch.isfinite(sl0).all() and tl.shape == sl0.shape == (B, 100, 5)
    y = torch.tensor(d["labels"], device=dev)
    z = sl0.clone().requires_grad_(True)
    opt = torch.optim.SGD([z], lr=0.2)
    losses = []
    for _ in range(4):
      opt.zero_grad()
      out = torch_loss.distillation_objective(student, y, z, tl)
      losses.append(float(out["total_loss"]))
      out["total_loss"].backward()
      opt.step()
    print("SGD total_loss:", losses)
    assert all(b < a for a, b in zip(losses, losses[1:])), losses
  finally:
    teacher.close()
    student.close()
