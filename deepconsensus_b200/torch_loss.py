"""The training losses as PyTorch autograd functions, on the engine's GPU kernels (dcb_alignment_loss_grad,
dcb_distill_loss_grad), and a teacher engine's logits as a CUDA tensor.

  loss = alignment_loss(model, probs, labels)      # per-window AlignmentLoss [B], differentiable in probs
  loss.mean().backward()

  t = teacher_logits(teacher, rows)                # the teacher's forward, no autograd graph
  losses = distillation_objective(student, labels, student_logits, t)   # the distillation loop's compute_loss
  losses["total_loss"].backward()

probs is a CUDA float32 [B, L, 5] tensor on the engine's device (for example the softmax of a PyTorch model's logits,
or the DCB_OUT_ON_DEVICE probabilities of a forward), labels a CUDA integer [B, L] tensor of ids 0..4 over ' ATCG'.
The forward computes the loss and the gradient in one kernel and saves the gradient; backward scales it by the
incoming per-window gradient.  soft_alignments returns AlignmentLoss.eval(return_matches=True)'s matches [B, L, L].

The engine runs on its own CUDA stream, so each call first waits for torch's current stream (the inputs are ready),
and returns once the engine's work has finished (the outputs are ready for any stream).  This is the only module of the
package that imports torch.
"""
from __future__ import annotations

from typing import Any, Dict, Optional, Tuple

import torch

_INT_DTYPES = (torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64)


def _check_inputs(model, probs: torch.Tensor, labels: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
  if not isinstance(probs, torch.Tensor) or not isinstance(labels, torch.Tensor):
    raise ValueError("probs and labels must be torch tensors")
  if probs.device.type != "cuda" or labels.device.type != "cuda":
    raise ValueError("probs and labels must be CUDA tensors (got %s and %s)" % (probs.device, labels.device))
  if probs.device.index != model.device or labels.device.index != model.device:
    raise ValueError("probs and labels must be on the engine's device cuda:%d (got %s and %s)" %
                     (model.device, probs.device, labels.device))
  if probs.dtype != torch.float32:
    raise ValueError("probs must be float32, got %s" % probs.dtype)
  if labels.dtype not in _INT_DTYPES:
    raise ValueError("labels must be an integer tensor, got %s" % labels.dtype)
  if probs.dim() != 3 or probs.shape[2] != 5 or labels.shape != probs.shape[:2]:
    raise ValueError("probs must be [B, L, 5] and labels [B, L], got %s and %s" %
                     (tuple(probs.shape), tuple(labels.shape)))
  if not 1 <= probs.shape[1] <= 256:
    raise ValueError("window length must be in 1..256, got %d" % probs.shape[1])
  lab = labels.detach()
  if lab.numel() and (int(lab.min()) < 0 or int(lab.max()) > 4):
    raise ValueError("label ids must be in 0..4")
  return probs.detach().contiguous(), lab.to(torch.uint8).contiguous()


def _run(model, probs: torch.Tensor, labels: torch.Tensor, del_cost, loss_reg, want_grad: bool, want_matches: bool):
  B, L = labels.shape
  dev = probs.device
  loss = torch.empty(B, dtype=torch.float32, device=dev)
  grad = torch.empty((B, L, 5), dtype=torch.float32, device=dev) if want_grad else None
  matches = torch.empty((B, L, L), dtype=torch.float32, device=dev) if want_matches else None
  if B:
    torch.cuda.current_stream(dev).synchronize()
    out = dict(loss=loss.data_ptr(), grad=grad.data_ptr() if want_grad else 0,
               matches=matches.data_ptr() if want_matches else 0)
    model.alignment_loss_grad(probs.data_ptr(), labels.data_ptr(), del_cost=del_cost, loss_reg=loss_reg,
                              want_grad=want_grad, want_matches=want_matches, on_device=True, batch=B, length=L,
                              out=out)
  return loss, grad, matches


class AlignmentLossFunction(torch.autograd.Function):
  """forward(model, probs, labels, del_cost, loss_reg) -> loss [B]; backward -> grad * grad_output[:, None, None]."""

  @staticmethod
  def forward(ctx, model, probs, labels, del_cost, loss_reg):
    p, lab = _check_inputs(model, probs, labels)
    loss, grad, _ = _run(model, p, lab, del_cost, loss_reg, want_grad=True, want_matches=False)
    ctx.save_for_backward(grad)
    return loss

  @staticmethod
  def backward(ctx, grad_output):
    (grad,) = ctx.saved_tensors
    return None, grad * grad_output[:, None, None], None, None, None


def alignment_loss(model, probs: torch.Tensor, labels: torch.Tensor, del_cost: Optional[float] = None,
                   loss_reg: Any = "params") -> torch.Tensor:
  """Per-window AlignmentLoss [B] of probs against labels on `model`'s GPU (a deepconsensus_b200.engine.B200Model),
  differentiable in probs.  del_cost / loss_reg default to the model's params.json (loss_reg None: the hard min)."""
  return AlignmentLossFunction.apply(model, probs, labels, del_cost, loss_reg)


def soft_alignments(model, probs: torch.Tensor, labels: torch.Tensor, del_cost: Optional[float] = None,
                    loss_reg: Any = "params") -> torch.Tensor:
  """AlignmentLoss.eval(return_matches=True)'s matches [B, L, L]: the weight with which left-shifted label position i
  aligns to prediction position j.  No autograd graph."""
  p, lab = _check_inputs(model, probs, labels)
  with torch.no_grad():
    return _run(model, p, lab, del_cost, loss_reg, want_grad=False, want_matches=True)[2]


# ---------------------------------------------------------------------------------------------------- distillation
def teacher_logits(model, rows: torch.Tensor, strict: Optional[bool] = None) -> torch.Tensor:
  """The logits [B, L, 5] of `model`'s forward (a teacher engine) on a CUDA tensor of rows: float32 [B, R, L] or
  [B, R, L, 1], or packed uint8 [B, packed_window_bytes].  dcb_forward / dcb_forward_packed read the rows and write the
  logits in device memory, max_batch windows per call; the result is a CUDA float32 tensor without an autograd graph,
  as the distillation loop computes its teacher's logits outside the tape.  strict: the precision override of
  B200Model.forward.  An input id out of range raises DcbError (DCB_ERR_INPUT_RANGE), as forward() does."""
  from deepconsensus_b200 import engine
  if not isinstance(rows, torch.Tensor):
    raise ValueError("rows must be a torch tensor")
  if rows.device.type != "cuda" or rows.device.index != model.device:
    raise ValueError("rows must be on the engine's device cuda:%d (got %s)" % (model.device, rows.device))
  L = model.max_length
  x = rows.detach()
  if x.dtype == torch.uint8:
    if x.dim() != 2 or x.shape[1] != model.packed_window_bytes:
      raise ValueError("packed rows must be uint8 [B, %d], got %s" % (model.packed_window_bytes, tuple(x.shape)))
    run = model.forward_packed_raw
  elif x.dtype == torch.float32:
    if x.dim() == 4 and x.shape[3] == 1:
      x = x[..., 0]
    if x.dim() != 3 or tuple(x.shape[1:]) != (model.total_rows, L):
      raise ValueError("rows must be float32 [B, %d, %d(, 1)], got %s" % (model.total_rows, L, tuple(rows.shape)))
    run = model.forward_raw
  else:
    raise ValueError("rows must be float32 or packed uint8, got %s" % rows.dtype)
  B, mb = x.shape[0], model.max_batch
  x = x.contiguous()
  # device rows must start 16-byte aligned: a chunk that does not is copied (before torch's stream is waited for)
  chunks = []
  for b0 in range(0, B, mb):
    c = x[b0:b0 + mb]
    chunks.append((b0, c if c.data_ptr() % 16 == 0 else c.clone()))
  logits = torch.empty((B, L, 5), dtype=torch.float32, device=x.device)
  bq = torch.empty((2, min(B, mb), L), dtype=torch.uint8, device=x.device)   # bases / qualities, not kept
  if B:
    torch.cuda.current_stream(x.device).synchronize()
    flags = engine.DCB_ROWS_ON_DEVICE | engine.DCB_OUT_ON_DEVICE | model._precision_flag(strict)
    for b0, c in chunks:
      run(c.data_ptr(), c.shape[0], flags, bq[0].data_ptr(), bq[1].data_ptr(), logits_ptr=logits[b0].data_ptr())
  return logits


def _check_logits(model, teacher: torch.Tensor, student: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
  if not isinstance(teacher, torch.Tensor) or not isinstance(student, torch.Tensor):
    raise ValueError("teacher and student logits must be torch tensors")
  for name, t in (("teacher", teacher), ("student", student)):
    if t.device.type != "cuda" or t.device.index != model.device:
      raise ValueError("%s logits must be on the engine's device cuda:%d (got %s)" % (name, model.device, t.device))
    if t.dtype != torch.float32:
      raise ValueError("%s logits must be float32, got %s" % (name, t.dtype))
  if teacher.dim() != 3 or teacher.shape[2] != 5 or student.shape != teacher.shape:
    raise ValueError("teacher and student logits must both be [B, L, 5], got %s and %s" %
                     (tuple(teacher.shape), tuple(student.shape)))
  if not 1 <= teacher.shape[1] <= 256:
    raise ValueError("window length must be in 1..256, got %d" % teacher.shape[1])
  return teacher.detach().contiguous(), student.detach().contiguous()


class DistillationLossFunction(torch.autograd.Function):
  """forward(model, teacher, student, temperature, logit_loss) -> loss [B]; backward -> grad * grad_output[:, None,
  None] for the student, None for the teacher (a constant of the reference's tape)."""

  @staticmethod
  def forward(ctx, model, teacher, student, temperature, logit_loss):
    t, s = _check_logits(model, teacher, student)
    B, L = t.shape[:2]
    loss = torch.empty(B, dtype=torch.float32, device=t.device)
    grad = torch.empty((B, L, 5), dtype=torch.float32, device=t.device)
    if B:
      torch.cuda.current_stream(t.device).synchronize()
      model.distill_loss_grad(t.data_ptr(), s.data_ptr(), temperature, logit_loss, on_device=True, batch=B, length=L,
                              out=dict(loss=loss.data_ptr(), grad=grad.data_ptr()))
    ctx.save_for_backward(grad)
    return loss

  @staticmethod
  def backward(ctx, grad_output):
    (grad,) = ctx.saved_tensors
    return None, None, grad * grad_output[:, None, None], None, None


def distillation_loss(model, teacher_logits: torch.Tensor, student_logits: torch.Tensor, temperature: Any = "params",
                      logit_loss: Any = "params") -> torch.Tensor:
  """Per-window DistillationLoss [B] between CUDA float32 logits [B, L, 5], differentiable in the student's logits.
  temperature / logit_loss default to the student's params.json (evaluate.distill_settings of model.params)."""
  from deepconsensus_b200 import evaluate
  cfg = evaluate.distill_settings(model.params)
  T = cfg["temperature"] if temperature == "params" else temperature
  ident = cfg["logit_loss_identifier"] if logit_loss == "params" else logit_loss
  return DistillationLossFunction.apply(model, teacher_logits, student_logits, float(T), ident)


def distillation_objective(model, labels: torch.Tensor, student_logits: torch.Tensor,
                           teacher_logits: torch.Tensor) -> Dict[str, torch.Tensor]:
  """The distillation loop's compute_loss (model_distillation.py:242-270) for one batch: per window
  student_alpha * AlignmentLoss(labels, softmax(student_logits)) + distill_alpha * DistillationLoss(teacher, student),
  each of total_loss / student_loss / distill_loss reduced as tf.nn.compute_average_loss does (the sum over the batch
  divided by params.batch_size, the global batch size, also for a ragged batch).  `model` is a B200Model built from the
  student's params.json, which supplies the alphas, temperature, logit loss, del_cost, loss_reg and batch_size.
  Differentiable in student_logits."""
  from deepconsensus_b200 import evaluate
  cfg = evaluate.distill_settings(model.params)
  batch_size = model.params.get("batch_size")
  if not batch_size:
    raise ValueError("the student's params need batch_size (the global batch size compute_average_loss divides by)")
  student = alignment_loss(model, torch.softmax(student_logits, -1), labels)
  distill = distillation_loss(model, teacher_logits, student_logits)
  per_example = float(cfg["student_alpha"]) * student + float(cfg["distill_alpha"]) * distill
  bs = float(batch_size)
  return {"total_loss": per_example.sum() / bs, "student_loss": student.sum() / bs, "distill_loss": distill.sum() / bs}
