"""The alignment loss as a PyTorch autograd function, on the engine's GPU kernel (dcb_alignment_loss_grad).

  loss = alignment_loss(model, probs, labels)      # per-window AlignmentLoss [B], differentiable in probs
  loss.mean().backward()

probs is a CUDA float32 [B, L, 5] tensor on the engine's device (for example the softmax of a PyTorch model's logits,
or the DCB_OUT_ON_DEVICE probabilities of a forward), labels a CUDA integer [B, L] tensor of ids 0..4 over ' ATCG'.
The forward computes the loss and the gradient in one kernel and saves the gradient; backward scales it by the
incoming per-window gradient.  soft_alignments returns AlignmentLoss.eval(return_matches=True)'s matches [B, L, L].

The engine runs on its own CUDA stream, so each call first waits for torch's current stream (the inputs are ready),
and returns once the engine's work has finished (the outputs are ready for any stream).  This is the only module of the
package that imports torch.
"""
from __future__ import annotations

from typing import Any, Optional, Tuple

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
