"""The tf32x3 path's arithmetic on the CPU: the strict forward of the engine (csrc/strict_kernels.cu, in its launch
order and epilogue order) with every GEMM's operands split as csrc/tf32x3_kernels.cu splits them.

Each float32 operand x of a GEMM becomes big = tf32(x) and small = tf32(x - big), both rounded as cvt.rna.tf32.f32
(to 10 mantissa bits, ties away from zero), and the product is small.big + big.small + big.big.  The three products
are formed here exactly (float64) and rounded to float32 once; the device accumulates them in float32 on the tensor
cores, which is what separates the two.  Embedding, LayerNorm, attention and head are the oracle's float32.
"""
from __future__ import annotations

from typing import Dict

import numpy as np
import torch

from deepconsensus_b200 import params as params_lib
from deepconsensus_b200 import weights as weights_lib
from oracle import model as omodel


def tf32_rna(x: np.ndarray) -> np.ndarray:
  """cvt.rna.tf32.f32 on finite float32 values, returned as float32."""
  u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
  finite = (u & np.uint32(0x7F800000)) != np.uint32(0x7F800000)
  u = np.where(finite, u + np.uint32(0x1000), u) & np.uint32(0xFFFFE000)
  return u.astype(np.uint32).view(np.float32)


def split(x: np.ndarray):
  big = tf32_rna(x)
  return big, tf32_rna(np.asarray(x, np.float32) - big)


def mm3(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
  """a @ b as the tf32x3 GEMM forms it: small.big + big.small + big.big of the split operands."""
  ab, asml = (torch.from_numpy(t).double() for t in split(a.numpy()))
  bb, bsml = (torch.from_numpy(t).double() for t in split(b.numpy()))
  return (asml @ bb + ab @ bsml + ab @ bb).float()


def forward(rows: np.ndarray, params: params_lib.Params, w: weights_lib.Weights) -> Dict[str, np.ndarray]:
  """rows [B, R, L(,1)] float32 -> dict(logits [B, L, 5], probs [B, L, 5])."""
  rows = np.asarray(rows, dtype=np.float32)
  if rows.ndim == 4:
    rows = rows[..., 0]
  rows = omodel.format_rows(rows, params)
  B, _, L = rows.shape
  d, nh = params.hidden_size, params.num_heads
  dh = d // nh
  t = omodel._t
  with torch.no_grad():
    e = omodel.embed(t(rows).permute(0, 2, 1).contiguous(), params, w, None).reshape(B * L, -1)
    x = mm3(e, t(w["model/transformer_input_condenser/kernel"]))
    if params.add_pos_encoding:
      x = x + t(omodel.positional_encoding(L, d)).repeat(B, 1)
    mask = omodel.band_mask(L, params.attn_win_size)
    for n in range(params.num_hidden_layers):
      pre = "model/encoder_stack/layers/%d" % n
      for sub in (0, 1):
        spre = "%s/%d" % (pre, sub)
        if params.rezero:
          y, alpha = x, float(w[spre + "/alpha"])
        else:
          y, alpha = omodel.layer_norm(x, t(w[spre + "/layer_norm/gamma"]), t(w[spre + "/layer_norm/beta"])), 1.0
        lw = lambda name: t(w["%s/layer/%s" % (spre, name)])
        if sub == 0:
          q = mm3(y, lw("query_dense_layer/kernel").reshape(d, d)) * (dh ** -0.5)
          k = mm3(y, lw("key_dense_layer/kernel").reshape(d, d))
          v = mm3(y, lw("value_dense_layer/kernel").reshape(d, d))
          q, k, v = (z.reshape(B, L, nh, dh).permute(0, 2, 1, 3) for z in (q, k, v))
          logits = torch.where(mask, q @ k.transpose(-1, -2), torch.tensor(-1e9))
          o = (torch.softmax(logits, dim=-1) @ v).permute(0, 2, 1, 3).reshape(B * L, d)
          x = mm3(o, lw("output_dense_layer/kernel").reshape(d, d)) * alpha + x
        else:
          h = torch.relu(mm3(y, lw("filter_dense_layer/kernel")) + lw("filter_dense_layer/bias"))
          x = (mm3(h, lw("output_dense_layer/kernel")) + lw("output_dense_layer/bias")) * alpha + x
    z = omodel.layer_norm(x, t(w["model/encoder_stack/output_normalization/gamma"]),
                          t(w["model/encoder_stack/output_normalization/beta"]))
    logits = (z @ t(w["model/fc1/kernel"]) + t(w["model/fc1/bias"])).reshape(B, L, 5)
    probs = torch.softmax(logits, dim=-1)
  return dict(logits=logits.numpy(), probs=probs.numpy())
