"""ORACLE -- test infrastructure, not product code.

CPU restatement (NumPy + torch-CPU fp32) of the reference's model forward for the
hot path, written from the reference sources cited per function.  Only `tests/`,
`__graft_entry__.smoke()` and `bench.py`'s cpu-baseline / `--impl reference` legs
may import this package; the product (`deepconsensus_b200/`) never does.

PARITY STATUS -- pinned against the reference's own model code, not against TensorFlow's kernels:
the reference cannot be imported as-is in this image (tensorflow, tf-models-official, ml_collections,
pysam absent; no network), the bundled checkpoints ship without their data shard and the reference's
tests hold no numeric golden for the transformer output.  So the pin is:
  * tests/golden/ref_model_*.npz -- outputs of the UNMODIFIED reference files networks.py,
    encoder_stack.py, attention_layer.py, ffn_layer.py, data_providers.format_rows, model_configs.get_config
    and model_utils.modify_params, executed from /root/reference on a NumPy stand-in for the TF primitives
    they call (scripts/tf_shim.py, generator scripts/make_model_golden.py).  This oracle reproduces them to
    ~4e-6 on logits (tests/test_oracle_model.py::test_oracle_matches_reference_code), for ReZero and
    LayerNorm stacks, with/without the CCS-BQ row, P=20 and P=5, window 12 and 3, on real and synthetic
    windows.  That pins graph wiring, concat order, scaling, masks, residual wrappers and variable paths.
  * still restated (in tf_shim.py as here) from published behaviour: Keras 2.9 `Dense`, `EinsumDense`,
    `LayerNormalization`, `Softmax`, and tf-models-official 2.9.1 `OnDeviceEmbedding`,
    `RelativePositionEmbedding`.  A run of real TensorFlow has never been compared: to that extent parity
    is UNPINNED (float summation order inside TF's kernels; the exact timescale formula of the position
    embedding is from the published source).
  * the structural invariants of `networks_test.py` (shape, sum p = 1, zero attention outside the band)
    and the pure-function goldens of the L0/L4 helpers (tests/test_host_goldens.py).

Two arithmetic modes:
  * emulate=None   : float32 everywhere, op order of the reference (the oracle proper).
  * emulate="bf16" : identical graph, but operands of every tensor-core contraction are
                     rounded to bfloat16 at exactly the points the CUDA engine rounds
                     them; accumulation stays fp32.  The condenser, q/k/v and out-projection
                     weights are split-bf16 (hi + lo) as in the engine; LayerNorm runs in fp32
                     and its output is rounded as the next contraction's operand.
                     Used to separate kernel bugs from the documented bf16 rounding.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import numpy as np
import torch

from deepconsensus_b200 import params as params_lib
from deepconsensus_b200 import weights as weights_lib

LN_EPS = 1e-6  # encoder_stack.py:62-64,131-133


def _t(x) -> torch.Tensor:
  return torch.from_numpy(np.ascontiguousarray(np.asarray(x, dtype=np.float32)))


def _bf16(x: torch.Tensor) -> torch.Tensor:
  """Round-to-nearest-even to bfloat16, returned as float32 (== cvt.rn.bf16.f32)."""
  return x.to(torch.bfloat16).to(torch.float32)


def _hi_lo(x: torch.Tensor):
  hi = _bf16(x)
  return hi, _bf16(x - hi)


def _mm(a: torch.Tensor, b: torch.Tensor, emulate: Optional[str], split_b: bool = False) -> torch.Tensor:
  """a @ b with the engine's operand rounding: bf16 (1 product; split_b: the weights as a bf16 hi + lo pair, 2 products)
  or bf16x3 split (strict)."""
  if emulate is None:
    return a @ b
  if emulate == "bf16":
    if split_b:
      bh, bl = _hi_lo(b)
      return _bf16(a) @ bh + _bf16(a) @ bl
    return _bf16(a) @ _bf16(b)
  if emulate == "bf16x3":
    ah, al = _hi_lo(a)
    bh, bl = _hi_lo(b)
    return ah @ bh + (ah @ bl + al @ bh)
  raise ValueError(emulate)


def format_rows(rows: np.ndarray, params: params_lib.Params) -> np.ndarray:
  """Clip PW/IP to [0,*_MAX] and SN to [0,SN_MAX] (data_providers.py:128-184).

  rows: [R, L(,1)] or [B, R, L(,1)] float32 -> same without the channel axis.
  Other row groups pass through unclipped.
  """
  rows = np.array(rows, dtype=np.float32, copy=True)
  if rows.shape[-1] == 1 and rows.ndim >= 3 and rows.shape[-3] == params.total_rows:
    rows = rows[..., 0]
  (_, pw, ip, _, _, _, sn) = params_lib.get_indices(params.max_passes, params.use_ccs_bq)
  ax = rows.ndim - 2
  assert rows.shape[ax] == params.total_rows, rows.shape

  def clip(rng, hi):
    if hi:
      sl = [slice(None)] * rows.ndim
      sl[ax] = slice(*rng)
      rows[tuple(sl)] = np.clip(rows[tuple(sl)], 0, hi)

  clip(pw, params.PW_MAX)
  clip(ip, params.IP_MAX)
  clip(sn, params.SN_MAX)
  return rows


def positional_encoding(length: int, hidden: int) -> np.ndarray:
  """tf-models `RelativePositionEmbedding(hidden_size)` with min/max timescale 1 / 1e4.

  Call site networks.py:203-205,319-323.  [sin | cos] halves, float32 math.
  """
  nt = hidden // 2
  pos = np.arange(length, dtype=np.float32)
  inc = np.float32(math.log(1e4 / 1.0) / max(nt - 1, 1))
  inv = (np.float32(1.0) * np.exp(np.arange(nt, dtype=np.float32) * -inc)).astype(np.float32)
  scaled = pos[:, None] * inv[None, :]
  return np.concatenate([np.sin(scaled), np.cos(scaled)], axis=1).astype(np.float32)


def layer_norm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor) -> torch.Tensor:
  """Keras LayerNormalization(epsilon=1e-6) over the last axis, biased variance, fp32."""
  mean = x.mean(dim=-1, keepdim=True)
  var = ((x - mean) ** 2).mean(dim=-1, keepdim=True)
  return (x - mean) * torch.rsqrt(var + LN_EPS) * gamma + beta


def embed(rows_blr: torch.Tensor, params: params_lib.Params, w: weights_lib.Weights,
          emulate: Optional[str]) -> torch.Tensor:
  """Per-row embedding lookups + concat (networks.py:42-63,436-507).

  rows_blr: [B, L, R] float32 (already clipped).  id = int32 truncation; ccs_bq id is
  value+1 (networks.py:495); embeddings scaled by sqrt(width) (networks.py:54) and
  zeroed where id == 0 (networks.py:58-63).
  """
  parts = []
  for spec in params_lib.embedding_spec(params):
    vals = rows_blr[:, :, spec["row"]]
    if spec["shift"]:
      vals = vals + float(spec["shift"])
    ids = vals.to(torch.int32).to(torch.int64)          # tf.cast(float->int32) truncates
    table = _t(w[weights_lib.embedding_name(spec["table"])])
    vocab = table.shape[0]
    if int(ids.min()) < 0 or int(ids.max()) >= vocab:
      raise IndexError("embedding id out of range for table %s" % spec["table"])
    e = table[ids] * (spec["width"] ** 0.5)
    e = e * (ids != 0).to(e.dtype)[..., None]
    parts.append(e)
  out = torch.cat(parts, dim=-1)
  # bf16x3 splits the embedding into hi+lo inside _mm; plain bf16 rounds it here.
  return _bf16(out) if emulate == "bf16" else out


def band_mask(length: int, attn_win_size: Optional[int]) -> torch.Tensor:
  """tf.linalg.band_part(ones, w, w) > 0 (attention_layer.py:109-120)."""
  if not attn_win_size:
    return torch.ones(length, length, dtype=torch.bool)
  idx = torch.arange(length)
  return (idx[:, None] - idx[None, :]).abs() <= attn_win_size


def attention(y: torch.Tensor, pre: str, params: params_lib.Params, w: weights_lib.Weights,
              emulate: Optional[str], gain: float, collect: Optional[dict]) -> torch.Tensor:
  """`Attention.call` (attention_layer.py:169-221) on y [B, L, d]."""
  nh = params.num_heads
  d = params.hidden_size
  dh = d // nh
  B, L, _ = y.shape
  wq = _t(w[pre + "/query_dense_layer/kernel"]).reshape(d, d)
  wk = _t(w[pre + "/key_dense_layer/kernel"]).reshape(d, d)
  wv = _t(w[pre + "/value_dense_layer/kernel"]).reshape(d, d)
  wo = _t(w[pre + "/output_dense_layer/kernel"]).reshape(d, d)
  scale = dh ** -0.5
  y2 = y.reshape(B * L, d)
  if emulate:
    # engine folds the query scale into Wq and the ReZero gain into Wo before rounding
    q = _mm(y2, wq * scale, emulate, split_b=True)
    k = _mm(y2, wk, emulate, split_b=True)
    v = _mm(y2, wv, emulate, split_b=True)
    if emulate == "bf16":
      q, k, v = _bf16(q), _bf16(k), _bf16(v)   # stored as bf16 between kernels
      if collect is not None:
        collect.setdefault("qkv", []).append(torch.stack([q, k, v]).reshape(3, B, L, d).numpy())
  else:
    q = (y2 @ wq) * scale
    k = y2 @ wk
    v = y2 @ wv
  q = q.reshape(B, L, nh, dh).permute(0, 2, 1, 3)   # [B, N, F, H]
  k = k.reshape(B, L, nh, dh).permute(0, 2, 1, 3)   # [B, N, T, H]
  v = v.reshape(B, L, nh, dh).permute(0, 2, 1, 3)
  logits = q @ k.transpose(-1, -2)                 # [B, N, F, T]
  logits = logits + 0.0                            # attention bias is all zeros (networks.py:275-279)
  mask = band_mask(L, params.attn_win_size)
  logits = torch.where(mask, logits, torch.tensor(-1e9, dtype=logits.dtype))
  weights = torch.softmax(logits, dim=-1)
  if collect is not None:
    collect.setdefault("attention_scores", []).append(weights.numpy())
  o = weights @ v                                  # [B, N, F, H]
  o = o.permute(0, 2, 1, 3).reshape(B * L, d)
  if emulate == "bf16" and collect is not None:
    collect.setdefault("att", []).append(_bf16(o).reshape(B, L, d).numpy())
  if emulate:
    out = _mm(o, wo * gain, emulate, split_b=True)
  else:
    out = o @ wo
  return out.reshape(B, L, d)


def ffn(y: torch.Tensor, pre: str, w: weights_lib.Weights, emulate: Optional[str], gain: float,
        collect: Optional[dict] = None) -> torch.Tensor:
  """`FeedForwardNetwork.call`: relu(y W1 + b1) W2 + b2 (ffn_layer.py:83-86)."""
  B, L, d = y.shape
  w1 = _t(w[pre + "/filter_dense_layer/kernel"])
  b1 = _t(w[pre + "/filter_dense_layer/bias"])
  w2 = _t(w[pre + "/output_dense_layer/kernel"])
  b2 = _t(w[pre + "/output_dense_layer/bias"])
  y2 = y.reshape(B * L, d)
  if emulate:
    h = torch.relu(_mm(y2, w1, emulate) + b1)
    if emulate == "bf16" and collect is not None:
      collect.setdefault("hid", []).append(_bf16(h).reshape(B, L, -1).numpy())
    out = _mm(h, w2 * gain, emulate) + b2 * gain
  else:
    h = torch.relu(y2 @ w1 + b1)
    out = h @ w2 + b2
  return out.reshape(B, L, d)


def forward(rows: np.ndarray, params: params_lib.Params, w: weights_lib.Weights,
            emulate: Optional[str] = None, return_intermediates: bool = False,
            clip: bool = True) -> Dict[str, np.ndarray]:
  """rows [B,R,L(,1)] float32 -> dict(logits [B,L,5], probs [B,L,5], ...).

  `format_rows` (host clip) + `EncoderOnlyTransformer.call` (networks.py:221-239):
  squeeze/transpose (:268-273), encode (:436-520, :286-345), softmax (:238).

  return_intermediates: the residual after every stage ("embedded", "attn_n", "ffn_n"), the attention scores and,
  with emulate="bf16", the operands the engine stores as bf16 ("emb", per sub-layer "xb", per layer "qkv" [3, B, L, d],
  "att", "hid"), for the stage references of oracle/stages.py.
  """
  rows = np.asarray(rows, dtype=np.float32)
  if rows.ndim == 4:
    rows = rows[..., 0]
  if clip:
    rows = format_rows(rows, params)
  B, R, L = rows.shape
  assert R == params.total_rows, (R, params.total_rows)
  d = params.hidden_size
  inter = {} if return_intermediates else None
  with torch.no_grad():
    x = _t(rows).permute(0, 2, 1).contiguous()                      # [B, L, R]
    e = embed(x, params, w, emulate)                                # [B, L, E]
    if inter is not None and emulate == "bf16":
      inter["emb"] = e.numpy().copy()
    if params.condense_transformer_input:
      wc = _t(w["model/transformer_input_condenser/kernel"])
      h = _mm(e.reshape(B * L, -1), wc, emulate, split_b=True).reshape(B, L, d)
    else:
      h = e
    if params.add_pos_encoding:
      h = h + _t(positional_encoding(L, d))[None]
    if inter is not None:
      inter["embedded"] = h.numpy().copy()
    for n in range(params.num_hidden_layers):
      pre = "model/encoder_stack/layers/%d" % n
      for sub, fn in ((0, "attn"), (1, "ffn")):
        spre = "%s/%d" % (pre, sub)
        if params.rezero:
          y, alpha = h, float(w[spre + "/alpha"])
        else:
          y = layer_norm(h, _t(w[spre + "/layer_norm/gamma"]), _t(w[spre + "/layer_norm/beta"]))
          alpha = 1.0
        gain = alpha if emulate else 1.0     # engine folds alpha into Wo / W2 / b2
        if inter is not None and emulate == "bf16":
          inter.setdefault("xb", []).append(_bf16(y).numpy())   # the sub-layer's bf16 GEMM operand
        if fn == "attn":
          out = attention(y, spre + "/layer", params, w, emulate, gain, inter)
        else:
          out = ffn(y, spre + "/layer", w, emulate, gain, inter)
        if emulate:
          h = h + out
        else:
          h = h + alpha * out if params.rezero else h + out      # encoder_stack.py:88-92
        if inter is not None:
          inter["%s_%d" % (fn, n)] = h.numpy().copy()
    z = layer_norm(h, _t(w["model/encoder_stack/output_normalization/gamma"]),
                   _t(w["model/encoder_stack/output_normalization/beta"]))
    logits = z.reshape(B * L, d) @ _t(w["model/fc1/kernel"]) + _t(w["model/fc1/bias"])
    logits = logits.reshape(B, L, 5)
    probs = torch.softmax(logits, dim=-1)
  out = dict(logits=logits.numpy(), probs=probs.numpy(), final_output=z.numpy())
  if inter is not None:
    out["intermediates"] = inter
  return out
