"""Seeded synthetic pileup windows shaped like `pre_lib.extract_features` output.

Layout and value ranges follow the reference's feature construction
(pre_lib.py:704-744; row order data_providers.py:81-113) and the statistics of the
real fixture windows:

  * bases / ccs rows: ids 0..4 (' ATCG'), gaps where the alignment has none;
  * pw / ip rows: small integers (geometric), 0 wherever the base is a gap
    (pre_lib.py:221-226), a few out-of-range values (300) to exercise the clip;
  * strand rows: 1 or 2, constant along the window, for present subreads; 0 for absent;
  * ccs_bq row (optional): -1 at ccs gaps, else 0..93;
  * sn rows: 4 fractional values in [3.9, 13), constant along the window.

Returned as float32 [B, R, L, 1] -- the exact tensor `model.predict` receives
(quick_inference.py:363) -- before `format_rows` clipping.
"""
from __future__ import annotations

import numpy as np

from deepconsensus_b200 import params as params_lib


def make_rows(params: params_lib.Params, batch: int, seed: int = 20240921,
              full_depth: bool = False) -> np.ndarray:
  """float32 [batch, total_rows, max_length, 1] synthetic windows."""
  rng = np.random.Generator(np.random.PCG64(seed))
  P, L = params.max_passes, params.max_length
  R = params_lib.get_total_rows(P, params.use_ccs_bq)
  (bases, pw, ip, strand, ccs, bq, sn) = params_lib.get_indices(P, params.use_ccs_bq)
  rows = np.zeros((batch, R, L), dtype=np.float32)

  ccs_ids = rng.integers(1, 5, size=(batch, L))
  ccs_ids[rng.random((batch, L)) < 0.10] = 0
  n_sub = np.full(batch, P) if full_depth else rng.integers(1, P + 1, size=batch)
  present = (np.arange(P)[None, :] < n_sub[:, None])               # [B, P]

  sub = np.repeat(ccs_ids[:, None, :], P, axis=1)                   # [B, P, L]
  u = rng.random((batch, P, L))
  sub = np.where(u < 0.05, rng.integers(1, 5, size=(batch, P, L)), sub)
  sub = np.where((u >= 0.05) & (u < 0.10), 0, sub)
  # trailing pad gaps: each subread ends somewhere in the last fifth of the window
  end = rng.integers(L - L // 5, L + 1, size=(batch, P))
  sub = np.where(np.arange(L)[None, None, :] < end[:, :, None], sub, 0)
  sub = sub * present[:, :, None]
  rows[:, bases[0]:bases[1]] = sub

  def kinetics():
    k = np.minimum(255, rng.geometric(0.12, size=(batch, P, L))).astype(np.float32)
    k = np.where(rng.random((batch, P, L)) < 0.005, 300.0, k)
    return k * (sub != 0)
  rows[:, pw[0]:pw[1]] = kinetics()
  rows[:, ip[0]:ip[1]] = kinetics()

  st = rng.integers(1, 3, size=(batch, P)) * present
  rows[:, strand[0]:strand[1]] = st[:, :, None]
  rows[:, ccs[0]] = ccs_ids
  if params.use_ccs_bq:
    q = rng.integers(0, 94, size=(batch, L)).astype(np.float32)
    rows[:, bq[0]] = np.where(ccs_ids == 0, -1.0, q)
  rows[:, sn[0]:sn[1]] = rng.uniform(3.9, 13.0, size=(batch, 4, 1)).astype(np.float32)
  return rows[..., None]


def mean_drift_weights(params: params_lib.Params, weights, w2_offset: float = 0.1, b2_offset: float = 15.0,
                       wo_offset: float = 0.2):
  """A copy of `weights` whose sub-layer outputs carry a large common-mode component (a constant added to the attention
  output kernel, the FFN output kernel and the FFN output bias of every layer): the residual rows' mean runs away from
  zero while their spread stays put.  LayerNorm removes it in exact arithmetic; the engine's fp32 LayerNorm must too."""
  out = dict(weights)
  for n in range(params.num_hidden_layers):
    pre = "model/encoder_stack/layers/%d" % n
    out[pre + "/1/layer/output_dense_layer/kernel"] = weights[pre + "/1/layer/output_dense_layer/kernel"] + np.float32(w2_offset)
    out[pre + "/1/layer/output_dense_layer/bias"] = weights[pre + "/1/layer/output_dense_layer/bias"] + np.float32(b2_offset)
    out[pre + "/0/layer/output_dense_layer/kernel"] = weights[pre + "/0/layer/output_dense_layer/kernel"] + np.float32(wo_offset)
  return out
