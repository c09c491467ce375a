"""Model variables in the reference's checkpoint layout.

Names and shapes are those of the TF object-graph checkpoint the reference
restores in `initialize_model` (quick_inference.py:515-529); the list was read
from `testdata/model/checkpoint-1.index`.  A weight set
here is a plain `dict[str, np.ndarray(float32)]` keyed by those names (without
the `/.ATTRIBUTES/VARIABLE_VALUE` suffix).

`init_weights` draws a seeded set with the reference's initialisers so tests and
benchmarks have the right scales:
  * embeddings  N(0, width^-1/2)                    networks.py:51-53
  * q/k/v/out   U(+-sqrt(6/(fan_in+fan_out)))       attention_layer.py:70-107
  * Dense       glorot_uniform kernel, zero bias    networks.py:207-213,428-434; ffn_layer.py:51-59
  * ReZero      alpha: the reference initialises 0  (encoder_stack.py:57-60), which makes
                a fresh model the identity; tests draw alpha ~ U(0.1, 1) instead.
  * LayerNorm   gamma=1, beta=0 (+ small noise when `perturb_norm`).
"""
from __future__ import annotations

import math
from typing import Dict, Iterator, Tuple

import numpy as np

from deepconsensus_b200 import params as params_lib

Weights = Dict[str, np.ndarray]

_EMB_LAYER = {
    "bases": "bases_embedding_layer",
    "pw": "pw_embedding_layer",
    "ip": "ip_embedding_layer",
    "strand": "strand_embedding_layer",
    "sn": "sn_embedding_layer",
    "ccs_bq": "ccs_base_quality_scores_embedding_layer",
}


def embedding_name(table: str) -> str:
  return "model/%s/embeddings" % _EMB_LAYER[table]


def variable_shapes(params: params_lib.Params) -> Iterator[Tuple[str, Tuple[int, ...]]]:
  """(name, shape) for every inference variable of `params`' model."""
  d = params.hidden_size
  nh = params.num_heads
  dh = d // nh
  ff = params.filter_size
  for table, (vocab, width) in params_lib.table_vocab(params).items():
    yield embedding_name(table), (vocab, width)
  if params.condense_transformer_input:
    yield "model/transformer_input_condenser/kernel", (params_lib.embedded_width(params), d)
  for n in range(params.num_hidden_layers):
    pre = "model/encoder_stack/layers/%d" % n
    for proj in ("query", "key", "value"):
      yield "%s/0/layer/%s_dense_layer/kernel" % (pre, proj), (d, nh, dh)
    yield "%s/0/layer/output_dense_layer/kernel" % pre, (nh, dh, d)
    yield "%s/1/layer/filter_dense_layer/kernel" % pre, (d, ff)
    yield "%s/1/layer/filter_dense_layer/bias" % pre, (ff,)
    yield "%s/1/layer/output_dense_layer/kernel" % pre, (ff, d)
    yield "%s/1/layer/output_dense_layer/bias" % pre, (d,)
    for sub in (0, 1):
      if params.rezero:
        yield "%s/%d/alpha" % (pre, sub), ()
      else:
        yield "%s/%d/layer_norm/gamma" % (pre, sub), (d,)
        yield "%s/%d/layer_norm/beta" % (pre, sub), (d,)
  yield "model/encoder_stack/output_normalization/gamma", (d,)
  yield "model/encoder_stack/output_normalization/beta", (d,)
  yield "model/fc1/kernel", (d, 5)
  yield "model/fc1/bias", (5,)


def count_params(params: params_lib.Params) -> int:
  return sum(int(np.prod(s)) for _, s in variable_shapes(params))


def init_weights(params: params_lib.Params, seed: int = 0, perturb_norm: bool = True,
                 weight_gain: float = 1.0) -> Weights:
  """Seeded variables with the reference's initialiser distributions."""
  rng = np.random.Generator(np.random.PCG64(seed))
  d = params.hidden_size
  out: Weights = {}

  def glorot(shape, fan_in, fan_out):
    lim = weight_gain * math.sqrt(6.0 / (fan_in + fan_out))
    return rng.uniform(-lim, lim, size=shape).astype(np.float32)

  for name, shape in variable_shapes(params):
    leaf = name.rsplit("/", 1)[-1]
    if leaf == "embeddings":
      out[name] = rng.normal(0.0, shape[1] ** -0.5, size=shape).astype(np.float32)
    elif leaf == "alpha":
      out[name] = np.float32(rng.uniform(0.1, 1.0))
    elif leaf == "gamma":
      g = np.ones(shape, np.float32)
      if perturb_norm:
        g += rng.normal(0, 0.05, size=shape).astype(np.float32)
      out[name] = g
    elif leaf == "beta":
      b = np.zeros(shape, np.float32)
      if perturb_norm:
        b += rng.normal(0, 0.05, size=shape).astype(np.float32)
      out[name] = b
    elif leaf == "bias":
      # Keras default is zeros; trained checkpoints are not, so draw small values.
      out[name] = rng.normal(0, 0.02, size=shape).astype(np.float32)
    elif "_dense_layer/kernel" in name and "/0/layer/" in name:
      out[name] = glorot(shape, d, d)            # attention_layer.py:70-77,99
    else:                                        # Dense kernels: fan_in, fan_out = shape
      out[name] = glorot(shape, shape[0], shape[-1])
  return out


def check_weights(params: params_lib.Params, weights: Weights) -> None:
  """Raises if a variable is missing or mis-shaped (what assert_existing_objects_matched guards)."""
  for name, shape in variable_shapes(params):
    if name not in weights:
      raise KeyError("missing variable %s" % name)
    got = tuple(np.shape(weights[name]))
    if got != tuple(shape):
      raise ValueError("variable %s has shape %s, expected %s" % (name, got, tuple(shape)))
