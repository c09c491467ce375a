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


def _copy_checked(dst: Weights, src: Weights, dst_name: str, src_name: str) -> None:
  if dst_name not in dst or src_name not in src:
    raise ValueError("cannot copy %s to %s: the %s has no such variable" %
                     (src_name, dst_name, "student" if dst_name not in dst else "teacher"))
  got, want = np.shape(src[src_name]), np.shape(dst[dst_name])
  if tuple(got) != tuple(want):
    raise ValueError("cannot copy %s %s to %s %s: shapes differ" % (src_name, tuple(got), dst_name, tuple(want)))
  dst[dst_name] = np.array(src[src_name], dtype=np.float32)


def _layer_index(i, n: int, which: str) -> int:
  if isinstance(i, bool) or not isinstance(i, (int, np.integer)) or not -n <= int(i) < n:
    raise ValueError("%s encoder layer %r out of range for %d layers" % (which, i, n))
  return int(i) % n                  # a Python list index, as the reference indexes encoder_stack.layers


def student_from_teacher(teacher_weights: Weights, teacher_params: params_lib.Params,
                         student_params: params_lib.Params, student_init: Weights) -> Weights:
  """init_student_from_teacher (model_distillation.py:104-144) on reference-named variables: the student's initial
  variables `student_init` with the teacher's copied in, as student_params (the distillation config) asks.

    init_encoder_stack      for every pair of dict(zip(teacher_encoder_layers, student_encoder_layers)), the
                            attention and FFN layers' own variables, layers/t/{0,1}/layer/* -> layers/s/{0,1}/layer/*
                            (`.layer.get_weights()`: the wrappers' alpha and layer_norm/* are not copied)
    init_nonencoder_layers  the embeddings, the input condenser and fc1 (every layer with variables whose name does not
                            contain 'encoder_stack'; encoder_stack/output_normalization is not copied)

  Raises ValueError where Keras' set_weights would (a variable missing on either side, or a shape mismatch) and for an
  encoder layer index outside either stack."""
  out = {k: np.array(v, dtype=np.float32) for k, v in student_init.items()}
  if student_params.get("init_encoder_stack"):
    nt, ns = int(teacher_params.num_hidden_layers), int(student_params.num_hidden_layers)
    pairs = dict(zip(student_params.teacher_encoder_layers, student_params.student_encoder_layers))
    for t_id, s_id in pairs.items():
      t, s = _layer_index(t_id, nt, "teacher"), _layer_index(s_id, ns, "student")
      for sub in (0, 1):
        t_pre, s_pre = ("model/encoder_stack/layers/%d/%d/layer/" % (n, sub) for n in (t, s))
        t_names = sorted(k[len(t_pre):] for k in teacher_weights if k.startswith(t_pre))
        s_names = sorted(k[len(s_pre):] for k in out if k.startswith(s_pre))
        if t_names != s_names:
          raise ValueError("teacher layer %d/%d and student layer %d/%d hold different variables: %s vs %s" %
                           (t, sub, s, sub, t_names, s_names))
        for leaf in t_names:
          _copy_checked(out, teacher_weights, s_pre + leaf, t_pre + leaf)
  if student_params.get("init_nonencoder_layers"):
    for name in teacher_weights:
      if not name.startswith("model/encoder_stack/"):
        _copy_checked(out, teacher_weights, name, name)
  return out
