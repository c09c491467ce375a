"""A NumPy-backed stand-in for the slice of TensorFlow / Keras / tf-models / ml_collections that the
reference's MODEL code touches, so that `deepconsensus/models/{networks,encoder_stack,attention_layer,
ffn_layer,data_providers}.py` can be EXECUTED unmodified in this container (no TensorFlow here).

TEST INFRASTRUCTURE (used only by scripts/make_model_golden.py).  What this buys: the oracle
(oracle/model.py) is compared against the reference's own Python -- its op order, concat order, scaling,
masking, residual wiring, variable naming -- rather than against my reading of it.  What it does NOT buy:
the primitives below (Dense, EinsumDense, LayerNormalization, Softmax, tf.cast, band_part, and the two
tf-models layers OnDeviceEmbedding / RelativePositionEmbedding) are themselves restated from their
published behaviour (Keras 2.9, tf-models-official 2.9.1), in float32.
"""
import contextlib
import math
import sys
import types

import numpy as np

F32 = np.float32


class T(np.ndarray):
  """ndarray with the couple of Tensor methods the reference calls."""

  def set_shape(self, shape):
    assert tuple(self.shape) == tuple(shape), (self.shape, shape)

  def numpy(self):
    return np.asarray(self)


def _t(x):
  return np.asarray(x).view(T)


class TensorShape:
  def __init__(self, dims):
    self._dims = list(dims)

  def as_list(self):
    return list(self._dims)

  def __getitem__(self, i):
    return self._dims[i]


# --------------------------------------------------------------------------- keras base classes
def _snake_case(name):
  return "".join("_" + c.lower() if c.isupper() and i else c.lower() for i, c in enumerate(name))


class Layer:
  # attributes that hold arrays but are not variables (count_variables in make_model_golden.py skips the same)
  _NOT_VARIABLES = ("params", "attn_mask")

  def __init__(self, *args, name=None, dtype=None, **kwargs):
    self._built = False
    self.name = name or _snake_case(type(self).__name__)   # Keras' default name, without the uniquifying suffix

  def build(self, input_shape):
    self._built = True

  def __call__(self, *args, **kwargs):
    if not self._built:
      first = args[0] if args else next(iter(kwargs.values()))
      self.build(TensorShape(np.shape(first)))
      self._built = True
    return self.call(*args, **kwargs)

  def _variables(self):
    """(owner, attribute) of every variable this layer and its sublayers hold, in attribute order (layer.weights)."""
    out, seen = [], set()

    def walk(obj):
      if id(obj) in seen:
        return
      seen.add(id(obj))
      if isinstance(obj, Layer):
        for k, v in vars(obj).items():
          if k in self._NOT_VARIABLES:
            continue
          if isinstance(v, np.ndarray):
            out.append((obj, k))
          elif isinstance(v, (Layer, list, tuple)):
            walk(v)
        return
      for v in obj:   # a list of layers
        if isinstance(v, (Layer, list, tuple)):
          walk(v)

    walk(self)
    return out

  @property
  def trainable_weights(self):
    return [getattr(o, k) for o, k in self._variables()]

  def get_weights(self):
    return [np.array(getattr(o, k)) for o, k in self._variables()]

  def set_weights(self, weights):
    """keras Layer.set_weights: ValueError on a count or shape mismatch."""
    slots = self._variables()
    if len(weights) != len(slots):
      raise ValueError("layer %s expects %d weights, got %d" % (self.name, len(slots), len(weights)))
    for (o, k), w in zip(slots, weights):
      if np.shape(getattr(o, k)) != np.shape(w):
        raise ValueError("layer %s weight %s has shape %s, got %s" % (self.name, k, np.shape(getattr(o, k)),
                                                                      np.shape(w)))
    for (o, k), w in zip(slots, weights):
      setattr(o, k, np.array(w, dtype=F32))


class Model(Layer):
  def summary(self):
    pass

  def __call__(self, *args, **kwargs):
    if len(args) < 2 and "training" not in kwargs:   # keras passes the learning phase: inference
      kwargs["training"] = False
    return super().__call__(*args, **kwargs)

  @property
  def layers(self):
    """The directly tracked sublayers, in the order they were assigned (keras Model.layers)."""
    return [v for v in vars(self).values() if isinstance(v, Layer)]

  def get_layer(self, name=None, index=None):
    if index is not None:
      return self.layers[index]
    return next(layer for layer in self.layers if layer.name == name)


def _activation(a):
  if a is None:
    return lambda x: x
  if callable(a):
    return a
  if a == "relu":
    return relu
  raise NotImplementedError(a)


class Dense(Layer):
  """keras.layers.Dense: y = act(x @ kernel + bias), kernel [in, units]."""

  def __init__(self, units, activation=None, use_bias=True, kernel_initializer=None,
               bias_initializer=None, name=None, **kw):
    super().__init__(name=name)
    self.units, self.use_bias, self.activation = units, use_bias, _activation(activation)
    self.kernel = None
    self.bias = None

  def build(self, input_shape):
    self.kernel = np.zeros((input_shape.as_list()[-1], self.units), F32)
    if self.use_bias:
      self.bias = np.zeros((self.units,), F32)
    super().build(input_shape)

  def call(self, x):
    y = np.matmul(np.asarray(x, F32), self.kernel)
    if self.use_bias:
      y = y + self.bias
    return _t(self.activation(y).astype(F32))


class EinsumDense(Layer):
  """keras.layers.experimental.EinsumDense without bias: y = einsum(equation, x, kernel)."""

  def __init__(self, equation, output_shape, kernel_initializer=None, bias_axes=None, name=None, **kw):
    super().__init__(name=name)
    assert bias_axes is None
    self.equation, self.out_shape = equation, tuple(output_shape)
    self.kernel = None

  def build(self, input_shape):
    lhs, out = self.equation.split("->")
    a, k = lhs.split(",")
    sizes = dict(zip(a, input_shape.as_list()))
    # output_shape omits the batch dimension
    for letter, n in zip(out[1:], self.out_shape):
      if n is not None:
        sizes[letter] = n
    self.kernel = np.zeros([sizes[c] for c in k], F32)
    super().build(input_shape)

  def call(self, x):
    return _t(np.einsum(self.equation, np.asarray(x, F32), self.kernel).astype(F32))


class LayerNormalization(Layer):
  """keras LayerNormalization over the last axis: (x - mean) * rsqrt(var + eps) * gamma + beta."""

  def __init__(self, epsilon=1e-3, dtype=None, name=None, **kw):
    super().__init__(name=name)
    self.epsilon = epsilon
    self.gamma = self.beta = None

  def build(self, input_shape):
    n = input_shape.as_list()[-1]
    self.gamma, self.beta = np.ones((n,), F32), np.zeros((n,), F32)
    super().build(input_shape)

  def call(self, x):
    x = np.asarray(x, F32)
    mean = x.mean(-1, keepdims=True, dtype=F32)
    var = ((x - mean) ** 2).mean(-1, keepdims=True, dtype=F32)
    return _t(((x - mean) * (F32(1) / np.sqrt(var + F32(self.epsilon))) * self.gamma + self.beta).astype(F32))


def softmax(x, axis=-1, name=None):
  x = np.asarray(x, F32)
  e = np.exp(x - x.max(axis, keepdims=True))
  return _t((e / e.sum(axis, keepdims=True)).astype(F32))


class Softmax(Layer):
  def call(self, x):
    return softmax(x)


def relu(x):
  return _t(np.maximum(np.asarray(x), 0))


# --------------------------------------------------------------------------- tf-models layers [3P, restated]
class OnDeviceEmbedding(Layer):
  """official.nlp.modeling.layers.OnDeviceEmbedding: gather(embeddings, ids) * scale_factor."""

  def __init__(self, vocab_size, embedding_width, initializer=None, use_one_hot=False, scale_factor=None,
               name=None, **kw):
    super().__init__(name=name)
    self._vocab_size, self._embedding_width, self._scale_factor = vocab_size, embedding_width, scale_factor
    self.embeddings = np.zeros((vocab_size, embedding_width), F32)

  def call(self, inputs):
    ids = np.asarray(inputs).astype(np.int64)
    if ids.min() < 0 or ids.max() >= self._vocab_size:
      raise IndexError("InvalidArgumentError: embedding id out of range")   # TF CPU gather behaviour
    e = self.embeddings[ids]
    if self._scale_factor:
      e = e * F32(self._scale_factor)
    return _t(e.astype(F32))


class RelativePositionEmbedding(Layer):
  """official.nlp.modeling.layers.RelativePositionEmbedding(hidden_size, min_timescale=1, max_timescale=1e4)."""

  def __init__(self, hidden_size, min_timescale=1.0, max_timescale=1.0e4, name=None, **kw):
    super().__init__(name=name)
    self._hidden_size, self._min, self._max = hidden_size, min_timescale, max_timescale

  def call(self, inputs, length=None):
    length = np.shape(inputs)[1] if length is None else length
    position = np.arange(length, dtype=F32)
    num_timescales = self._hidden_size // 2
    log_inc = F32(math.log(float(self._max) / float(self._min)) / (float(num_timescales) - 1))
    inv = (F32(self._min) * np.exp(np.arange(num_timescales, dtype=F32) * -log_inc)).astype(F32)
    scaled = position[:, None] * inv[None, :]
    return _t(np.concatenate([np.sin(scaled), np.cos(scaled)], axis=1).astype(F32))


# --------------------------------------------------------------------------- module assembly
class ConfigDict(dict):
  def __getattr__(self, k):
    try:
      return self[k]
    except KeyError as e:
      raise AttributeError(k) from e

  def __setattr__(self, k, v):
    self[k] = v


def band_part(x, lower, upper):
  x = np.asarray(x)
  n, m = x.shape[-2:]
  i, j = np.arange(n)[:, None], np.arange(m)[None, :]
  keep = ((lower < 0) | (i - j <= lower)) & ((upper < 0) | (j - i <= upper))
  return _t(np.where(keep, x, 0).astype(x.dtype))


def cast(x, dtype):
  x = np.asarray(x)
  if dtype in ("int32", np.int32):
    return _t(np.trunc(x).astype(np.int32))     # float -> int32 truncates toward zero
  return _t(x.astype(F32))


class _Anything:
  """Permissive placeholder for names only used in type annotations (tf.data.Dataset, tf.train.Example ...)."""

  def __getattr__(self, k):
    if k.startswith("__"):
      raise AttributeError(k)
    return _Anything()

  def __call__(self, *a, **k):
    return _Anything()

  def __getitem__(self, k):
    return _Anything()

  def __mro_entries__(self, bases):
    return (object,)


class _NS(_Anything):
  """Namespace with explicit attributes and a permissive fallback for everything else."""

  def __init__(self, **kw):
    self.__dict__.update(kw)


def install():
  """Registers stub modules: tensorflow, tensorflow.compat.v2, ml_collections, official..., pysam, absl."""
  tf = types.ModuleType("tensorflow")

  def _fallback(name):
    if name.startswith("__"):
      raise AttributeError(name)
    return _Anything()
  tf.__getattr__ = _fallback
  tf.float32, tf.int32, tf.int64, tf.string = "float32", "int32", "int64", "string"
  tf.Tensor, tf.TensorShape = np.ndarray, TensorShape
  tf.cast = cast
  tf.squeeze = lambda x, axis=None: _t(np.squeeze(x, axis))
  tf.transpose = lambda x, perm=None: _t(np.transpose(x, perm))
  tf.zeros_like = lambda x: _t(np.zeros_like(np.asarray(x)))
  tf.zeros = lambda shape, dtype=None: _t(np.zeros(shape, F32))
  tf.ones = lambda shape, dtype=None: _t(np.ones(shape, F32))
  tf.reduce_sum = lambda x, axis=None: _t(np.sum(x, axis=axis))
  tf.expand_dims = lambda x, axis: _t(np.expand_dims(x, axis))
  tf.concat = lambda xs, axis: _t(np.concatenate([np.asarray(x) for x in xs], axis=axis))
  tf.einsum = lambda eq, *ops: _t(np.einsum(eq, *[np.asarray(o, F32) for o in ops]).astype(F32))
  tf.where = lambda c, a, b: _t(np.where(c, a, F32(b) if np.isscalar(b) else b).astype(F32))
  tf.not_equal = lambda a, b: np.not_equal(a, b)
  tf.reshape = lambda x, s: _t(np.reshape(x, s))
  tf.clip_by_value = lambda x, clip_value_min, clip_value_max: _t(np.clip(x, clip_value_min, clip_value_max))
  tf.convert_to_tensor = lambda x: _t(np.asarray(x))
  tf.name_scope = lambda name: contextlib.nullcontext()
  tf.function = lambda f=None, **kw: f if f is not None else (lambda g: g)
  tf.Variable = lambda initial_value=None, trainable=True, **kw: np.array(initial_value, dtype=F32)
  tf.zeros_initializer = lambda: (lambda shape, dtype=None: np.zeros(shape, F32))
  tf.random_normal_initializer = lambda mean=0.0, stddev=1.0: None
  tf.nn = _NS(softmax=softmax, relu=relu, dropout=lambda x, rate: x)
  tf.linalg = types.SimpleNamespace(band_part=band_part)
  tf.io = _NS(FixedLenFeature=lambda *a, **k: None, gfile=None)
  tf.math = _NS(log=np.log)
  keras = _NS()
  keras.Model, keras.Input = Model, None
  keras.layers = _NS(Layer=Layer, Dense=Dense, LayerNormalization=LayerNormalization,
                                       Softmax=Softmax, Flatten=None, Reshape=None, Dropout=None,
                                       experimental=_NS(EinsumDense=EinsumDense))
  keras.initializers = _NS(RandomUniform=lambda minval, maxval: None)
  keras.regularizers = _NS(l2=lambda *a: None)
  keras.applications = _NS()
  tf.keras = keras
  compat = types.ModuleType("tensorflow.compat")
  v2 = types.ModuleType("tensorflow.compat.v2")
  v2.__dict__.update(tf.__dict__)
  compat.v2 = v2
  tf.compat = compat
  sys.modules.update({"tensorflow": tf, "tensorflow.compat": compat, "tensorflow.compat.v2": v2})

  mlc = types.ModuleType("ml_collections")
  mlc.ConfigDict = ConfigDict
  mlc.FrozenConfigDict = ConfigDict
  cd_pkg = types.ModuleType("ml_collections.config_dict")
  cd_mod = types.ModuleType("ml_collections.config_dict.config_dict")
  cd_mod.ConfigDict = cd_mod.FrozenConfigDict = ConfigDict
  cd_pkg.config_dict = cd_mod
  cd_pkg.ConfigDict = cd_pkg.FrozenConfigDict = ConfigDict
  cd_pkg.placeholder = lambda field_type, required=False: None    # model_configs.get_config's unset fields
  mlc.config_dict = cd_pkg
  sys.modules.update({"ml_collections": mlc, "ml_collections.config_dict": cd_pkg,
                      "ml_collections.config_dict.config_dict": cd_mod})

  layers = types.ModuleType("official.nlp.modeling.layers")
  layers.OnDeviceEmbedding, layers.RelativePositionEmbedding = OnDeviceEmbedding, RelativePositionEmbedding
  for name in ("official", "official.nlp", "official.nlp.modeling"):
    sys.modules[name] = types.ModuleType(name)
  sys.modules["official.nlp.modeling"].layers = layers
  sys.modules["official.nlp.modeling.layers"] = layers

  pysam = types.ModuleType("pysam")
  for i, n in enumerate(["CMATCH", "CINS", "CDEL", "CREF_SKIP", "CSOFT_CLIP", "CHARD_CLIP", "CPAD", "CEQUAL",
                         "CDIFF", "CBACK"]):
    setattr(pysam, n, i)
  sys.modules["pysam"] = pysam
  return tf


# --------------------------------------------------------------------------- ops of models/losses_and_metrics.py
# Used only by scripts/make_loss_golden.py and scripts/make_distill_golden.py.  Reductions over small float axes are
# summed in order, left to right, as Eigen's inner-dimension reducer does below its packet size; reduce_logsumexp follows tf.math.reduce_logsumexp
# (max subtracted, replaced by 0 where it is not finite).
def _np_dtype(dtype):
  if dtype is None:
    return None
  name = getattr(dtype, "name", None) or str(dtype)
  return np.dtype({"float32": "float32", "float64": "float64", "int32": "int32", "int64": "int64",
                   "bool": "bool"}[name])


def _cast_any(x, dtype):
  x, dt = np.asarray(x), _np_dtype(dtype)
  if dt.kind in "iu" and x.dtype.kind == "f":
    x = np.trunc(x)
  return _t(x.astype(dt))


def _fold_sum(x, axis):
  x = np.asarray(x)
  if x.dtype.kind != "f":
    return x.sum(axis=axis)
  x = np.moveaxis(x, axis, 0)
  acc = np.zeros(x.shape[1:], x.dtype)
  for t in range(x.shape[0]):
    acc = (acc + x[t]).astype(x.dtype)
  return acc


def _reduce_sum(x, axis=None, keepdims=False):
  x = np.asarray(x)
  if axis is None:
    out = _fold_sum(x.reshape(-1), 0)
  else:
    axes = [axis] if np.isscalar(axis) else list(axis)
    out = x
    for a in sorted([a % x.ndim for a in axes], reverse=True):
      out = _fold_sum(out, a)
    if keepdims:
      for a in sorted(a % x.ndim for a in axes):
        out = np.expand_dims(out, a)
  return _t(np.asarray(out))


def _reduce_logsumexp(x, axis):
  x = np.asarray(x)
  raw = x.max(axis=axis, keepdims=True)
  m = np.where(np.isfinite(raw), raw, np.zeros_like(raw))
  s = _fold_sum(np.exp(x - m), axis % x.ndim)
  return _t((np.log(s) + np.squeeze(m, axis)).astype(x.dtype))


def _tf_slice(x, begin, size):
  x = np.asarray(x)
  idx = tuple(slice(int(b), None if int(s) == -1 else int(b) + int(s)) for b, s in zip(begin, size))
  return _t(x[idx])


def _gather(params, indices, axis=None, batch_dims=0):
  params, indices = np.asarray(params), np.asarray(indices)
  if batch_dims:
    assert params.ndim == 2 and indices.ndim == 2, "only the [B, L] batch gather of left_shift_sequence"
    return _t(np.take_along_axis(params, indices, axis=1))
  return _t(np.take(params, indices, axis=axis or 0))


def _gather_nd(params, indices):
  params, indices = np.asarray(params), np.asarray(indices)
  return _t(params[tuple(np.moveaxis(indices, -1, 0))])


def _scatter_nd(indices, updates, shape):
  out = np.zeros([int(s) for s in shape], np.asarray(updates).dtype)
  np.add.at(out, tuple(np.moveaxis(np.asarray(indices), -1, 0)), np.asarray(updates))
  return _t(out)


def _fill(dims, value):
  v = np.asarray(value)
  dt = np.int32 if v.dtype.kind in "iu" else v.dtype
  return _t(np.full([int(d) for d in np.atleast_1d(dims)], v, dt))


def _pad(x, paddings, constant_values=0):
  x = np.asarray(x)
  return _t(np.pad(x, [(int(a), int(b)) for a, b in paddings], constant_values=np.asarray(constant_values, x.dtype)))


def _one_hot(indices, depth, dtype=None):
  idx = np.asarray(indices).astype(np.int64)
  ok = (idx >= 0) & (idx < depth)
  out = (np.arange(depth) == np.where(ok, idx, -1)[..., None]).astype(_np_dtype(dtype) or np.float32)
  return _t(out)


def _xlogy(x, y):
  x, y = np.asarray(x), np.asarray(y)
  with np.errstate(divide="ignore", invalid="ignore"):
    return _t(np.where(x == 0, np.zeros_like(x * y), x * np.log(y)).astype(np.result_type(x, y)))


def _softmax_folded(x, axis=-1, name=None):
  """tf.nn.softmax: subtract the max, exp, sum (in order), divide."""
  x = np.asarray(x)
  e = np.exp(x - x.max(axis, keepdims=True))
  return _t((e / np.expand_dims(_fold_sum(e, axis % x.ndim), axis)).astype(x.dtype))


def _reduce_mean(x, axis=None):
  """tf.math.reduce_mean: the in-order sum divided by the element count, in the input's dtype."""
  x = np.asarray(x)
  n = x.size if axis is None else x.shape[axis]
  return _t((np.asarray(_reduce_sum(x, axis)) / x.dtype.type(n)).astype(x.dtype))


# The two Keras logit losses DistillationLoss is used with (Keras is not part of the reference tree; restated from the
# documented semantics of keras/losses.py, Keras 2.x): y_true is the first argument.
def _mean_squared_error(y_true, y_pred):
  y_true, y_pred = np.asarray(y_true), np.asarray(y_pred)
  return _reduce_mean(np.square(y_pred - y_true), axis=-1)


_KERAS_EPSILON = 1e-7          # keras.backend.epsilon()


def _kl_divergence(y_true, y_pred):
  y_true, y_pred = np.asarray(y_true), np.asarray(y_pred)
  dt = y_true.dtype.type
  y_true = np.clip(y_true, dt(_KERAS_EPSILON), dt(1))
  y_pred = np.clip(y_pred, dt(_KERAS_EPSILON), dt(1))
  return _reduce_sum(y_true * np.log(y_true / y_pred), axis=-1)


_KERAS_LOSSES = {"mean_squared_error": _mean_squared_error, "mse": _mean_squared_error, "MSE": _mean_squared_error,
                 "kl_divergence": _kl_divergence, "kullback_leibler_divergence": _kl_divergence,
                 "kld": _kl_divergence, "KLD": _kl_divergence}


def _keras_losses_get(identifier):
  """tf.keras.losses.get for the identifiers above (callables pass through)."""
  if callable(identifier):
    return identifier
  if identifier not in _KERAS_LOSSES:
    raise ValueError("Unknown loss function: %r" % (identifier,))
  return _KERAS_LOSSES[identifier]


class _TensorArray:
  def __init__(self, dtype, size=0, clear_after_read=True, **kw):
    self._items = {}

  def write(self, i, v):
    self._items[int(i)] = np.asarray(v)
    return self

  def read(self, i):
    return _t(self._items[int(i)])

  def stack(self):
    return _t(np.stack([self._items[i] for i in sorted(self._items)]))


class _Loss:
  def __init__(self, reduction=None, name=None):
    self.reduction = reduction

  def __call__(self, y_true, y_pred):
    return _t(np.asarray(self.call(y_true, y_pred)).mean(dtype=np.float32))


class _Weight:
  def __init__(self):
    self.value = np.float32(0)

  def assign_add(self, v):
    self.value = np.float32(self.value + np.float32(v))

  def assign(self, v):
    self.value = np.float32(v)

  def __array__(self, dtype=None, copy=None):
    return np.asarray(self.value, dtype=dtype)


class _Metric:
  def __init__(self, name=None, **kw):
    self.name = name

  def add_weight(self, name=None, shape=None, initializer=None):
    return _Weight()


class _Mean(_Metric):
  def __init__(self, name=None, **kw):
    super().__init__(name)
    self.reset_states()

  def update_state(self, values, sample_weight=None):
    v = np.asarray(values, np.float64).reshape(-1)
    self._sum += v.sum()
    self._n += v.size

  def result(self):
    return _t(np.float32(self._sum / self._n if self._n else 0.0))

  def reset_states(self):
    self._sum, self._n = 0.0, 0


class _Accuracy(_Mean):
  def update_state(self, y_true, y_pred, sample_weight=None):
    super().update_state(np.asarray(y_true) == np.asarray(y_pred))


def install_losses_ops(tf):
  """Adds what losses_and_metrics.py (and dc_constants.py) use to the stand-in installed by install()."""
  tf.bool = "bool"
  tf.newaxis = None
  tf.cast = _cast_any
  tf.shape = lambda x: np.array(np.shape(x), np.int32)
  tf.range = lambda *a, dtype=None: _t(np.arange(*[int(v) for v in a], dtype=_np_dtype(dtype) or np.int32))
  tf.broadcast_to = lambda x, shape: _t(np.broadcast_to(np.asarray(x), [int(s) for s in shape]))
  tf.sort = lambda x, axis=-1: _t(np.sort(np.asarray(x), axis=axis))
  tf.where = lambda c, a, b: _t(np.where(np.asarray(c), np.asarray(a), np.asarray(b)))
  tf.gather, tf.gather_nd, tf.scatter_nd = _gather, _gather_nd, _scatter_nd
  tf.reduce_sum = _reduce_sum
  tf.reduce_min = lambda x, axis=None: _t(np.asarray(x).min(axis=axis))
  tf.reduce_max = lambda x, axis=None: _t(np.asarray(x).max(axis=axis))
  tf.reduce_logsumexp = _reduce_logsumexp
  tf.argmax = lambda x, axis=None, output_type=None: _t(
      np.asarray(x).argmax(axis=-1 if axis is None else axis).astype(_np_dtype(output_type) or np.int64))
  tf.one_hot = _one_hot
  tf.convert_to_tensor = lambda x, dtype=None, **kw: _t(np.asarray(x, dtype=_np_dtype(dtype)))
  tf.constant = lambda x, dtype=None: _t(np.asarray(x, dtype=_np_dtype(dtype)))
  tf.clip_by_value = lambda x, lo, hi: _t(np.clip(np.asarray(x), np.asarray(lo, np.asarray(x).dtype),
                                                  np.asarray(hi, np.asarray(x).dtype)))
  tf.expand_dims = lambda x, axis: _t(np.expand_dims(np.asarray(x), axis))
  tf.squeeze = lambda x, axis=None: _t(np.squeeze(np.asarray(x), tuple(axis) if isinstance(axis, list) else axis))
  tf.slice = _tf_slice
  tf.pad = _pad
  tf.transpose = lambda x, perm=None: _t(np.transpose(np.asarray(x), perm))
  tf.fill = _fill
  tf.concat = lambda xs, axis: _t(np.concatenate([np.asarray(x) for x in xs], axis=axis))
  tf.stack = lambda xs, axis=0: _t(np.stack([np.asarray(x) for x in xs], axis=axis))
  tf.roll = lambda x, shift, axis: _t(np.roll(np.asarray(x), shift, axis))
  tf.reshape = lambda x, s: _t(np.reshape(np.asarray(x), [int(v) for v in s]))
  tf.maximum = lambda a, b: _t(np.maximum(a, b))
  tf.logical_and = lambda a, b: _t(np.logical_and(a, b))
  tf.logical_or = lambda a, b: _t(np.logical_or(a, b))
  tf.logical_not = lambda a: _t(np.logical_not(a))
  tf.equal = lambda a, b: _t(np.equal(a, b))
  tf.ones_like = lambda x: _t(np.ones_like(np.asarray(x)))
  tf.zeros = lambda shape, dtype=None: _t(np.zeros(shape, _np_dtype(dtype) or np.float32))
  tf.TensorArray = _TensorArray
  tf.debugging = _NS(assert_equal=lambda x, y, message=None: None)
  tf.math = _NS(log=lambda x: _t(np.log(np.asarray(x))), xlogy=_xlogy,
                count_nonzero=lambda x, axis=None: _t(np.count_nonzero(np.asarray(x), axis=axis)),
                divide_no_nan=lambda a, b: _t(np.float32(0) if float(np.asarray(b)) == 0 else
                                              np.float32(np.asarray(a) / np.asarray(b))),
                reduce_mean=_reduce_mean)
  tf.nn.softmax = _softmax_folded
  tf.keras.losses = _NS(Loss=_Loss, Reduction=_NS(AUTO="auto", NONE="none", SUM="sum"), get=_keras_losses_get)
  tf.keras.metrics = _NS(Metric=_Metric, Mean=_Mean, Accuracy=_Accuracy)
  tf.metrics = tf.keras.metrics
  sys.modules["tensorflow.compat.v2"].__dict__.update(tf.__dict__)
  return tf
