"""Model params for the hot path, without ml_collections / TensorFlow.

Host-side mirror of the params surface `deepconsensus run` uses:

* `get_config(name)`            <- models/model_configs.py:252-379
* `read_params_from_json(path)` <- models/model_utils.py:434-465
* `modify_params(params, ...)`  <- models/model_utils.py:237-354 (inference part)
* `get_total_rows`, `get_indices` <- models/data_providers.py:61-113

Only the keys that shape the inference path are derived; training-only keys in a
`params.json` are carried through untouched so a reference checkpoint directory
can be pointed at directly.
"""
from __future__ import annotations

import json
import os
from typing import Any, Dict, Iterator, Optional, Tuple


class Params(dict):
  """dict with attribute access (the subset of ConfigDict behaviour the path needs)."""

  def __getattr__(self, key: str) -> Any:
    try:
      return self[key]
    except KeyError as e:
      raise AttributeError(key) from e

  def __setattr__(self, key: str, value: Any) -> None:
    self[key] = value

  def __delattr__(self, key: str) -> None:
    del self[key]

  def copy(self) -> "Params":
    return Params(self)


# transformer_basic_params.py:33-67 ("base" size).  Only merged for keys that a
# config does not already define (model_utils.py:347-354), which is why
# num_heads stays 2 (model_configs.py:84) and hidden_size stays 280.
_TRANSFORMER_BASE = dict(
    default_batch_size=2048, default_batch_size_tpu=32768, max_length=256,
    initializer_gain=1.0, vocab_size=33708, hidden_size=512,
    num_hidden_layers=6, num_heads=8, filter_size=2048,
    layer_postprocess_dropout=0.1, attention_dropout=0.1, relu_dropout=0.1,
    label_smoothing=0.1, learning_rate=2.0, learning_rate_decay_rate=1.0,
    learning_rate_warmup_steps=16000, optimizer_adam_beta1=0.9,
    optimizer_adam_beta2=0.997, optimizer_adam_epsilon=1e-09,
    extra_decode_length=50, beam_size=4, alpha=0.6, use_tpu=False,
    static_batch=False, allow_ffn_pad=True,
)
_TRANSFORMER_SIZES = {
    "base": _TRANSFORMER_BASE,
    "big": dict(_TRANSFORMER_BASE, default_batch_size=4096,
                default_batch_size_tpu=16384, hidden_size=1024,
                filter_size=4096, num_heads=16),
    "tiny": dict(_TRANSFORMER_BASE, default_batch_size=1024,
                 default_batch_size_tpu=1024, hidden_size=32, num_heads=4,
                 filter_size=256),
}


def get_total_rows(max_passes: int, use_ccs_bq: bool) -> int:
  """Rows of one example: 4 per subread + ccs + [ccs_bq] + 4 sn (data_providers.py:61-78)."""
  return 4 * max_passes + (6 if use_ccs_bq else 5)


def get_indices(max_passes: int, use_ccs_bq: bool) -> Tuple[Tuple[int, int], ...]:
  """(start, end) row ranges: bases, pw, ip, strand, ccs, ccs_bq, sn (data_providers.py:81-113)."""
  p = max_passes
  ccs = (4 * p, 4 * p + 1)
  if use_ccs_bq:
    bq, sn = (4 * p + 1, 4 * p + 2), (4 * p + 2, 4 * p + 6)
  else:
    bq, sn = (0, 0), (4 * p + 1, 4 * p + 5)
  return ((0, p), (p, 2 * p), (2 * p, 3 * p), (3 * p, 4 * p), ccs, bq, sn)


def _base_config() -> Params:
  """Defaults every config starts from (model_configs.py:272-338)."""
  p = Params()
  p.trial = 1
  p.rezero = False                   # old checkpoints: LayerNorm wrappers (:286)
  p.PW_MAX, p.IP_MAX, p.SN_MAX, p.CCS_BQ_MAX, p.STRAND_MAX = 255, 255, 500, 95, 2
  p.use_bases = p.use_pw = p.use_ip = p.use_strand = p.use_sn = p.use_ccs = True
  p.use_ccs_bq = False
  p.per_base_hidden_size = p.pw_hidden_size = p.ip_hidden_size = 1
  p.sn_hidden_size = p.strand_hidden_size = p.ccs_bq_hidden_size = 1
  p.total_rows = None
  p.vocab_size = 5
  p.seed = 1
  p.remove_label_gaps = False
  p.loss_function = "alignment_loss"
  p.del_cost, p.loss_reg, p.band_width = 10.0, 0.1, None
  p.max_length = 100
  p.model_config_name = "transformer_learn_values"
  p.dataset_config_name = "ccs"
  p.tpu_scale_factor = 1
  return p


def _set_transformer(p: Params) -> None:
  """model_configs.py:76-123 (architecture keys only)."""
  p.model_name = "transformer"
  p.add_pos_encoding = True
  p.num_heads = 2
  p.layer_norm = False               # never read by the model (SURVEY G.6)
  p.rezero = True
  p.condense_transformer_input = False
  p.transformer_model_size = "base"
  p.attn_win_size = 12
  p.num_channels = 1
  p.layer_postprocess_dropout = p.attention_dropout = p.relu_dropout = 0.1
  p.batch_size = 256


def _set_learn_values(p: Params) -> None:
  """model_configs.py:126-139."""
  _set_transformer(p)
  p.model_name = "transformer_learn_values"
  p.per_base_hidden_size = p.pw_hidden_size = p.ip_hidden_size = 8
  p.strand_hidden_size = 2
  p.sn_hidden_size = p.ccs_bq_hidden_size = 8
  p.condense_transformer_input = True
  p.transformer_input_size = 280


def get_config(config_name: Optional[str] = None) -> Params:
  """`"{model}+{dataset}"` -> params (model_configs.py:252-379)."""
  p = _base_config()
  if config_name is None:
    return p
  model_cfg, data_cfg = config_name.split("+")
  p.model_config_name, p.dataset_config_name = model_cfg, data_cfg
  if model_cfg == "transformer":
    _set_transformer(p)
  elif model_cfg == "transformer_learn_values":
    _set_learn_values(p)
  elif model_cfg == "transformer_learn_values_distill":
    _set_learn_values(p)             # model_configs.py:150-190
    p.model_name = "transformer_learn_values_distill"
    p.num_hidden_layers, p.filter_size = 5, 2048
    p.layer_postprocess_dropout, p.attention_dropout, p.relu_dropout = 0.0, 0.1, 0.0
    p.init_encoder_stack = p.init_nonencoder_layers = True
    p.teacher_encoder_layers, p.student_encoder_layers = [1, 2, 3, 4, 5], [0, 1, 2, 3, 4]
    p.distill_alpha, p.student_alpha, p.temperature = 1.0e5, 1.0, 1.0
    p.logit_loss_identifier = "mean_squared_error"
  else:
    raise ValueError("Unknown model_config_name: %s" % model_cfg)
  if data_cfg in ("test", "custom"):
    p.max_passes = 20                # model_configs.py:146,203
    if data_cfg == "test":
      p.batch_size = 1
  elif data_cfg == "test_bq":
    p.max_passes, p.use_ccs_bq, p.batch_size = 20, True, 1  # :220-233
  else:
    # The OSS reference never defines the poa/ccs/ecoli setters (SURVEY G.5).
    raise ValueError(
        "dataset_config_name is %s. Must be one of: test, test_bq, custom" % data_cfg)
  return p


def read_params_from_json(checkpoint_path: str) -> Params:
  """params.json next to a checkpoint, merged over the base config (model_utils.py:434-465)."""
  p = get_config()
  d = checkpoint_path if os.path.isdir(checkpoint_path) else os.path.dirname(checkpoint_path)
  with open(os.path.join(d, "params.json"), "r") as f:
    p.update(json.load(f))
  p.total_rows = get_total_rows(p.max_passes, p.use_ccs_bq)
  return p


def modify_params(params: Params, max_length: Optional[int] = None,
                  is_training: bool = False, **_unused) -> None:
  """Derived keys for inference (model_utils.py:237-354, device/TPU branches dropped)."""
  if not is_training:
    for k in ("tf_dataset", "train_path", "eval_path", "test_path", "inference_path"):
      params.pop(k, None)
  if max_length is not None:
    params.max_length = max_length
  if params.get("max_length") is None:
    raise ValueError("No params.max_length provided.")
  params.total_rows = get_total_rows(params.max_passes, params.use_ccs_bq)
  if "transformer_learn_values" in params.model_name:
    dim = (params.use_bases * params.per_base_hidden_size
           + params.use_pw * params.pw_hidden_size
           + params.use_ip * params.ip_hidden_size
           + params.use_strand * params.strand_hidden_size
           + params.use_ccs_bq * params.ccs_bq_hidden_size)
    # NOTE: faithful to model_utils.py:320-331 -- this counts ccs_bq once per
    # subread; it is overwritten by transformer_input_size when condensing.
    params.hidden_size = (params.max_passes * dim
                          + params.use_ccs * params.per_base_hidden_size
                          + params.use_ccs_bq * params.ccs_bq_hidden_size
                          + params.use_sn * params.sn_hidden_size * 4)
  else:
    params.hidden_size = params.total_rows
  if "transformer" in params.model_name and params.hidden_size % 2 != 0:
    params.hidden_size += 1
  if "transformer_learn_values" in params.model_name:
    params.default_batch_size = params.get("batch_size", 1)
    if params.condense_transformer_input:
      params.hidden_size = params.transformer_input_size
  if "transformer" in params.model_name:
    for k, v in _TRANSFORMER_SIZES[params.get("transformer_model_size", "base")].items():
      if k not in params:
        params[k] = v


def embedding_spec(params: Params) -> Iterator[Dict[str, Any]]:
  """Yields, in concat order, one dict per embedded input row.

  Order and table sharing follow `EncoderOnlyLearnedValuesTransformer.encode`
  (networks.py:457-504): bases[P], pw[P], ip[P], strand[P], ccs (bases table),
  [ccs_bq (+1 shift)], sn[4].
  """
  (bases, pw, ip, strand, ccs, bq, sn) = get_indices(params.max_passes, params.use_ccs_bq)
  groups = []
  if params.use_bases:
    groups.append(("bases", bases, params.per_base_hidden_size, 0))
  if params.use_pw:
    groups.append(("pw", pw, params.pw_hidden_size, 0))
  if params.use_ip:
    groups.append(("ip", ip, params.ip_hidden_size, 0))
  if params.use_strand:
    groups.append(("strand", strand, params.strand_hidden_size, 0))
  if params.use_ccs:
    groups.append(("bases", ccs, params.per_base_hidden_size, 0))
  if params.use_ccs_bq:
    groups.append(("ccs_bq", bq, params.ccs_bq_hidden_size, 1))
  if params.use_sn:
    groups.append(("sn", sn, params.sn_hidden_size, 0))
  off = 0
  for table, (lo, hi), width, shift in groups:
    for r in range(lo, hi):
      yield dict(table=table, row=r, width=width, shift=shift, offset=off)
      off += width


def table_vocab(params: Params) -> Dict[str, Tuple[int, int]]:
  """table name -> (vocab, width) (networks.py:375-421)."""
  out = {}
  if params.use_bases or params.use_ccs:
    out["bases"] = (5, params.per_base_hidden_size)
  if params.use_pw:
    out["pw"] = (params.PW_MAX + 1, params.pw_hidden_size)
  if params.use_ip:
    out["ip"] = (params.IP_MAX + 1, params.ip_hidden_size)
  if params.use_strand:
    out["strand"] = (params.STRAND_MAX + 1, params.strand_hidden_size)
  if params.use_ccs_bq:
    out["ccs_bq"] = (params.CCS_BQ_MAX, params.ccs_bq_hidden_size)
  if params.use_sn:
    out["sn"] = (params.SN_MAX + 1, params.sn_hidden_size)
  return out


def embedded_width(params: Params) -> int:
  """E: width of the concatenated embedding fed to the condenser."""
  return sum(s["width"] for s in embedding_spec(params))


def synthetic_params(max_passes: int = 20, max_length: int = 120, use_ccs_bq: bool = False,
                     num_hidden_layers: int = 6, rezero: bool = True,
                     attn_win_size: Optional[int] = 12) -> Params:
  """Params for the BASELINE.json synthetic configs (no params.json on disk)."""
  p = get_config("transformer_learn_values+test_bq" if use_ccs_bq
                 else "transformer_learn_values+test")
  p.max_passes = max_passes
  p.rezero = rezero
  p.attn_win_size = attn_win_size
  p.num_hidden_layers = num_hidden_layers
  modify_params(p, max_length=max_length)
  return p
