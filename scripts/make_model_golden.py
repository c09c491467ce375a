"""Generates tests/golden/ref_model_*.npz by EXECUTING the reference's own model code
(deepconsensus/models/{networks,encoder_stack,attention_layer,ffn_layer,data_providers,model_configs,
model_utils}.py, unmodified, from /root/reference) on the NumPy stand-in for TensorFlow in scripts/tf_shim.py.

What is pinned by these vectors (and checked by tests/test_oracle_model.py::test_oracle_matches_reference_code):
  * the reference's forward graph as written: row slicing, per-row embedding + concat order, the sqrt(width)
    scaling, the condenser, positional encoding add, band mask construction, the attention einsum wiring and
    head split, ReZero / pre-LayerNorm residual wrappers, FFN, final norm, fc1, softmax;
  * the checkpoint variable paths (weights are assigned through the same attribute paths a TF checkpoint uses);
  * params: model_configs.get_config + model_utils.modify_params run for real, and the derived keys are stored.
What is NOT pinned: TensorFlow's own kernels (the primitives are restated in tf_shim.py in float32), so float
summation order inside matmul/softmax/LN is NumPy's, not Eigen's.

Weights are NOT stored: they are regenerated from deepconsensus_b200.weights.init_weights(params, seed).
Run here (needs /root/reference); outputs are committed.
"""
import contextlib
import os
import sys
import types

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "scripts"))
REF = "/root/reference"
OUT = os.path.join(REPO, "tests", "golden")

import tf_shim  # noqa: E402


class RefConfigDict(tf_shim.ConfigDict):
  """ml_collections.ConfigDict surface that model_configs / modify_params use."""

  @contextlib.contextmanager
  def unlocked(self):
    yield self

  def lock(self):
    return self

  def __delattr__(self, k):
    del self[k]


def import_reference():
  tf = tf_shim.install()
  tf.config = types.SimpleNamespace(experimental=types.SimpleNamespace(list_physical_devices=lambda kind: []))
  sys.modules["tensorflow.compat.v2"].config = tf.config
  import ml_collections
  ml_collections.ConfigDict = RefConfigDict
  cd = sys.modules["ml_collections.config_dict"]
  cd.ConfigDict = RefConfigDict
  cd.placeholder = lambda t: None
  sys.modules["ml_collections.config_dict.config_dict"].ConfigDict = RefConfigDict
  for name in ("official.modeling", "official.modeling.optimization"):
    sys.modules[name] = types.ModuleType(name)
  sys.modules["official.modeling"].optimization = sys.modules["official.modeling.optimization"]
  absl = types.ModuleType("absl"); logging = types.ModuleType("absl.logging")
  logging.vlog = logging.info = logging.warning = lambda *a, **k: None
  absl.logging = logging
  sys.modules.setdefault("absl", absl); sys.modules.setdefault("absl.logging", logging)
  sys.path.insert(0, REF)
  from deepconsensus.models import model_configs, model_utils, networks, data_providers
  return model_configs, model_utils, networks, data_providers


def assign_weights(model, weights):
  """Assigns by checkpoint variable path: 'model/encoder_stack/layers/0/0/layer/query_dense_layer/kernel' is
  the attribute path model.encoder_stack.layers[0][0].layer.query_dense_layer.kernel."""
  for name, value in weights.items():
    parts = name.split("/")
    assert parts[0] == "model", name
    obj = model
    for p in parts[1:-1]:
      obj = obj[int(p)] if p.isdigit() else getattr(obj, p)
    cur = getattr(obj, parts[-1])
    assert cur is not None, f"variable {name} not created by the reference model"
    assert tuple(np.shape(cur)) == tuple(np.shape(value)), (name, np.shape(cur), np.shape(value))
    setattr(obj, parts[-1], np.array(value, dtype=np.float32))


def count_variables(obj, seen=None):
  """Counts ndarray-valued attributes reachable through Layer attributes/lists (the model's variables)."""
  seen = set() if seen is None else seen
  n = 0
  if id(obj) in seen:
    return 0
  seen.add(id(obj))
  if isinstance(obj, (list, tuple)):
    return sum(count_variables(o, seen) for o in obj)
  if isinstance(obj, tf_shim.Layer):
    for k, v in vars(obj).items():
      if k in ("params", "attn_mask"):   # attn_mask: a constant built in build(), not a variable
        continue
      if isinstance(v, np.ndarray):
        n += 1
      else:
        n += count_variables(v, seen)
  return n


def clip_boundaries(rows, p):
  """Puts values on every clip and id boundary of `p` into synthetic rows [B, R, L, 1] (in place): PW / IP at, just
  above and far beyond their maxima and below 0, SN on both sides of SN_MAX and far above 255, ccs_bq on its largest
  id, strand on its largest id."""
  from deepconsensus_b200 import params as params_lib
  (bases, pw, ip, strand, ccs, bq, sn) = params_lib.get_indices(p.max_passes, p.use_ccs_bq)
  for lo_hi, mx in ((pw, p.PW_MAX), (ip, p.IP_MAX)):
    for i, v in enumerate((mx, mx + 0.5, mx + 1, 300.0, -3.0, mx - 0.5)):
      rows[i % rows.shape[0], lo_hi[0]:lo_hi[1], 10 * i:10 * i + 10, 0] = v
  sn_values = ((p.SN_MAX - 0.5, p.SN_MAX, 1500.0, 255.5), (256.0, p.SN_MAX + 0.25, 0.0, 300.7),
               (p.SN_MAX + 0.5, 511.9, -2.0, p.SN_MAX - 1))
  for b, vals in enumerate(sn_values[:rows.shape[0]]):
    rows[b, sn[0]:sn[1], :, 0] = np.array(vals, np.float32)[:, None]
  rows[0, bq[0], :50, 0] = p.CCS_BQ_MAX - 2                  # id CCS_BQ_MAX - 1: the table's last row
  rows[1, bq[0], 50:, 0] = p.CCS_BQ_MAX - 2.5                # truncation toward zero: the id below it
  rows[2, bq[0], :, 0] = -1.0                                # id 0: the zero vector
  rows[0, strand[0]:strand[1], :, 0] = (np.arange(strand[1] - strand[0]) % (p.STRAND_MAX + 1))[:, None]
  rows[1, strand[0]:strand[1], :, 0] = p.STRAND_MAX
  return rows


CASES = [
    # name, config, overrides, window source, seed.  (The reference's testdata windows are 85 rows = no CCS-BQ row.)
    dict(name="rezero_p20", config="transformer_learn_values+test", over={}, src="real", n=6, seed=11),
    dict(name="layernorm_p20", config="transformer_learn_values+test",
         over=dict(rezero=False, num_hidden_layers=5), src="real", n=6, seed=12),
    dict(name="rezero_p20_bq", config="transformer_learn_values+test", over=dict(use_ccs_bq=True),
         src="synthetic", n=4, seed=13),
    dict(name="layernorm_p20_bq", config="transformer_learn_values+test",
         over=dict(use_ccs_bq=True, rezero=False, num_hidden_layers=5), src="synthetic", n=3, seed=15),
    dict(name="rezero_p5_win3", config="transformer_learn_values+test",
         over=dict(max_passes=5, attn_win_size=3, num_hidden_layers=2), src="synthetic", n=3, seed=14),
    # BASELINE configs[1] shape (20 subreads x 120 bp, 6 layers) and configs[4] shape (32 subreads x 200 bp)
    dict(name="c2_p20_l120", config="transformer_learn_values+test", over={}, src="synthetic", L=120, n=4, seed=16),
    dict(name="c5_p32_l200", config="transformer_learn_values+test", over=dict(max_passes=32), src="synthetic",
         L=200, n=3, seed=17),
    dict(name="c5_p32_l200_ln_bq", config="transformer_learn_values+test",
         over=dict(max_passes=32, use_ccs_bq=True, rezero=False, num_hidden_layers=5), src="synthetic", L=200, n=2,
         seed=18),
    # Embedding layouts a params.json can describe besides the default one (tests/test_embedding_layouts.py says which
    # embed / condenser paths each reaches).  E = embedded width, Epad = E rounded up to 16.
    # E = 127, Epad 128; widths 6/5/3/1/4 put 3+ input rows in one 8-column chunk; no positional table.
    dict(name="layout_narrow_nopos", config="transformer_learn_values+test",
         over=dict(max_passes=7, per_base_hidden_size=6, pw_hidden_size=5, ip_hidden_size=3, strand_hidden_size=1,
                   sn_hidden_size=4, PW_MAX=100, IP_MAX=60, SN_MAX=30, add_pos_encoding=False, num_hidden_layers=2),
         src="synthetic", L=40, n=3, seed=21),
    # E = 126 (2 padding columns); the ccs_bq and strand tables off their default widths; pre-LayerNorm.
    dict(name="layout_bq5_strand3_ln", config="transformer_learn_values+test",
         over=dict(max_passes=3, use_ccs_bq=True, ccs_bq_hidden_size=5, strand_hidden_size=3, rezero=False,
                   num_hidden_layers=2),
         src="synthetic", L=40, n=3, seed=22),
    # E = Epad = 1136: 71 condenser k-steps (odd) and not one chunk on the width-8 fast path.
    dict(name="layout_wide16_bq", config="transformer_learn_values+test",
         over=dict(max_passes=20, use_ccs_bq=True, per_base_hidden_size=16, pw_hidden_size=16, ip_hidden_size=16,
                   strand_hidden_size=4, ccs_bq_hidden_size=16, sn_hidden_size=16, num_hidden_layers=2),
         src="synthetic", L=100, n=3, seed=23),
    # E = 66, Epad 80 (14 padding columns, 5 k-steps); the window fills one 128-token tile exactly; no positional table.
    dict(name="layout_p1_l128_nopos_ln", config="transformer_learn_values+test",
         over=dict(max_passes=1, add_pos_encoding=False, rezero=False, num_hidden_layers=2),
         src="synthetic", L=128, n=3, seed=24),
    # E = 1704, Epad 1712 (107 k-steps); 261 input rows of ids in the embed kernel's shared memory.
    dict(name="layout_p64", config="transformer_learn_values+test",
         over=dict(max_passes=64, num_hidden_layers=1),
         src="synthetic", L=100, n=3, seed=25),
    # Clip maxima off their defaults, at the largest values packed rows hold; rows on every clip boundary.
    dict(name="layout_clip_maxima_bq", config="transformer_learn_values+test",
         over=dict(max_passes=20, use_ccs_bq=True, PW_MAX=255, IP_MAX=9, SN_MAX=1000, STRAND_MAX=3, CCS_BQ_MAX=256,
                   num_hidden_layers=2),
         src="synthetic", L=100, n=3, seed=26, edit=clip_boundaries),
]


def main():
  model_configs, model_utils, networks, data_providers = import_reference()
  from deepconsensus_b200 import weights as W, synthetic
  from deepconsensus_b200 import params as P
  real = np.load(os.path.join(OUT, "real_windows_human_1m.npz"))["rows"]
  only = set(sys.argv[1:])
  for case in CASES:
    if only and case["name"] not in only:
      continue
    params = model_configs.get_config(case["config"])
    for k, v in case["over"].items():
      params[k] = v
    max_length = case.get("L", 100 if case["src"] == "real" else 40)
    model_utils.modify_params(params, max_length=max_length, is_training=False)
    # our host-side params for the same request (validates deepconsensus_b200.params against the reference)
    mine = P.get_config(case["config"])
    for k, v in case["over"].items():
      mine[k] = v
    P.modify_params(mine, max_length=max_length)
    derived = ["total_rows", "hidden_size", "max_length", "max_passes", "num_hidden_layers", "filter_size",
               "num_heads", "attn_win_size", "transformer_input_size", "rezero", "use_ccs_bq"]
    for k in derived:
      assert params[k] == mine[k], (k, params[k], mine[k])

    if case["src"] == "real":
      rows = real[:case["n"]].astype(np.float32)[..., None]
    else:
      rows = synthetic.make_rows(mine, case["n"], seed=case["seed"])
      rows = rows.reshape(case["n"], mine.total_rows, max_length, 1).astype(np.float32)
    if "edit" in case:
      rows = case["edit"](rows, mine)
    assert rows.shape[1] == params.total_rows

    model = networks.EncoderOnlyLearnedValuesTransformer(params)
    # build all variables the way the reference does (model_utils.get_model: a call on zeros)
    model(np.zeros((1, params.total_rows, max_length, 1), np.float32), training=False)
    weights = W.init_weights(mine, seed=case["seed"])
    assign_weights(model, weights)
    nvar = count_variables(model)
    assert nvar == len(weights), (nvar, len(weights))

    # the reference's input formatting (clipping), per example as process_feature_dict does
    formatted = np.stack([np.asarray(data_providers.format_rows(subreads=r, params=params)) for r in rows])
    inter = model.get_intermediate_outputs(formatted, training=False)
    probs = np.asarray(model(formatted, training=False), np.float32)
    logits = np.asarray(inter["logits"], np.float32)
    out = dict(rows=rows[..., 0].astype(np.float32), formatted=formatted[..., 0].astype(np.float32), probs=probs, logits=logits,
               final_output=np.asarray(inter["final_output"], np.float32),
               config=np.array(case["config"]), seed=np.array(case["seed"]),
               overrides=np.array(repr(case["over"])), max_length=np.array(max_length),
               derived=np.array(repr({k: params[k] for k in derived})))
    for k in ("transformer_input", "encoder_input"):
      if k in inter:
        out[k] = np.asarray(inter[k], np.float32)
    path = os.path.join(OUT, f"ref_model_{case['name']}.npz")
    np.savez_compressed(path, **out)
    print(case["name"], "rows", rows.shape, "probs", probs.shape, "nvar", nvar,
          "pmax mean", float(probs.max(-1).mean()), "->", path)


if __name__ == "__main__":
  main()
