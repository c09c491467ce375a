"""Generates tests/golden/ref_student_init.json by EXECUTING the reference's own init_student_from_teacher
(deepconsensus/models/model_distillation.py:104-144, unmodified, from the checkout at REF) on the NumPy stand-in for
TensorFlow in scripts/tf_shim.py, with teacher and student built by the reference's networks.py as
scripts/make_model_golden.py builds them (Layer.get_weights / set_weights / Model.layers / get_layer restated there).

Every variable of both models gets a distinct seeded value (deepconsensus_b200.weights.init_weights); after the call,
each student variable is traced to where its value came from: the teacher variable it now equals, or "own".  Cases:
  distill_default     the transformer_learn_values_distill config (5-layer student, teacher layers [1..5] onto student
                      layers [0..4], both init flags set) from a 6-layer transformer_learn_values teacher, ReZero
  rezero_pair         ReZero, 3-layer teacher, 2-layer student, layers [2, 0] onto [0, 1], encoder stack only
  layernorm_pair      pre-LayerNorm, 3-layer teacher and student, layers [1, 1, 0] onto [0, 2, 1] (the dict keeps the
                      last student layer of a repeated teacher layer), both init flags set, CCS base qualities
tests/test_distill_grad_host.py rebuilds the same params and checks weights.student_from_teacher against the mapping.
Needs a checkout of google/deepconsensus v1.2 at REF and no GPU; the output is committed.
"""
import json
import os
import sys
import types

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "scripts"))
OUT = os.path.join(REPO, "tests", "golden", "ref_student_init.json")

import make_model_golden as mmg  # noqa: E402
import tf_shim  # noqa: E402

L = 40
CASES = [
    dict(name="distill_default", teacher=("transformer_learn_values+test", {}),
         student=("transformer_learn_values_distill+test", {}), seeds=(31, 32)),
    dict(name="rezero_pair", teacher=("transformer_learn_values+test", dict(num_hidden_layers=3)),
         student=("transformer_learn_values_distill+test",
                  dict(num_hidden_layers=2, teacher_encoder_layers=[2, 0], student_encoder_layers=[0, 1],
                       init_nonencoder_layers=False)), seeds=(33, 34)),
    dict(name="layernorm_pair", teacher=("transformer_learn_values+test",
                                         dict(num_hidden_layers=3, rezero=False, use_ccs_bq=True)),
         student=("transformer_learn_values_distill+test",
                  dict(num_hidden_layers=3, rezero=False, use_ccs_bq=True, teacher_encoder_layers=[1, 1, 0],
                       student_encoder_layers=[0, 2, 1])), seeds=(35, 36)),
]


def import_distillation():
  model_configs, model_utils, networks, _ = mmg.import_reference()
  tf = sys.modules["tensorflow"]
  tf_shim.install_losses_ops(tf)
  absl = sys.modules["absl"]
  for name in ("app", "flags"):
    mod = types.ModuleType("absl." + name)
    mod.__getattr__ = lambda k: tf_shim._Anything()
    setattr(absl, name, mod)
    sys.modules["absl." + name] = mod
  cf = types.ModuleType("ml_collections.config_flags")
  cf.config_flags = tf_shim._Anything()
  sys.modules["ml_collections.config_flags"] = cf
  sys.modules["ml_collections"].config_flags = cf
  from deepconsensus.models import model_distillation
  return model_configs, model_utils, networks, model_distillation


def build(model_configs, model_utils, networks, config, over, seed):
  from deepconsensus_b200 import params as P, weights as W
  params = model_configs.get_config(config)
  for k, v in over.items():
    params[k] = v
  model_utils.modify_params(params, max_length=L, is_training=False)
  mine = P.get_config(config)
  for k, v in over.items():
    mine[k] = v
  P.modify_params(mine, max_length=L)
  model = networks.EncoderOnlyLearnedValuesTransformer(params)
  model(np.zeros((1, params.total_rows, L, 1), np.float32), training=False)
  weights = W.init_weights(mine, seed=seed)
  mmg.assign_weights(model, weights)
  assert mmg.count_variables(model) == len(weights)
  return params, model, weights


def read(model, name):
  obj = model
  for p in name.split("/")[1:-1]:
    obj = obj[int(p)] if p.isdigit() else getattr(obj, p)
  return np.asarray(getattr(obj, name.split("/")[-1]))


def main():
  model_configs, model_utils, networks, md = import_distillation()
  out = {}
  for case in CASES:
    tp, teacher, tw = build(model_configs, model_utils, networks, *case["teacher"], case["seeds"][0])
    sp, student, sw = build(model_configs, model_utils, networks, *case["student"], case["seeds"][1])
    md.init_student_from_teacher(student, teacher, sp)
    by_value = {tw[k].tobytes() + repr(np.shape(tw[k])).encode(): k for k in tw}
    assert len(by_value) == len(tw)
    sources = {}
    for name in sorted(sw):
      v = read(student, name).astype(np.float32)
      key = v.tobytes() + repr(v.shape).encode()
      if key in by_value:
        sources[name] = by_value[key]
      else:
        assert v.tobytes() == sw[name].tobytes(), name
        sources[name] = "own"
    out[case["name"]] = dict(teacher=dict(config=case["teacher"][0], overrides=case["teacher"][1],
                                          seed=case["seeds"][0]),
                             student=dict(config=case["student"][0], overrides=case["student"][1],
                                          seed=case["seeds"][1]),
                             max_length=L, sources=sources)
    n_copied = sum(v != "own" for v in sources.values())
    print(case["name"], "copied", n_copied, "of", len(sources))
  with open(OUT, "w") as f:
    json.dump(out, f, indent=1, sort_keys=True)
  print("->", OUT)


if __name__ == "__main__":
  main()
