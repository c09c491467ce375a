"""Writes tests/golden/engine_logits_pre_ffn_fusion.npz: the bf16 engine's logits, bases and qualities for seeded small
batches, as computed by the build before the FFN's up- and down-projection were fused into one kernel.

  python scripts/make_engine_logits_golden.py [--out PATH]      (on a GPU; DCB200_LIB selects the build)

The fused FFN performs the same operations in the same order (the same wgmma shapes and K order, the same bias, ReLU and
bf16 rounding of the hidden activation, one fp32 accumulator per output), so tests/test_gpu_ffn_fused.py requires these
outputs bit for bit.  Every config is stored as JSON next to its outputs, so the test rebuilds parameters, weights and
rows from the file alone.  Configs with many windows keep a sample of their windows (KEEP) to stay small.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from deepconsensus_b200 import params as params_lib, synthetic, weights as weights_lib  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "engine_logits_pre_ffn_fusion.npz")


def configs(num_sms):
  """name -> synthetic_params arguments, filter_size, windows and seeds."""
  c = dict(
      bench=dict(P=20, L=120, layers=6, windows=8),                                # the bench workload's model
      ff128=dict(P=20, L=100, layers=2, ff=128, windows=5),                        # one hidden chunk: nothing in launch 2
      ff256=dict(P=20, L=100, layers=2, ff=256, windows=5),
      ff640=dict(P=20, L=100, layers=2, ff=640, windows=5),                        # five chunks: an odd split
      preln_bq=dict(P=20, L=100, layers=3, rezero=False, bq=True, windows=4),
      p32_l200=dict(P=32, L=200, layers=2, windows=3),                             # windows packed across tiles
      ragged=dict(P=20, L=100, layers=1, ff=256, windows=4 * num_sms + 3),        # several tiles per CTA, odd count
  )
  for i, (name, cfg) in enumerate(sorted(c.items())):
    cfg.setdefault("ff", 2048)
    cfg.setdefault("rezero", True)
    cfg.setdefault("bq", False)
    cfg.update(wseed=300 + i, rseed=400 + i)
  return c


def make(cfg):
  p = params_lib.synthetic_params(cfg["P"], cfg["L"], use_ccs_bq=cfg["bq"], num_hidden_layers=cfg["layers"],
                                  rezero=cfg["rezero"])
  p.filter_size = cfg["ff"]
  return p, weights_lib.init_weights(p, seed=cfg["wseed"]), synthetic.make_rows(p, cfg["windows"], seed=cfg["rseed"])


KEEP = 16   # configs with more windows keep the first KEEP, every KEEP-th and the last KEEP


def kept(windows):
  if windows <= 3 * KEEP:
    return np.arange(windows)
  return np.unique(np.concatenate([np.arange(KEEP), np.arange(0, windows, KEEP), np.arange(windows - KEEP, windows)]))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--out", default=OUT)
  args = ap.parse_args()
  import torch
  from deepconsensus_b200 import engine
  cfgs = configs(torch.cuda.get_device_properties(0).multi_processor_count)
  out = dict(configs=np.array(json.dumps(cfgs)))
  for name, cfg in cfgs.items():
    p, w, rows = make(cfg)
    model = engine.B200Model(p, w, max_batch=cfg["windows"])
    r = model.forward(rows, want_logits=True)
    model.close()
    idx = kept(cfg["windows"])
    for k in ("bases", "quals", "logits"):
      out["%s/%s" % (name, k)] = np.ascontiguousarray(r[k][idx])
    out["%s/windows" % name] = idx
    print(name, cfg, "kept", len(idx), "windows")
  os.makedirs(os.path.dirname(args.out), exist_ok=True)
  np.savez_compressed(args.out, **out)
  print("wrote", args.out, os.path.getsize(args.out), "bytes")


if __name__ == "__main__":
  main()
