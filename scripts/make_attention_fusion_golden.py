"""Writes tests/golden/engine_pre_attention_fusion.npz: the bf16 engine's logits, bases and qualities for seeded small
batches, as computed by the build before the q/k/v projection and the banded attention were fused into one kernel.

  python scripts/make_attention_fusion_golden.py [--out PATH]      (on a GPU; DCB200_LIB selects the build)

The fused kernel runs the same q/k/v wgmmas in the same K order, rounds them to bf16 the same way and runs the same
per-query-block attention arithmetic, so tests/test_gpu_attention_fused.py requires these outputs bit for bit.  The
configs cover window lengths around the 16-row query blocks and the 128-token tile, band widths from 1 to full
attention, ReZero and pre-LN models with and without ccs_bq, and a ragged batch whose tiles do not split evenly over
the SMs.  For the configs marked `debug` the debug capture's q/k/v and attention images of every layer are stored too.
Every config is stored as JSON next to its outputs, so the test rebuilds parameters, weights and rows from the file
alone; configs with many windows keep a sample of their windows (KEEP) to stay small.
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

OUT = os.path.join(ROOT, "tests", "golden", "engine_pre_attention_fusion.npz")


def configs(num_sms):
  """name -> synthetic_params arguments (win: attn_win_size, None = full attention), filter_size, windows, seeds and
  whether the debug images are kept."""
  c = dict(
      l1_win1=dict(L=1, win=1, windows=2, debug=True),
      l15_win12=dict(L=15, win=12, windows=2, debug=True),
      l16_full=dict(L=16, win=None, windows=2, debug=True),
      l17_win16_preln=dict(L=17, win=16, rezero=False, windows=2, debug=True),
      l64_win64_bq=dict(L=64, win=64, bq=True, windows=3),
      l100_win12_preln_bq=dict(L=100, win=12, rezero=False, bq=True, layers=3, windows=4),
      l120_bench=dict(L=120, win=12, layers=6, windows=8),                  # the bench workload's model
      l127_win1=dict(L=127, win=1, windows=3),
      l128_full=dict(L=128, win=None, layers=1, windows=1, debug=True),
      l128_win200_preln=dict(L=128, win=200, rezero=False, windows=3),
      ragged=dict(L=120, win=12, layers=1, ff=256, windows=4 * num_sms + 3),  # several tiles per CTA, odd halves
  )
  for i, (name, cfg) in enumerate(sorted(c.items())):
    cfg.setdefault("P", 20)
    cfg.setdefault("layers", 2)
    cfg.setdefault("ff", 512)
    cfg.setdefault("rezero", True)
    cfg.setdefault("bq", False)
    cfg.setdefault("debug", False)
    cfg.update(wseed=500 + i, rseed=600 + i)
  return c


def make(cfg):
  p = params_lib.synthetic_params(cfg["P"], cfg["L"], use_ccs_bq=cfg["bq"], num_hidden_layers=cfg["layers"],
                                  rezero=cfg["rezero"], attn_win_size=cfg["win"])
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
    if cfg["debug"]:
      model.set_debug(True)
    r = model.forward(rows, want_logits=True)
    if cfg["debug"]:
      tokens = cfg["windows"] * cfg["L"]
      for n in range(cfg["layers"]):
        out["%s/qkv%d" % (name, n)] = model.debug_operand(1 + 2 * n, "qkv", tokens)
        out["%s/att%d" % (name, n)] = model.debug_operand(1 + 2 * n, "att", tokens)
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
