"""The three precisions side by side: device time of one forward of 1024 windows with bf16, tf32x3 and fp32 engines,
called in turn (median of `--iters` calls each), at the bench workload (P = 20, L = 120, 6 layers) and at L = 100; then a
torch.profiler split of the tf32x3 forward by kernel class and the GEMMs' rate from their shapes.  Prints one JSON line
with the card's name and power limit read in the same run.

  python scripts/time_precision.py [--iters 20] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from deepconsensus_b200 import engine, params as params_lib, synthetic, weights as weights_lib  # noqa: E402

PRECISIONS = ("bf16", "tf32x3", "fp32")
KERNEL_CLASSES = (("gemm", "tf32x3_gemm"), ("attention", "strict_attention"), ("layernorm", "strict_layernorm"),
                  ("embed", "strict_embed"), ("head", "strict_head"))


def gemm_flops(p, windows):
  """2 M K N of every GEMM of one forward (the useful products; 3xTF32 issues three times as many)."""
  m, d, ff = windows * int(p.max_length), int(p.hidden_size), int(p.filter_size)
  e = sum(s["width"] for s in params_lib.embedding_spec(p))
  return 2 * m * (e * d + int(p.num_hidden_layers) * (4 * d * d + 2 * d * ff))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--iters", type=int, default=20)
  ap.add_argument("--batch", type=int, default=1024)
  ap.add_argument("--out", default="")
  a = ap.parse_args()
  card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                        text=True).stdout.strip()
  result = dict(card=card, batch=a.batch, iters=a.iters, workloads={})
  for passes, length in ((20, 120), (20, 100)):
    p = params_lib.synthetic_params(passes, length)
    w = weights_lib.init_weights(p, seed=1)
    rows = synthetic.make_rows(p, a.batch, seed=2)
    models = {pr: engine.B200Model(p, w, max_batch=a.batch, precision=pr) for pr in PRECISIONS}
    ms = {pr: [] for pr in PRECISIONS}
    for pr in PRECISIONS:                      # warm-up
      models[pr].forward(rows)
    for _ in range(a.iters):
      for pr in PRECISIONS:
        models[pr].forward(rows)
        ms[pr].append(models[pr].last_ms)
    med = {pr: float(np.median(v)) for pr, v in ms.items()}
    entry = dict(median_ms=med, tf32x3_speedup_over_fp32=med["fp32"] / med["tf32x3"],
                 tf32x3_vs_bf16=med["tf32x3"] / med["bf16"], gemm_tflop=gemm_flops(p, a.batch) / 1e12)
    if (passes, length) == (20, 120):
      import torch
      from torch.profiler import ProfilerActivity, profile
      m3 = models["tf32x3"]
      with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
          m3.forward(rows)
      split = {k: 0.0 for k, _ in KERNEL_CLASSES}
      split["other"] = 0.0
      for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        if not t:
          continue
        cls = next((k for k, pat in KERNEL_CLASSES if pat in ev.key), "other")
        split[cls] += t / 3 / 1e3          # ms per forward
      entry["tf32x3_profile_ms"] = split
      entry["tf32x3_gemm_tflops_useful"] = gemm_flops(p, a.batch) / (split["gemm"] * 1e-3) / 1e12
      entry["tf32x3_gemm_tflops_issued"] = 3 * entry["tf32x3_gemm_tflops_useful"]
      del torch
    for m in models.values():
      m.close()
    result["workloads"]["P%d_L%d" % (passes, length)] = entry
  line = json.dumps(result)
  print(line)
  if a.out:
    with open(a.out, "w") as f:
      f.write(line + "\n")


if __name__ == "__main__":
  main()
