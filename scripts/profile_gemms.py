"""Per-GEMM kernel times of the bench workload, and the L2 -> shared-memory rate the GEMM's operand ring can reach.

  python scripts/profile_gemms.py --out DIR [--steps K]

Writes DIR/profile_gemms.json (and DIR/trace.json, the torch.profiler trace it was read from):
  kernels  torch.profiler (CUDA activities) over K pipelined steps of the bench workload (P20, L120, 6 layers, batch
           1024, packed rows resident in HBM).  The row-epilogue GEMM is one kernel for three launches of a layer, so
           each launch is named by the kernel before it: the condenser follows the embedding, the out-projection the
           attention, the FFN down-projection the FFN up-projection.  Builds with the fused FFN launch it twice per
           layer, named by their order in the layer: ffn_first and ffn_second, each over half of the tiles and the
           whole filter, with the row epilogue.  Builds that keep q/k/v on the SM (window-aligned layout) run the
           q/k/v projection and the attention as one kernel, also launched twice per layer: qkv_att_first and
           qkv_att_second; the out-projection then follows qkv_att_second.
  l2_read  for each GEMM, the bytes its CTAs read from L2 per launch (weights once per work item, activations,
           residual), computed from the shapes and the tiling, over its kernel time.
  hbm      for each FFN launch and each fused q/k/v + attention launch, the activation bytes it reads and writes in
           HBM (the weights stay in L2), computed from the image shapes, over its kernel time and against the H100
           SXM data sheet's 3.35 TB/s.
  timeline how the launches of one step sit on the GPU's clock: the span from its first kernel start to its last
           kernel end, the sum of kernel durations and the gap from each kernel to the next (negative where launches
           overlap), medians over the profiled steps.
  l2_ceiling  scripts/l2_stream.cu, compiled into a temporary directory: every SM streams the same L2-resident 1.18 MB
           weight image through the GEMM's 4-stage bulk-copy ring with consumers that only release the slots.
The card's name, power limit and clocks are recorded beside the numbers.  DCB200_LIB selects another build of the
library (engine.py), so two builds can be profiled by the same script.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from deepconsensus_b200 import params as params_lib, synthetic, weights as weights_lib  # noqa: E402

KDP = 288          # padded hidden size (csrc/common.h kDP)
TILE = 128         # tokens per tile (kTileM)


def gpu_info():
  q = "name,power.limit,clocks.max.sm,clocks.sm"
  try:
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=10).stdout.strip()
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
  except Exception as e:  # noqa: BLE001
    return dict(error=str(e))


def l2_bytes(role, ntiles, ff, epad, tokens):
  """Bytes the CTAs of one launch read from L2.  Weights cross from L2 once per work item: `tokens` tokens for the
  resident-A GEMMs (q/k/v, FFN up: a tile pair, or one tile in builds before pairs), one 128-token tile for the row
  GEMMs.  Split-bf16 weights (q/k/v, out-projection, condenser) count twice, and so do the row GEMMs' A k-steps."""
  a_tile = TILE * 2
  passes = ntiles * TILE // tokens if role in ("qkv", "ffn_up") else ntiles
  if role == "qkv":
    return passes * (864 * 2 * KDP * 2) + ntiles * a_tile * KDP
  if role == "ffn_up":
    return passes * (ff * KDP * 2) + ntiles * a_tile * KDP
  res = ntiles * TILE * KDP * 4    # fp32 residual image, read by the row epilogue
  if role == "out_proj":
    return passes * (KDP * 2 * KDP * 2) + ntiles * 2 * a_tile * KDP + res
  if role == "ffn_down":
    return passes * (KDP * ff * 2) + ntiles * a_tile * ff + res
  if role == "condenser":
    return passes * (KDP * 2 * epad * 2) + ntiles * 2 * a_tile * epad
  if role in ("ffn_first", "ffn_second"):    # one tile per work item: the whole of W1 and W2, xb, the residual
    n = ffn_half_tiles(role, ntiles)
    return n * (ff * KDP * 2 * 2 + a_tile * KDP + TILE * KDP * 4)
  if role in ("qkv_att_first", "qkv_att_second"):   # one tile per work item: the split-bf16 q/k/v weights, xb
    return ffn_half_tiles(role, ntiles) * (864 * 2 * KDP * 2 + a_tile * KDP)
  return None


def ffn_half_tiles(role, ntiles):
  """Tiles of the two-launch kernel `role` (FFN or q/k/v + attention): the first takes ceil(ntiles / 2), the second
  the rest."""
  return (ntiles + 1) // 2 if role in ("ffn_first", "qkv_att_first") else ntiles // 2


HBM_TBPS = 3.35    # H100 SXM data sheet


def hbm_bytes(role, ntiles, ff):
  """Activation bytes one FFN launch reads and writes in HBM: bf16 xb / hidden images and the fp32 residual image
  (the next layer's xb is counted for every layer).  ffn_first / ffn_second: xb in, residual in and out, next xb out
  for the launch's half of the tiles.  qkv_att_first / qkv_att_second: xb in, the attention image out."""
  if role in ("ffn_first", "ffn_second", "qkv_att_first", "qkv_att_second"):
    ntiles = ffn_half_tiles(role, ntiles)
  xb = ntiles * TILE * KDP * 2
  x = ntiles * TILE * KDP * 4
  hid = ntiles * TILE * ff * 2
  return {"ffn_up": xb + hid, "ffn_down": hid + x + x + xb,
          "ffn_first": xb + x + x + xb, "ffn_second": xb + x + x + xb,
          "qkv_att_first": xb + xb, "qkv_att_second": xb + xb}.get(role)


def timeline(kernels, roles):
  """How the launches of one step sit on the GPU's clock.  A step runs from one embedding kernel to the kernel before
  the next.  span_us: first kernel start to last kernel end; kernel_us: the sum of kernel durations; gaps_us: from each
  kernel's end to the next one's start, named by the two roles (negative where the next launch overlaps the one
  before it).  Each is the median over the profiled steps; between_steps_us is the gap from a step's last kernel to
  the next step's first."""
  steps, cur = [], []
  for e, r in zip(kernels, roles):
    if r == "embed" and cur:
      steps.append(cur)
      cur = []
    cur.append((r, float(e["ts"]), float(e["dur"])))
  if cur:
    steps.append(cur)
  full = [s for s in steps if len(s) == len(steps[0])]
  gaps, spans, sums = {}, [], []
  for s in full:
    spans.append(max(t + d for _, t, d in s) - s[0][1])
    sums.append(sum(d for _, _, d in s))
    for i in range(1, len(s)):
      name = "%02d %s->%s" % (i, s[i - 1][0], s[i][0])
      gaps.setdefault(name, []).append(s[i][1] - (s[i - 1][1] + s[i - 1][2]))
  between = [b[0][1] - max(t + d for _, t, d in a) for a, b in zip(steps, steps[1:])]
  med = lambda v: float(np.median(v)) if v else None  # noqa: E731
  g = {k: med(v) for k, v in gaps.items()}
  return dict(steps=len(full), launches_per_step=len(steps[0]) if steps else 0, span_us=med(spans),
              kernel_us=med(sums), idle_us=med([a - b for a, b in zip(spans, sums)]),
              gap_sum_us=float(sum(g.values())), between_steps_us=med(between), gaps_us=g)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--out", required=True)
  ap.add_argument("--steps", type=int, default=20)
  ap.add_argument("--warmup", type=int, default=5)
  ap.add_argument("--batch", type=int, default=1024)
  ap.add_argument("--tokens", type=int, default=256,
                  help="tokens a q/k/v or FFN-up work item covers, i.e. per weight pass from L2 (256 = tile pairs; "
                       "128 for builds with one tile per item)")
  ap.add_argument("--label", default="")
  args = ap.parse_args()
  os.makedirs(args.out, exist_ok=True)
  result = dict(label=args.label, library=os.environ.get("DCB200_LIB", "in-tree libdcb200.so"), gpu=gpu_info())

  # ---- the L2 -> SM ceiling, in a process of its own
  with tempfile.TemporaryDirectory() as td:
    exe = os.path.join(td, "l2_stream")
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-o", exe,
                    os.path.join(ROOT, "scripts", "l2_stream.cu")], check=True)
    result["l2_ceiling"] = [json.loads(subprocess.run([exe, "40", str(kb)], capture_output=True, text=True,
                                                      check=True).stdout) for kb in (4096, 4608)]

  import torch
  from torch.profiler import ProfilerActivity, profile
  from deepconsensus_b200 import engine as engine_lib

  p = params_lib.synthetic_params(max_passes=20, max_length=120, num_hidden_layers=6)
  w = weights_lib.init_weights(p, seed=1)
  B = args.batch
  model = engine_lib.B200Model(p, w, max_batch=B, device=0)
  stride = model.packed_window_bytes
  NBUF = 4
  dev = []
  for i in range(NBUF):
    rows = synthetic.make_rows(p, B, seed=20240921 + 1 + i)[..., 0]
    d = model.alloc_device(B * stride)
    model.memcpy_h2d(d, model.pack_rows(rows))
    dev.append(d)
  bases, quals = model.alloc_device(B * p.max_length), model.alloc_device(B * p.max_length)
  FL = engine_lib.DCB_ROWS_ON_DEVICE | engine_lib.DCB_OUT_ON_DEVICE

  def run(steps):
    pending = None
    for i in range(steps):
      t = model.submit_packed_raw(dev[i % NBUF], B, FL, bases, quals)
      if pending is not None:
        model.wait_raw(pending)
      pending = t
    model.wait_raw(pending)

  run(args.warmup)
  torch.cuda.synchronize()
  trace = os.path.join(args.out, "trace.json")
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    run(args.steps)
    torch.cuda.synchronize()
  prof.export_chrome_trace(trace)
  with open(trace) as f:
    events = json.load(f)["traceEvents"]
  kernels = sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e["ts"])

  def role_of(name, prev):
    if "ffn_gemm_kernel" in name:
      return "ffn_second" if prev == "ffn_first" else "ffn_first"
    if "qkv_attention_kernel" in name:
      return "qkv_att_second" if prev == "qkv_att_first" else "qkv_att_first"
    m = re.search(r"gemm_kernel<(\d+), (\d+), (\d+), (true|false)>", name)
    if m:
      epi = int(m.group(3))
      if epi == 0:
        return "qkv"
      if epi == 2:
        return "ffn_up"
      return {"embed": "condenser", "attention": "out_proj", "qkv_att_second": "out_proj",
              "ffn_up": "ffn_down"}.get(prev, "row_other")
    for key in ("embed", "attention", "head", "unpack", "stitch"):
      if key in name:
        return key
    return "other"

  per = {}
  prev = None
  roles = []
  for e in kernels:
    r = role_of(e["name"], prev)
    prev = r
    roles.append(r)
    d = per.setdefault(r, dict(launches=0, us=[], name=e["name"].split("(")[0]))
    d["launches"] += 1
    d["us"].append(float(e["dur"]))
  ntiles = B * ((p.max_length + TILE - 1) // TILE * TILE) // TILE     # window-aligned layout (the default)
  epad = (params_lib.embedded_width(p) + 15) // 16 * 16
  out = {}
  total = sum(sum(d["us"]) for d in per.values())
  for r, d in per.items():
    us = np.array(d["us"])
    rec = dict(kernel=d["name"], launches=d["launches"], ms_per_step=float(us.sum()) / 1e3 / args.steps,
               mean_us=float(us.mean()), median_us=float(np.median(us)), share=float(us.sum() / total))
    nb = l2_bytes(r, ntiles, p.filter_size, epad, args.tokens)
    if nb is not None:
      rec["l2_read_bytes_per_launch"] = nb
      rec["l2_read_tbps"] = nb / (float(np.median(us)) * 1e-6) / 1e12
    hb = hbm_bytes(r, ntiles, p.filter_size)
    if hb is not None:
      rec["hbm_bytes_per_launch"] = hb
      rec["hbm_tbps"] = hb / (float(np.median(us)) * 1e-6) / 1e12
      rec["hbm_share_of_3_35_tbps"] = rec["hbm_tbps"] / HBM_TBPS
    out[r] = rec
  result.update(kernels=out, steps=args.steps, batch=B, ntiles=ntiles, tokens=args.tokens,
                kernel_ms_per_step=total / 1e3 / args.steps, timeline=timeline(kernels, roles), gpu_after=gpu_info())
  with open(os.path.join(args.out, "profile_gemms.json"), "w") as f:
    json.dump(result, f, indent=1)
  print(json.dumps(result))
  for d in dev + [bases, quals]:
    model.free_device(d)
  model.close()


if __name__ == "__main__":
  main()
