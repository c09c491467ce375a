"""Feature construction, host against device, on one H100: what each stage of the front end costs next to the model.

  python scripts/time_features.py [--copies 60] [--out time_features.json]

Inputs: the human_1m BAM fixture repeated `--copies` times (so that every timed window exceeds a second) and seeded
synthetic ZMWs (15 kb CCS, 20 passes, about 8 % insertion columns; tests/test_prep_records_host.py makes them).  Prints
the card and its power limit, then
  host construction (csrc/bam_prep.cpp) in windows/s at 1, 4 and all worker threads,
  decode + validate + export alone (raw-record mode) at the same thread counts,
  device time of dcb_features_layout / dcb_features_pack per 1 024 windows (CUDA events, median of 20),
  `run` end to end with features="host" and "gpu" alternated, and the share of windows the skip decision removes.
  --smart-windows: only the device cost of CCS smart windows (tests/golden/human_1m/ccs_smart.bam, repeated x4):
  dcb_features_layout_smart plus dcb_features_ccs of the overflow windows per 1 024 windows, against
  dcb_features_layout's fixed cut of the same ZMWs.
Needs a GPU: there is no fallback."""
import argparse, gzip, json, os, shutil, struct, subprocess, sys, tempfile, time, zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
from deepconsensus_b200 import engine, params as params_lib, preprocess, run as run_lib, weights as weights_lib  # noqa: E402
import test_prep_records_host as host_side  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
EOF_BLOCK = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def repeat_bam(src, dst, copies):
  """A BAM holding the records of `src` `copies` times behind one header."""
  raw = open(src, "rb").read()
  members, pos = [], 0
  while pos < len(raw):
    size = (raw[pos + 16] | (raw[pos + 17] << 8)) + 1
    members.append(raw[pos:pos + size])
    pos += size
  plain = b"".join(gzip.decompress(m) for m in members)
  p = 4
  p += 4 + struct.unpack_from("<i", plain, p)[0]
  n_ref = struct.unpack_from("<i", plain, p)[0]
  p += 4
  for _ in range(n_ref):
    p += 4 + struct.unpack_from("<i", plain, p)[0] + 4
  data = plain[:p] + plain[p:] * copies
  with open(dst, "wb") as f:
    for i in range(0, len(data), 0xff00):
      blk = data[i:i + 0xff00]
      c = zlib.compressobj(6, zlib.DEFLATED, -15)
      comp = c.compress(blk) + c.flush()
      bs = len(comp) + 25
      f.write(bytes([31, 139, 8, 4, 0, 0, 0, 0, 0, 255, 6, 0, 66, 67, 2, 0, bs & 255, bs >> 8]) + comp)
      f.write(struct.pack("<II", zlib.crc32(blk), len(blk)))
    f.write(EOF_BLOCK)


def stream_rate(bams, P, L, threads, records):
  s = preprocess.BamFeatureStream(*bams, P, L, False, 5, threads=threads, records=records)
  t0, zmws, windows = time.time(), 0, 0
  while (z := s.next_zmw_records() if records else s.next_zmw(want_rows=False, want_packed=True)) is not None:
    zmws += 1
    windows += 0 if records else len(z["window_pos"])
  dt = time.time() - t0
  s.close()
  return dict(threads=threads, seconds=round(dt, 3), zmws=zmws, windows=windows)


def device_times(model, records, reps=20):
  lay = model.features_layout(records, 5)
  n = len(lay["window_pos"])
  dev = model.alloc_device(max(n, 1) * model.packed_window_bytes)
  a, b = [], []
  for _ in range(reps + 2):                                        # two warm-up rounds
    a.append(model.features_layout(records, 5)["ms"])
    b.append(model.features_pack(np.arange(n), out=dev)["ms"])
  model.free_device(dev)
  per = lambda ms: round(float(np.median(ms[2:])) * 1024 / n, 4)
  return dict(windows=n, layout_ms_per_1024_windows=per(a), pack_ms_per_1024_windows=per(b),
              upload_bytes_per_window=round(sum(v.nbytes for v in records.values()) / n))


def smart_window_times(reps=20):
  """Median device ms per 1 024 windows: fixed-width layout vs smart layout + full-width CCS of the overflow windows."""
  P, L = 20, 100
  bam = os.path.join(GOLDEN, "human_1m")
  recs = {}
  for smart in (False, True):
    s = preprocess.BamFeatureStream(os.path.join(bam, "subreads_to_ccs.bam"), os.path.join(bam, "ccs_smart.bam"), P, L, False, 5,
                                    records=True, use_ccs_smart_windows=smart)
    zs = []
    while (z := s.next_zmw_records()) is not None:
      zs.append(z)
    s.close()
    recs[smart] = engine.concat_records(zs * 4)
  p = params_lib.synthetic_params(P, L)
  model = engine.B200Model(p, weights_lib.init_weights(p, seed=3), max_batch=64)
  res = {}
  for smart, key in ((False, "fixed"), (True, "smart")):
    lay_ms, ccs_ms = [], []
    for _ in range(reps + 2):                                      # two warm-up rounds
      lay = model.features_layout(recs[smart], 5)
      lay_ms.append(lay["ms"])
      if smart:
        over = np.nonzero(lay["overflow"])[0]
        ccs_ms.append(model.features_ccs(over, lay["window_width"][over])["ms"])
    n = len(lay["window_pos"])
    per = lambda ms: round(float(np.median(ms[2:])) * 1024 / n, 4)
    res[key] = dict(windows=n, layout_ms_per_1024_windows=per(lay_ms))
    if smart:
      res[key].update(overflow_windows=int(len(over)), overflow_ccs_ms_per_1024_windows=per(ccs_ms))
  model.close()
  return res


def main():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument("--copies", type=int, default=60)
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--out", default=None)
  ap.add_argument("--smart-windows", action="store_true")
  a = ap.parse_args()
  import torch
  if not torch.cuda.is_available():
    raise SystemExit("time_features.py measures on a GPU; none is present")
  res = dict(card=subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                 capture_output=True, text=True).stdout.strip().splitlines()[0],
             host_cpus=os.cpu_count(), copies=a.copies)
  print(json.dumps(res), flush=True)
  if a.smart_windows:
    res["smart_windows"] = smart_window_times()
    print(json.dumps(res, indent=1))
    if a.out:
      os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
      json.dump(res, open(a.out, "w"), indent=1)
    return
  tmp = tempfile.mkdtemp()
  try:
    bams = tuple(os.path.join(tmp, n) for n in ("subreads_to_ccs.bam", "ccs.bam"))
    for n, dst in zip(("subreads_to_ccs.bam", "ccs.bam"), bams):
      repeat_bam(os.path.join(GOLDEN, "human_1m", n), dst, a.copies)
    P, L = 20, 100
    thread_counts = sorted({1, 4, os.cpu_count() or 1})
    res["host_construction"] = [stream_rate(bams, P, L, t, False) for t in thread_counts]
    windows = res["host_construction"][0]["windows"]
    for r in res["host_construction"]:
      r["windows_per_s"] = round(r["windows"] / r["seconds"])
    res["decode_export"] = [stream_rate(bams, P, L, t, True) for t in thread_counts]
    for r in res["decode_export"]:
      r["windows_per_s"] = round(windows / r["seconds"])          # the windows these ZMWs make
    print(json.dumps(dict(host_construction=res["host_construction"], decode_export=res["decode_export"])), flush=True)

    p = params_lib.synthetic_params(P, L)
    model = engine.B200Model(p, weights_lib.init_weights(p, seed=3), max_batch=1024)
    fixture = engine.concat_records(host_side.read_records(tuple(os.path.join(GOLDEN, "human_1m", n) for n in
                                                                 ("subreads_to_ccs.bam", "ccs.bam")), P, L, 0, 5) * 4)
    rng = np.random.default_rng(1)
    synth = engine.concat_records([host_side.set_clip(host_side.random_zmw(rng, 20, 15000, edge_cases=False), 5)
                                   for _ in range(8)])
    res["device"] = dict(fixture_x4=device_times(model, fixture), synthetic_15kb_20_passes=device_times(model, synth))
    model.close()
    print(json.dumps(res["device"]), flush=True)

    shutil.copytree(os.path.join(GOLDEN, "ckpt", "model"), os.path.join(tmp, "model"))
    runs = []
    for rnd in range(a.rounds + 1):                                # round 0 warms the page cache and is dropped
      for features in ("host", "gpu"):
        out = os.path.join(tmp, features + ".fastq")
        t0 = time.time()
        run_lib.run(subreads_to_ccs=bams[0], ccs_bam=bams[1], checkpoint=os.path.join(tmp, "model", "checkpoint-1"),
                    output=out, batch_zmws=100, batch_size=1024, min_quality=0, random_weights=3,
                    cpus=os.cpu_count() or 1, features=features)
        st = json.load(open(out + ".inference.json"))
        if rnd:
          runs.append(dict(features=features, wall_s=round(time.time() - t0, 2), windows=st["windows"],
                           seconds_features=round(st["seconds_features"], 2),
                           seconds_model_and_stitch=round(st["seconds_model_and_stitch"], 2),
                           windows_skipped=st.get("windows_skipped")))
    res["run"] = runs
    same = open(os.path.join(tmp, "host.fastq"), "rb").read() == open(os.path.join(tmp, "gpu.fastq"), "rb").read()
    res["run_outputs_identical"] = same
    sk = [r for r in runs if r["features"] == "gpu"][0]
    res["share_of_windows_skipped_at_q45"] = round(sk["windows_skipped"] / sk["windows"], 4)
  finally:
    shutil.rmtree(tmp, ignore_errors=True)
  print(json.dumps(res, indent=1))
  if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
  main()
