"""`evaluate` from BAMs, the parts that need no GPU: the argument checks of the second input form, the ZMW selection it
shares with training-mode `preprocess` (on the fixture's host stream, no engine), and the compiled kernels of
dcb_features_eval and of dcb_evaluate's device label check."""
import collections
import gzip
import json
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

from deepconsensus_b200 import engine, evaluate, preprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def fx(golden_dir):
  d = os.path.join(golden_dir, "human_1m")
  return dict(subreads_to_ccs=os.path.join(d, "subreads_to_ccs.bam"), ccs_bam=os.path.join(d, "ccs.bam"),
              truth_to_ccs=os.path.join(d, "truth_to_ccs.bam"), truth_bed=os.path.join(d, "truth.bed"),
              truth_split=os.path.join(d, "truth_split.tsv"), digest=os.path.join(d, "training_digest.json.gz"),
              ckpt=os.path.join(golden_dir, "ckpt", "model"),
              eval_tf=os.path.join(d, "tf_examples", "eval", "eval.tfrecord.gz"))


def _cli(fx, tmp_path, extra):
  base = ["--checkpoint", fx["ckpt"], "--out_dir", str(tmp_path / "out")]
  return subprocess.run([sys.executable, "-m", "deepconsensus_b200.evaluate"] + base + extra, capture_output=True,
                        text=True, cwd=ROOT)


def _bam_flags(fx):
  out = []
  for k in ("subreads_to_ccs", "ccs_bam", "truth_to_ccs", "truth_bed", "truth_split"):
    out += ["--" + k, fx[k]]
  return out


def test_the_two_input_forms_are_exclusive(fx, tmp_path):
  bam = {k: fx[k] for k in ("subreads_to_ccs", "ccs_bam", "truth_to_ccs", "truth_bed", "truth_split")}
  with pytest.raises(ValueError, match="exclusive"):
    evaluate.run(fx["ckpt"], [fx["eval_tf"]], str(tmp_path), split=["eval"], **bam)
  with pytest.raises(ValueError, match="exclusive"):
    evaluate.run(fx["ckpt"], [fx["eval_tf"]], str(tmp_path), subreads_to_ccs=fx["subreads_to_ccs"])
  with pytest.raises(ValueError, match="either --eval_path or the BAM inputs"):
    evaluate.run(fx["ckpt"], None, str(tmp_path))
  with pytest.raises(ValueError, match="also need --truth_bed"):
    evaluate.run(fx["ckpt"], None, str(tmp_path), split=["eval"], **dict(bam, truth_bed=None))
  with pytest.raises(ValueError, match="at least one --split"):
    evaluate.run(fx["ckpt"], None, str(tmp_path), **bam)
  r = _cli(fx, tmp_path, ["--eval_path", fx["eval_tf"], "--split", "eval"] + _bam_flags(fx))
  assert r.returncode == 2 and "exclusive" in r.stderr, r.stderr
  assert not os.path.exists(str(tmp_path / "out"))


@pytest.mark.parametrize("split", ["validation", "Eval", ""])
def test_a_split_the_split_file_never_produces_is_refused(fx, tmp_path, split):
  bam = {k: fx[k] for k in ("subreads_to_ccs", "ccs_bam", "truth_to_ccs", "truth_bed", "truth_split")}
  with pytest.raises(ValueError, match="assigns its contigs only to eval, test, train"):
    evaluate.run(fx["ckpt"], None, str(tmp_path), split=["eval", split], **bam)
  r = _cli(fx, tmp_path, ["--split", "test", "--split", split] + _bam_flags(fx))
  assert r.returncode == 2 and "assigns its contigs only to" in r.stderr, r.stderr


def test_a_split_file_without_a_split_refuses_every_split(fx, tmp_path):
  other = tmp_path / "human_split.tsv"
  other.write_text("tig00003218\tchrM\n")
  bam = {k: fx[k] for k in ("subreads_to_ccs", "ccs_bam", "truth_to_ccs", "truth_bed")}
  with pytest.raises(ValueError, match="only to no split"):
    evaluate.run(fx["ckpt"], None, str(tmp_path), split=["eval"], truth_split=str(other), **bam)


def test_smart_windows_and_one_cpu_are_refused(fx, tmp_path):
  r = _cli(fx, tmp_path, ["--split", "eval", "--use_ccs_smart_windows"] + _bam_flags(fx))
  assert r.returncode == 2 and "--use_ccs_smart_windows is not supported" in r.stderr, r.stderr
  r = _cli(fx, tmp_path, ["--split", "eval", "--cpus", "1"] + _bam_flags(fx))
  assert r.returncode == 2 and "cpus to 0 or >=2" in r.stderr, r.stderr
  bam = {k: fx[k] for k in ("subreads_to_ccs", "ccs_bam", "truth_to_ccs", "truth_bed", "truth_split")}
  with pytest.raises(ValueError, match="--use_ccs_smart_windows is not supported"):
    evaluate.run(fx["ckpt"], None, str(tmp_path), split=["eval"], use_ccs_smart_windows=True, **bam)


@pytest.mark.parametrize("cpus", [0, 2])
def test_zmw_selection_counts_the_fixture_summary(fx, cpus):
  """preprocess.select_zmw on the host stream alone gives the ZMW counters of the reference's summary."""
  with gzip.open(fx["digest"], "rt") as f:
    want = json.load(f)["use_ccs_bq"]["0"]["summary"]
  bed, split_of = preprocess.read_truth_bed(fx["truth_bed"]), preprocess.read_truth_split(fx["truth_split"])
  stream = preprocess.BamFeatureStream(fx["subreads_to_ccs"], fx["ccs_bam"], 20, 100, threads=cpus, records=True,
                                       truth_to_ccs=fx["truth_to_ccs"])
  counter = collections.Counter()
  picked = []
  try:
    while (z := stream.next_zmw_records()) is not None:
      p = preprocess.select_zmw(stream, z, 5, counter, bed, split_of)
      if p is not None:
        picked.append((z["name"], p[1]))
        assert set(p[0]) >= {"cigar", "bases", "pos", "ccs0"}
  finally:
    stream.close()
  got = {k: v for k, v in counter.items()}
  assert {k: v for k, v in got.items() if k.startswith("n_zmw")} == {k: v for k, v in want.items() if k.startswith("n_zmw")}
  for k in ("zmw_total_bp", "zmw_trimmed_insertions", "zmw_trimmed_insertions_bp"):
    assert got[k] == want[k], k
  assert len(picked) == want["n_zmw_pass"]
  assert collections.Counter(s for _, s in picked) == {s: want["n_zmw_" + s] for s in ("train", "eval", "test")}


def test_count_zmw_windows_follows_the_summary_rules():
  c = collections.Counter()
  kept = preprocess.count_zmw_windows(c, 100, 4, 512, np.array([0, 1, 2, 0], np.uint8), "eval")
  assert kept.tolist() == [True, True, False, True]
  assert dict(c) == {"example_width_bucket_100": 6, "n_examples_no_ccs_idx": 2, "n_examples_label_overflow": 1,
                     "n_examples_adjusted_label": 1, "n_examples_skip_large_windows_keep": 3, "n_examples_eval": 3,
                     "n_examples": 3}
  preprocess.count_zmw_windows(c, 100, 1, 100, np.array([2], np.uint8), "train")
  assert c["n_examples_train"] == 0 and "n_examples_train" in c and c["n_examples_label_overflow"] == 2


def test_evaluation_input_kernels_have_no_spills_and_no_atomics():
  cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
  lib = engine.library_path()
  if not os.path.exists(cuobjdump) or not os.path.exists(lib):
    pytest.skip("needs cuobjdump and the built library")
  res = subprocess.run([cuobjdump, "-res-usage", lib], capture_output=True, text=True).stdout
  sass = subprocess.run([cuobjdump, "-sass", lib], capture_output=True, text=True).stdout
  for kernel in ("eval_compact_kernel", "eval_emit_kernel", "copy_label_ids_kernel"):
    m = re.search(r"Function [^\n]*%s[^\n]*:\n[^\n]*" % kernel, res)
    assert m, kernel
    assert "STACK:0 " in m.group(0) and "LOCAL:0" in m.group(0), m.group(0)
    body = re.search(r"Function : [^\n]*%s[^\n]*\n(.*?)\n\s*\.{10,}" % kernel, sass, re.S)
    assert body, kernel
    assert not re.search(r"\b(ATOM|RED|ATOMS)\b", body.group(1)), kernel
