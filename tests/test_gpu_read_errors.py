"""`read_yield --error_profile` on the GPU (dcb_read_errors): per-read rows against the restatement on the repository
fixture, the hand-built alignments and a seeded homopolymer-rich contig for every batch budget and `--cpus`, the
cross-checks against read_identity's counts, the refusal of a slice that is too short, and the CLI end to end."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from deepconsensus_b200 import calculate_baseq_calibration as cbc
from deepconsensus_b200 import engine
from deepconsensus_b200 import read_yield

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import baseq_calibration_oracle as bco  # noqa: E402
import read_errors_oracle as oracle  # noqa: E402
import read_errors_synth as synth  # noqa: E402
import read_yield_oracle as ryo  # noqa: E402
from test_gpu_read_yield import assert_same_reads, regions_of, synthetic  # noqa: E402
from test_read_errors_host import HAND, REF  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M, I, D, N, S, H, P, EQ, X = range(9)


@pytest.fixture(scope="module")
def model():
  m = cbc._default_model()
  yield m
  m.close()


@pytest.fixture(scope="module")
def fx(golden_dir, tmp_path_factory):
  bam, fasta, _ = bco.unpack_fixture(golden_dir, tmp_path_factory.mktemp("fixture"))
  return dict(bam=bam, fasta=fasta)


def assert_same_rows(got, want):
  assert_same_reads(got, want)
  assert got["errors"].shape == (len(want), engine.ERRORS_COLS)
  for k, r in enumerate(want):
    assert got["errors"][k].tolist() == r["errors"], (k, r["pos"])


def assert_cross_checks(got, want):
  counted = ~got["past_reference"]
  for k in np.flatnonzero(counted):
    counts = {c: int(got[c][k]) for c in ryo.COUNT_KEYS}
    ops = want[k]["ops"]
    assert oracle.cross_checks(got["errors"][k].tolist(), counts, ops.count(I), ops.count(D)), k
  assert not got["errors"][~counted].any()


@pytest.mark.parametrize("region", [None, "chr20:0-100000"])
def test_fixture_rows_match_the_restatement(fx, model, region):
  want = oracle.per_read(fx["bam"], fx["fasta"], regions_of(fx["bam"], fx["fasta"], region), 0)
  got = read_yield.read_identity(fx["bam"], fx["fasta"], region, 0, 2, model, error_profile=True)
  assert_same_rows(got, want)
  assert_cross_checks(got, want)
  plain = read_yield.read_identity(fx["bam"], fx["fasta"], region, 0, 2, model)
  assert "errors" not in plain and set(got) == set(plain) | {"errors"}
  for k in plain:
    assert np.array_equal(got[k], plain[k]) if k != "contigs_without_reference" else got[k] == plain[k]
  for q in (0, 20):
    assert read_yield.error_summary(got, q) == oracle.summary(want, q)
  assert sum(got["errors"][:, engine.ERRORS_RUNS:engine.ERRORS_RUNS + engine.ERRORS_BINS].sum(axis=0)) > 0


def test_hand_built_alignments_match_the_restatement(model, tmp_path):
  recs = [dict(r, name="h%d" % k) for k, (r, _, _) in enumerate(HAND)]
  bam, fasta = str(tmp_path / "h.bam"), str(tmp_path / "h.fa")
  bco.write_bam(bam, [("c1", len(REF))], recs)
  bco.write_fasta(fasta, [("c1", REF)])
  want = oracle.per_read(bam, fasta, [("c1", 0, len(REF))], 0)
  for batch in (1, 1 << 26):
    got = read_yield.read_identity(bam, fasta, None, 0, 1, model, error_profile=True, batch_bases=batch)
    assert_same_rows(got, want)
    assert_cross_checks(got, want)


@pytest.fixture(scope="module")
def hp_synth(tmp_path_factory):
  d = tmp_path_factory.mktemp("hp_synthetic")
  rng = np.random.default_rng(20261018)
  ref = synth.hp_rich_contig(rng)
  _, dc = synthetic(rng, ref=ref, n_reads=400)
  dc += synth.planted_reads(rng, ref)
  _, ccs = synthetic(np.random.default_rng(20261019), ref=ref, n_reads=300)
  out = dict(ref=ref, dc=str(d / "dc.bam"), ccs=str(d / "ccs.bam"), fasta=str(d / "ref.fa"))
  for name, recs in (("dc", dc), ("ccs", ccs)):
    bco.write_bam(out[name], [("c1", len(ref)), ("c0", 100)], recs)
  bco.write_fasta(out["fasta"], [("c1", ref)], width=70)
  return out


@pytest.mark.parametrize("region,min_mapq", [(None, 0), ("c1:3000-16000,c1:15000-25000", 30)])
def test_homopolymer_rich_rows_match_the_restatement_for_any_batch(hp_synth, model, region, min_mapq):
  want = oracle.per_read(hp_synth["dc"], hp_synth["fasta"], regions_of(hp_synth["dc"], hp_synth["fasta"], region),
                         min_mapq)
  # the long runs are covered whole by some reads and cut by others
  long_bins = sum(r["errors"][5 * oracle.BINS + 20] for r in want)
  assert long_bins > 0 and sum(any(r["errors"]) for r in want) > 100
  summaries = []
  for cpus, batch in ((1, 1), (5, 500), (1, 20000), (5, 1 << 26)):
    got = read_yield.read_identity(hp_synth["dc"], hp_synth["fasta"], region, min_mapq, cpus, model, batch_bases=batch,
                                   error_profile=True)
    assert_same_rows(got, want)
    assert_cross_checks(got, want)
    summaries.append(read_yield.error_summary(got, 20))
  assert all(s == oracle.summary(want, 20) for s in summaries)


def test_a_slice_that_misses_a_neighbour_is_refused(model, tmp_path):
  rng = np.random.default_rng(3)
  ref = list(rng.choice(list("ACGT"), 400))
  ref[98] = "C" if ref[99] != "C" else "G"     # [99, 151) holds whole runs at both ends
  ref[151] = "C" if ref[150] != "C" else "G"
  ref = "".join(ref)
  recs = [dict(name="a", refid=0, pos=100, mapq=60, flag=0, cigar=[(I, 1), (M, 50)], seq=ref[99] + ref[100:150],
               qual=[30] * 51)]
  bam, fasta = str(tmp_path / "s.bam"), str(tmp_path / "s.fa")
  bco.write_bam(bam, [("c1", len(ref))], recs)
  bco.write_fasta(fasta, [("c1", ref)])
  with cbc.AlignmentReader(bam, fasta, 1) as r:
    b = next(r.batches("c1", 0, len(ref), 0))
    bases = r.reference("c1", 0, len(ref))
  ok = model.read_errors(b, bases[99:151], 99, len(ref))["errors"]
  want = oracle.per_read(bam, fasta, [("c1", 0, len(ref))], 0)[0]["errors"]
  assert ok[0].tolist() == want and sum(want[engine.ERRORS_INS_EVENTS:engine.ERRORS_INS_BASES]) == 1
  for lo, hi in ((100, 151), (99, 150)):   # pos - 1, then endpos, missing
    with pytest.raises(RuntimeError, match="dcb_read_errors: read 0"):
      model.read_errors(b, bases[lo:hi], lo, len(ref))
  assert np.array_equal(model.read_errors(b, bases, 0, len(ref))["errors"], ok)   # the engine stays usable


def test_cli_with_a_baseline_writes_the_restatement_json(hp_synth, tmp_path):
  regions = [("c1", 0, 28000)]
  want = ryo.with_baseline(*[dict(ryo.summary(reads, 20, ["c0"]), errors=oracle.summary(reads, 20)) for reads in (
      oracle.per_read(hp_synth[k], hp_synth["fasta"], regions, 30) for k in ("dc", "ccs"))])
  args = [sys.executable, "-m", "deepconsensus_b200.read_yield", "--bam", hp_synth["dc"], "--ref", hp_synth["fasta"],
          "--baseline_bam", hp_synth["ccs"], "--region", "c1:0-28000", "--min_quality", "20", "--min_mapq", "30",
          "--cpus", "3"]
  out = tmp_path / "e.json"
  p = subprocess.run(args + ["--error_profile", "--output_json", str(out)], capture_output=True, text=True, cwd=ROOT)
  assert p.returncode == 0, p.stderr
  got = json.loads(out.read_text())
  assert got == json.loads(json.dumps(want))
  assert sum(got["errors"]["runs"]) > 0 and sum(got["baseline"]["errors"]["runs"]) > 0
  # without the flag the JSON is read_yield's: the restatement's, and byte for byte the profile's minus `errors`
  plain = tmp_path / "y.json"
  p = subprocess.run(args + ["--output_json", str(plain)], capture_output=True, text=True, cwd=ROOT)
  assert p.returncode == 0, p.stderr
  for obj in (want, want["baseline"], got, got["baseline"]):
    del obj["errors"]
  assert json.loads(plain.read_text()) == json.loads(json.dumps(want))
  assert plain.read_text() == json.dumps(got, indent=1) + "\n"
