"""`read_yield` on the GPU (dcb_read_identity): per-read counts and the JSON object against the restatement on the
repository fixture and on seeded synthetic alignments, reads on the predicted-quality boundary, the N-operation
failure, the cross-check against calibration's counts, and the CLI end to end."""
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
import read_yield_oracle as oracle  # noqa: E402

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


def regions_of(bam, fasta, region):
  refs, _ = bco.read_bam(bam)
  contigs = {k: len(v) for k, v in bco.read_fasta(fasta).items()}
  return [(r.contig, r.start, r.stop) for r in cbc.get_regions(dict(refs), contigs, region)]


def assert_same_reads(got, want):
  assert got["pos"].tolist() == [r["pos"] for r in want]
  assert got["contig"].tolist() == [r["contig"] for r in want]
  for k in oracle.COUNT_KEYS + ("length", "past_reference"):
    assert got[k].tolist() == [r[k] for r in want], k
  np.testing.assert_allclose(got["avg_q"], [r["avg_q"] for r in want], rtol=0, atol=1e-9)


@pytest.mark.parametrize("region", [None, "chr20:0-100000"])
def test_fixture_reads_and_json_match_the_restatement(fx, model, region):
  want_reads = oracle.per_read(fx["bam"], fx["fasta"], regions_of(fx["bam"], fx["fasta"], region), 0)
  got = read_yield.read_identity(fx["bam"], fx["fasta"], region, 0, 2, model)
  assert_same_reads(got, want_reads)
  missing = oracle.contigs_without_reference(fx["bam"], fx["fasta"])
  for q in (0, 20, 30):
    assert read_yield.yield_summary(got, q) == oracle.summary(want_reads, q, missing)
  if region is None:   # 26 primary reads (the supplementary record is dropped), 12 of them past the 200 kb subset
    assert (len(got["pos"]), int(got["past_reference"].sum())) == (26, 12)


def test_fixture_statuses(fx, model):
  with cbc.AlignmentReader(fx["bam"], fx["fasta"], 2) as r:
    b = next(r.batches("chr20", 0, 200000, 0, max_bases=1 << 30))
    ref = r.reference("chr20", 0, 200000)
  res = model.read_identity(b, ref, 0, 200000)
  past = res["status"] == engine.DCB_IDENTITY_PAST_CONTIG
  assert past.sum() == 12
  assert np.isin(res["status"][~past], [engine.DCB_IDENTITY_OK, engine.DCB_IDENTITY_BORDERLINE]).all()
  assert (res["counts"][past] == 0).all() and (res["counts"][~past].sum(axis=1) > 0).all()


# ----------------------------------------------------------------------------------------------- synthetic alignments
def synthetic(rng, ref=None, contig_len=6000, n_reads=300):
  """A contig with lowercase and N bases (or `ref`), and reads with random cigars (every operation but N) copied from it
  with a per-read error rate, qualities around a per-read level, every filtered flag, mapq 0 / 30 / 60, and reads that cross the contig
  end."""
  ref = ref or "".join(rng.choice(list("ACGTacgtN"), contig_len, p=[0.2] * 4 + [0.0495] * 4 + [0.002]))
  contig_len = len(ref)
  recs = []
  for k in range(n_reads):
    ops = []
    if rng.random() < 0.3:
      ops.append((H, int(rng.integers(1, 20))))
    if rng.random() < 0.4:
      ops.append((S, int(rng.integers(1, 15))))
    kinds = [M, EQ, X] if rng.random() < 0.3 else [M, M, M, M, M, M, EQ, X, I, D, P]
    for _ in range(int(rng.integers(1, 25))):
      op = int(rng.choice(kinds))
      ops.append((op, int(rng.integers(1, 200) if op in (M, EQ, X) else rng.integers(1, 4))))
    if rng.random() < 0.4:
      ops.append((S, int(rng.integers(1, 15))))
    if rng.random() < 0.3:
      ops.append((H, int(rng.integers(1, 20))))
    if not any(op in (M, EQ, X) for op, _ in ops):
      ops.append((M, int(rng.integers(1, 10))))
    rlen = sum(n for op, n in ops if op in (M, D, EQ, X))
    pos = int(rng.integers(max(contig_len - rlen, 1), contig_len)) if rng.random() < 0.1 else int(
        rng.integers(0, max(contig_len - rlen, 1)))
    err = float(rng.choice([0.0, 0.0005, 0.001, 0.01, 0.1]))
    seq, r = [], pos
    for op, n in ops:
      for _ in range(n if op in (M, I, S, EQ, X) else 0):
        copy = op in (M, EQ, X) and r < contig_len and rng.random() >= err
        seq.append(ref[r].upper() if copy and ref[r] != "N" else str(rng.choice(list("ACGTN"))))
        r += op in (M, EQ, X)
      r += n if op == D else 0
    flag = int(rng.choice([0, 0, 0, 0, 0, 16, 0x4, 0x100, 0x200, 0x400, 0x800]))
    level = int(rng.choice([10, 18, 25, 35, 50]))
    qual = [int(q) for q in np.clip(level + rng.integers(-5, 6, len(seq)), 0, 93)]
    recs.append(dict(name="r%d" % k, refid=0, pos=pos, mapq=int(rng.choice([60, 60, 30, 0])), flag=flag, cigar=ops,
                     seq="".join(seq), qual=qual))
  return ref, recs


@pytest.fixture(scope="module")
def synth(tmp_path_factory):
  d = tmp_path_factory.mktemp("synthetic")
  ref, dc = synthetic(np.random.default_rng(20261018))
  _, ccs = synthetic(np.random.default_rng(20261019), ref=ref)
  out = dict(ref=ref, dc=str(d / "dc.bam"), ccs=str(d / "ccs.bam"), fasta=str(d / "ref.fa"))
  for name, recs in (("dc", dc), ("ccs", ccs)):
    bco.write_bam(out[name], [("c1", len(ref)), ("c0", 100)], recs)
  bco.write_fasta(out["fasta"], [("c1", ref)], width=70)
  return out


@pytest.mark.parametrize("region,min_mapq", [(None, 0), ("c1:0-3000,c1:1000-4500", 30), ("c1", 60)])
def test_synthetic_alignments_match_the_restatement(synth, model, region, min_mapq):
  want = oracle.per_read(synth["dc"], synth["fasta"], regions_of(synth["dc"], synth["fasta"], region), min_mapq)
  assert any(r["past_reference"] for r in want) == (region != "c1:0-3000,c1:1000-4500")
  for cpus, batch in ((1, 1 << 26), (5, 500)):
    got = read_yield.read_identity(synth["dc"], synth["fasta"], region, min_mapq, cpus, model, batch_bases=batch)
    assert_same_reads(got, want)
    assert got["contigs_without_reference"] == ["c0"]
    for q in (0, 20):
      assert read_yield.yield_summary(got, q) == oracle.summary(want, q, ["c0"])


def test_reads_on_the_quality_boundary_are_decided_as_the_reference_decides(model, tmp_path):
  # four bases of quality q - 1 and five of q + 1 among q's: 6377 bases put round(avg_phred, 5) just below q (by 7e-10),
  # 6378 just on it (by 9e-11)
  rng = np.random.default_rng(7)
  ref = "".join(rng.choice(list("ACGT"), 8000))
  recs = []
  for k, (n, q) in enumerate(((6377, 20), (6378, 20), (6377, 30), (6378, 30))):
    qual = [q - 1] * 4 + [q + 1] * 5 + [q] * (n - 9)
    qual = qual[n // 3:] + qual[:n // 3]
    recs.append(dict(name="b%d" % k, refid=0, pos=100 * k, mapq=60, flag=0, cigar=[(M, n)], seq=ref[100 * k:100 * k + n],
                     qual=qual))
  bam, fasta = str(tmp_path / "b.bam"), str(tmp_path / "b.fa")
  bco.write_bam(bam, [("c1", len(ref))], recs)
  bco.write_fasta(fasta, [("c1", ref)])
  with cbc.AlignmentReader(bam, fasta, 1) as r:
    b = next(r.batches("c1", 0, len(ref), 0, max_bases=1 << 30))
  assert (model.read_identity(b, np.frombuffer(ref.encode(), np.uint8), 0, len(ref))["status"] ==
          engine.DCB_IDENTITY_BORDERLINE).all()
  want = oracle.per_read(bam, fasta, [("c1", 0, len(ref))], 0)
  assert [oracle.passes_quality(r["qual"], 20) for r in want] == [False, True, True, True]
  assert [oracle.passes_quality(r["qual"], 30) for r in want] == [False, False, False, True]
  got = read_yield.read_identity(bam, fasta, None, 0, 1, model)
  assert got["avg_q"].tolist() == [r["avg_q"] for r in want]   # NumPy's own mean where it decides
  for q in (20, 30):
    assert read_yield.yield_summary(got, q) == oracle.summary(want, q)


def test_a_reference_skip_fails_naming_the_read_and_the_engine_stays_usable(synth, model, tmp_path):
  ref = synth["ref"]
  recs = [dict(name="plain", refid=0, pos=10, mapq=60, flag=0, cigar=[(M, 20)], seq=ref[10:30].upper(), qual=[30] * 20),
          dict(name="spliced", refid=0, pos=50, mapq=60, flag=0, cigar=[(M, 5), (N, 40), (M, 5)], seq="ACGTA" * 2,
               qual=[30] * 10)]
  bam = str(tmp_path / "n.bam")
  bco.write_bam(bam, [("c1", len(ref))], recs)
  with pytest.raises(read_yield.ReadYieldError, match=r"read spliced at c1:50: its cigar has an N"):
    read_yield.read_identity(bam, synth["fasta"], None, 0, 1, model)
  with pytest.raises(ValueError, match="spliced"):
    oracle.per_read(bam, synth["fasta"], [("c1", 0, len(ref))], 0)
  want = oracle.per_read(synth["dc"], synth["fasta"], [("c1", 0, len(ref))], 0)
  assert_same_reads(read_yield.read_identity(synth["dc"], synth["fasta"], None, 0, 2, model), want)


def test_counts_agree_with_calibration(model, tmp_path):
  # ACGT-only contig, reads ending 10+ bases before its end, one calibration interval over it, every quality counted:
  # calibration counts matches as matches and mismatches, insertions and soft clips as mismatches
  rng = np.random.default_rng(11)
  contig = 5000
  ref, recs = synthetic(rng, contig_len=contig, n_reads=200)
  ref = ref.upper().replace("N", "A")
  for r in recs:
    r["mapq"] = 60
    rlen = sum(n for op, n in r["cigar"] if op in (M, D, EQ, X))
    r["pos"] = min(r["pos"], contig - rlen - 10)
  recs = [r for r in recs if r["pos"] >= 0]
  bam, fasta = str(tmp_path / "c.bam"), str(tmp_path / "c.fa")
  bco.write_bam(bam, [("c1", contig)], recs)
  bco.write_fasta(fasta, [("c1", ref)])
  cal = cbc.calibration_counts(bam, fasta, "c1", contig, 60, "skip", cpus=2, model=model)
  got = read_yield.read_identity(bam, fasta, "c1", 60, 2, model)
  assert not got["past_reference"].any()
  assert int(got["matches"].sum()) == int(cal[:, 0].sum())
  assert int((got["mismatches"] + got["insertions"] + got["soft_clipped"]).sum()) == int(cal[:, 1].sum())


def test_cli_with_a_baseline_writes_the_restatement_json(synth, tmp_path):
  out = tmp_path / "y.json"
  p = subprocess.run([sys.executable, "-m", "deepconsensus_b200.read_yield", "--bam", synth["dc"], "--ref", synth["fasta"],
                      "--baseline_bam", synth["ccs"], "--region", "c1:0-5000", "--min_quality", "20", "--min_mapq", "30",
                      "--cpus", "3", "--output_json", str(out)], capture_output=True, text=True, cwd=ROOT)
  assert p.returncode == 0, p.stderr
  regions = [("c1", 0, 5000)]
  dc = oracle.summary(oracle.per_read(synth["dc"], synth["fasta"], regions, 30), 20, ["c0"])
  ccs = oracle.summary(oracle.per_read(synth["ccs"], synth["fasta"], regions, 30), 20, ["c0"])
  got = json.loads(out.read_text())
  assert got == json.loads(json.dumps(oracle.with_baseline(dc, ccs)))
  assert got["yield"]["emQ20"] > 0 and got["baseline"]["yield"]["emQ20"] > 0


def test_cli_on_the_fixture(fx, tmp_path):
  out = tmp_path / "y.json"
  p = subprocess.run([sys.executable, "-m", "deepconsensus_b200.read_yield", "--bam", fx["bam"], "--ref", fx["fasta"],
                      "--region", "chr20:0-199999", "--output_json", str(out)], capture_output=True, text=True, cwd=ROOT)
  assert p.returncode == 0, p.stderr
  want = oracle.summary(oracle.per_read(fx["bam"], fx["fasta"], [("chr20", 0, 199999)], 0), 20,
                        oracle.contigs_without_reference(fx["bam"], fx["fasta"]))
  assert json.loads(out.read_text()) == json.loads(json.dumps(want))
