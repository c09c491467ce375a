"""`calculate_baseq_calibration` on the GPU (dcb_calib_count): the reference's CSV byte for byte on its fixture, its
contig-end failure, and the NumPy restatement on seeded synthetic alignments."""
import os
import subprocess
import sys

import numpy as np
import pytest

from deepconsensus_b200 import calculate_baseq_calibration as cbc
from deepconsensus_b200 import calibration

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import baseq_calibration_oracle as oracle  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def fx(golden_dir, tmp_path_factory):
  bam, fasta, gold = oracle.unpack_fixture(golden_dir, tmp_path_factory.mktemp("fixture"))
  return dict(bam=bam, fasta=fasta, gold=gold)


@pytest.fixture(scope="module")
def model():
  m = cbc._default_model()
  yield m
  m.close()


def test_every_golden_configuration_gives_the_reference_csv(fx, model):
  for c in fx["gold"]["configs"]:
    counts = cbc.calibration_counts(fx["bam"], fx["fasta"], c["region"], c["interval_length"], c["min_mapq"],
                                    c["dc_calibration"], cpus=2, model=model)
    assert cbc.csv_text(counts) == c["csv"], (c["region"], c["interval_length"], c["min_mapq"], c["dc_calibration"])


def test_cli_writes_the_reference_csv(fx, tmp_path):
  c = next(c for c in fx["gold"]["configs"] if c["dc_calibration"] == "10,0.9,2.6")
  out = tmp_path / "bq.csv"
  p = subprocess.run([sys.executable, "-m", "deepconsensus_b200.calculate_baseq_calibration", "--bam", fx["bam"], "--ref",
                      fx["fasta"], "--output_csv", str(out), "--region", c["region"], "--interval_length",
                      str(c["interval_length"]), "--min_mapq", str(c["min_mapq"]), "--dc_calibration", c["dc_calibration"],
                      "--cpus", "3"], capture_output=True, text=True, cwd=ROOT)
  assert p.returncode == 0, p.stderr
  assert out.read_bytes() == c["csv"].encode()


def test_the_whole_contig_default_fails_at_the_contig_end_and_the_engine_stays_usable(fx, model):
  assert fx["gold"]["whole_contig_default"]["exception"] == "IndexError"   # the reference fails too
  names = {r["name"] for r in oracle.read_bam(fx["bam"])[1]}
  with pytest.raises(cbc.CalibrationError, match=r"at chr20:200000: a counted base lies past the end") as e:
    cbc.calibration_counts(fx["bam"], fx["fasta"], None, 1000, 60, "skip", cpus=2, model=model)
  assert str(e.value).split(" ")[1] in names
  c = fx["gold"]["configs"][0]
  counts = cbc.calibration_counts(fx["bam"], fx["fasta"], c["region"], c["interval_length"], c["min_mapq"],
                                  c["dc_calibration"], model=model)
  assert cbc.csv_text(counts) == c["csv"]


def test_an_out_of_range_calibrated_quality_fails_naming_the_read(fx, model):
  names = {r["name"] for r in oracle.read_bam(fx["bam"])[1]}
  with pytest.raises(cbc.CalibrationError, match=r"at chr20:\d+: its quality falls outside the 100 quality bins") as e:
    cbc.calibration_counts(fx["bam"], fx["fasta"], "chr20:1324-2000", 1000, 60, "0,1,100", model=model)
  assert str(e.value).split(" ")[1] in names
  with pytest.raises(IndexError):   # the restatement (and the reference) fail there too
    oracle.count(fx["bam"], fx["fasta"], [("chr20", 1324, 2000)], 1000, 60, calibration.parse_calibration_string("0,1,100"))


def test_batch_sizes_and_decode_threads_do_not_change_the_counts(fx, model):
  want = cbc.calibration_counts(fx["bam"], fx["fasta"], "chr20:0-199999", 500, 0, "10,0.9,2.6", cpus=1, model=model)
  for batch_bases, cpus in ((1, 1), (20000, 4), (300000, 16), (1 << 30, 7)):
    got = cbc.calibration_counts(fx["bam"], fx["fasta"], "chr20:0-199999", 500, 0, "10,0.9,2.6", cpus=cpus, model=model,
                                 batch_bases=batch_bases)
    np.testing.assert_array_equal(got, want)


# ----------------------------------------------------------------------------------------------- synthetic alignments
M, I, D, N, S, H, P, EQ, X = range(9)


def synthetic(rng, contig_len=6000, n_reads=220):
  """A contig with lowercase and N bases, and reads with random cigars (H / P / N / = / X among them), qualities
  0-99, some starting or ending exactly on interval starts (multiples of 700 and 1000), soft clips and insertions
  there, reads that consume no reference, and reads the filters drop."""
  ref = "".join(rng.choice(list("ACGTACGTACGTacgtN"), contig_len))
  recs = []
  for k in range(n_reads):
    ops = []
    if rng.random() < 0.3:
      ops.append((H, int(rng.integers(1, 20))))
    if rng.random() < 0.4:
      ops.append((S, int(rng.integers(1, 15))))
    if rng.random() < 0.05:
      ops.append((I, int(rng.integers(1, 6))))                  # no reference consumed at all
    else:
      for _ in range(int(rng.integers(1, 25))):
        op = int(rng.choice([M, M, EQ, EQ, X, I, D, N, P]))
        ops.append((op, int(rng.integers(1, 40))))
    if rng.random() < 0.4:
      ops.append((S, int(rng.integers(1, 15))))
    if rng.random() < 0.3:
      ops.append((H, int(rng.integers(1, 20))))
    if not any(op in (M, I, S, EQ, X) for op, _ in ops):
      ops.append((M, int(rng.integers(1, 10))))
    rlen = sum(n for op, n in ops if op in (M, D, N, EQ, X))
    edge = int(rng.choice([700, 1000])) * int(rng.integers(1, 5))
    mode = rng.random()
    if mode < 0.25:
      pos = edge                                                # starts on an interval start
    elif mode < 0.5:
      pos = max(edge - max(rlen, 1), 0)                         # ends on one (a trailing clip sits at endpos)
    else:
      pos = int(rng.integers(0, contig_len - rlen - 10))
    pos = min(pos, contig_len - rlen - 10)
    nq = sum(n for op, n in ops if op in (M, I, S, EQ, X))
    flag = int(rng.choice([0, 0, 0, 0, 16, 0x800, 0x100, 0x400]))
    recs.append(dict(name="r%d" % k, refid=0, pos=pos, mapq=int(rng.choice([60, 60, 60, 30, 0])), flag=flag, cigar=ops,
                     seq="".join(rng.choice(list("ACGTACGTN"), nq)), qual=[int(q) for q in rng.integers(0, 100, nq)]))
  return ref, recs


@pytest.fixture(scope="module")
def synth(tmp_path_factory):
  d = tmp_path_factory.mktemp("synthetic")
  rng = np.random.default_rng(20261018)
  ref, recs = synthetic(rng)
  bam, fasta = str(d / "reads.bam"), str(d / "ref.fa")
  oracle.write_bam(bam, [("c1", len(ref)), ("c0", 100)], recs)
  oracle.write_fasta(fasta, [("c1", ref)], width=70)
  return dict(bam=bam, fasta=fasta, ref=ref)


@pytest.mark.parametrize("region,interval_length,min_mapq,cal", [
    ("c1:0-5900", 1000, 60, "skip"),
    ("c1:0-5900", 700, 0, "0,1,-3"),
    ("c1:100-2100,c1:700-3500", 7, 30, "10,0.9,2.6"),
    ("c1:1400-2800", 1, 0, "skip"),
    ("c1:0-4200,c1:0-4200", 100, 60, "0,1,-3"),
])
def test_synthetic_alignments_match_the_restatement(synth, model, region, interval_length, min_mapq, cal):
  regions = [(r.contig, r.start, r.stop) for r in cbc.get_regions({"c1": 1, "c0": 1}, {"c1": len(synth["ref"])}, region)]
  want = oracle.count(synth["bam"], synth["fasta"], regions, interval_length, min_mapq,
                      calibration.parse_calibration_string(cal))
  assert want.sum() > 0
  for cpus, batch in ((1, 1 << 26), (5, 500)):
    got = cbc.calibration_counts(synth["bam"], synth["fasta"], region, interval_length, min_mapq, cal, cpus=cpus,
                                 model=model, batch_bases=batch)
    np.testing.assert_array_equal(got, want)
