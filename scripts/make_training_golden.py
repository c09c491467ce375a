"""Digest of the reference's own training-mode preprocessing output for its BAM fixtures.

deepconsensus/testdata/human_1m/tf_examples{,_bq}/{train,eval,test}/*.tfrecord.gz hold the labelled examples the
reference's `deepconsensus preprocess` (v1.2.0, ins_trim=5, without / with --use_ccs_bq) wrote from
testdata/human_1m/{subreads_to_ccs,ccs,truth_to_ccs}.bam, truth.bed and truth_split.tsv.  This script reduces every
example to (split, name, window_pos, num_passes, row shape, sha1 of the float32 rows, of the CCS base qualities and of
the float32 label) and stores both summary.training.json files next to them ->
tests/golden/human_1m/training_digest.json.gz; byte copies of the truth inputs sit next to it.  The 4 MB train files
are not copied.  Run where the reference exists; the output is committed.
"""
import gzip
import hashlib
import importlib.util
import json
import os

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference/deepconsensus/testdata/human_1m/"
spec = importlib.util.spec_from_file_location("mg", os.path.join(REPO, "scripts", "make_golden.py"))
mg = importlib.util.module_from_spec(spec)
spec.loader.exec_module(mg)


def sha(a, dt):
  return hashlib.sha1(np.ascontiguousarray(a, dt).tobytes()).hexdigest()


def digest(config_dir):
  out = []
  for split in ("train", "eval", "test"):
    for ex in mg.read_tfrecords(os.path.join(REF, config_dir, split, split + ".tfrecord.gz")):
      shape = [int(s) for s in ex["subreads/shape"]]
      rows = np.frombuffer(ex["subreads/encoded"][0], "<f4").reshape(shape)[..., 0]
      label = np.frombuffer(ex["label/encoded"][0], "<f4")
      assert [int(s) for s in ex["label/shape"]] == [shape[1]]
      out.append(dict(split=split, name=ex["name"][0].decode(), window_pos=int(ex["window_pos"][0]),
                      num_passes=int(ex["subreads/num_passes"][0]), shape=shape[:2], rows_sha1=sha(rows, "<f4"),
                      bq_sha1=sha(np.asarray(ex["ccs_base_quality_scores"], np.int64), "<i8"),
                      label_sha1=sha(label, "<f4")))
  with open(os.path.join(REF, config_dir, "summary", "summary.training.json")) as f:
    summary = json.load(f)
  return dict(summary=summary, examples=out)


def main():
  gold = dict(source="deepconsensus/testdata/human_1m/tf_examples{,_bq}", use_ccs_bq={"0": digest("tf_examples"),
                                                                                      "1": digest("tf_examples_bq")})
  path = os.path.join(REPO, "tests", "golden", "human_1m", "training_digest.json.gz")
  with gzip.open(path, "wt") as f:
    json.dump(gold, f)
  print({k: len(v["examples"]) for k, v in gold["use_ccs_bq"].items()}, "examples ->", path)


if __name__ == "__main__":
  main()
