"""Host-side mirrors vs (a) the reference's own test goldens and (b) fixtures produced by executing
the reference's pure functions (scripts/make_golden.py -> tests/golden/ref_*.json)."""
import json
import os

import numpy as np
import pytest

from deepconsensus_b200 import calibration, constants, params as params_lib, stitch_utils, utils, weights


def _load(golden_dir, name):
  with open(os.path.join(golden_dir, name)) as f:
    return json.load(f)


# ---- utils (reference: utils/utils_test.py:38-110)
def test_vocab_and_constants(golden_dir):
  g = _load(golden_dir, "ref_utils.json")["constants"]
  assert constants.SEQ_VOCAB == g["SEQ_VOCAB"] == " ATCG"
  assert constants.GAP == g["GAP"] and constants.EMPTY_QUAL == g["EMPTY_QUAL"]
  assert list(constants.DC_FEATURES) == g["DC_FEATURES"]
  assert constants.REFERENCE_VERSION == g["version"]


@pytest.mark.parametrize("scores,expected", [([], ""), ([0, 10, 20, 30, 40], "!+5?I")])
def test_quality_scores_to_string_reference_goldens(scores, expected):   # utils_test.py:60-64
  assert utils.quality_scores_to_string(np.array(scores, dtype=int)) == expected


@pytest.mark.parametrize("string,expected", [("", []), ("!", [0]), ("I", [40]), ("5", [20]), ("!+5?I", [0, 10, 20, 30, 40])])
def test_quality_string_to_array_reference_goldens(string, expected):    # utils_test.py:69-77
  assert utils.quality_string_to_array(string) == expected


@pytest.mark.parametrize("q,expected", [(np.array([1]), 0.9999), ([1, 2, 3], 1.9235), (np.array([1, 2, 3]), 1.9235),
                                        (np.array([1, -1, 3]), 1.8858), (np.array([-1, -1, -1]), 0.0)])
def test_avg_phred_reference_goldens(q, expected):                        # utils_test.py:82-110
  assert abs(utils.avg_phred(q) - expected) < 1e-3


def test_utils_against_executed_reference(golden_dir):
  g = _load(golden_dir, "ref_utils.json")
  for case in g["avg_phred"]:
    q = np.array(case["q"])
    assert utils.avg_phred(q) == pytest.approx(case["avg_phred"], rel=1e-12, abs=1e-12)
    assert utils.quality_scores_to_string(np.maximum(q, 0)) == case["string"]
    assert utils.quality_string_to_array(case["string"]) == np.maximum(q, 0).tolist()
  for case in g["encoded"]:
    assert utils.encoded_sequence_to_string(np.array(case["ids"])) == case["string"]


# ---- calibration (reference: calibration_lib_test.py:38-125)
@pytest.mark.parametrize("s,exp", [("skip", (False, 0.0, 1.0, 0.0)), ("10,1.0,0.2222", (True, 10.0, 1.0, 0.2222)),
                                   ("-10,1.0,0.2222", (True, -10.0, 1.0, 0.2222)), ("-10,-1.0,-0.2222", (True, -10.0, -1.0, -0.2222))])
def test_parse_calibration_string(s, exp):
  cv = calibration.parse_calibration_string(s)
  assert (cv.enabled, cv.threshold, cv.w, cv.b) == exp


@pytest.mark.parametrize("s", ["ABCD", "A,BC,D", "10,1.0", "10,AB,1.0", "10,0.1.1,1.0"])
def test_parse_calibration_string_errors(s):
  with pytest.raises(Exception):
    calibration.parse_calibration_string(s)


@pytest.mark.parametrize("vals,s,exp", [([0, 1, 2, 3, 4], "0,0,1", [1, 1, 1, 1, 1]), ([0, 1, 2, 3, 4], "0,1,1", [1, 2, 3, 4, 5]),
                                        ([0, 1, 2, 3, 4, 5], "3,1,1", [0, 1, 2, 3, 5, 6])])
def test_calibrate_reference_goldens(vals, s, exp):                        # calibration_lib_test.py:106-125
  out = calibration.calibrate_quality_scores(np.array(vals), calibration.parse_calibration_string(s))
  assert np.array_equal(out, np.array(exp))


def test_calibration_against_executed_reference(golden_dir):
  for case in _load(golden_dir, "ref_calibration.json"):
    cv = calibration.parse_calibration_string(case["string"])
    assert (cv.enabled, cv.threshold, cv.w, cv.b) == (case["enabled"], case["threshold"], case["w"], case["b"])
    q = np.array(case["q"], dtype=np.float32)
    out = calibration.calibrate_quality_scores(q, cv) if cv.enabled else q
    assert str(np.asarray(out).dtype) == case["out_dtype"]        # float32 when threshold == 0, float64 otherwise
    assert np.array_equal(np.asarray(out, np.float64), np.array(case["out"]))


# ---- stitch (reference: stitch_utils_test.py:67-218 behaviours, values from the executed reference)
def test_stitch_against_executed_reference(golden_dir):
  g = _load(golden_dir, "ref_stitch.json")
  assert len(g["cases"]) >= 100
  outcomes = set()
  for case in g["cases"]:
    preds = []
    for w in case["windows"]:
      if w["dropped"]:
        continue
      o = stitch_utils.DCModelOutput(molecule_name=case["name"], window_pos=w["window_pos"], ec=1.0, np_num_passes=3, rq=0.99, rg="rg")
      o.sequence, o.quality_string = w["sequence"], w["quality_string"]
      preds.append(o)
    cnt = stitch_utils.OutcomeCounter()
    fq = stitch_utils.stitch_to_fastq(case["name"], preds, case["max_length"], case["min_quality"], case["min_length"], cnt)
    assert fq == case["fastq"]
    assert cnt.__dict__ == case["counter"]
    outcomes.add(tuple(sorted(k for k, v in case["counter"].items() if v)))
  assert len(outcomes) >= 4     # success + several distinct filter outcomes are exercised


def test_get_full_sequence_fill_n(golden_dir):
  g = _load(golden_dir, "ref_stitch.json")["fill_n"]
  o1 = stitch_utils.DCModelOutput("m", 0, 0, 0, 0, "", "ACGT ", "!!!!!")
  o3 = stitch_utils.DCModelOutput("m", 10, 0, 0, 0, "", "TTTTT", "IIIII")
  assert list(stitch_utils.get_full_sequence([o1, o3], 5, fill_n=True)) == g["result"]
  assert stitch_utils.get_full_sequence([o1, o3], 5) == (None, "")


def test_remove_gaps_and_format():
  assert stitch_utils.remove_gaps("A C G", "12345") == ("ACG", "135")
  assert stitch_utils.format_as_fastq("n", "ACGT", "IIII") == "@n\nACGT\n+\nIIII\n"
  assert stitch_utils.is_quality_above_threshold("+" * 10, 10)       # all-Q10 read passes min_quality 10 (stitch_utils.py:103-108)


# ---- params / row layout (reference: data_providers_test.py:323-365, model_utils_test.py:65-170)
@pytest.mark.parametrize("P,bq,rows", [(20, False, 85), (20, True, 86), (25, False, 105), (25, True, 106)])
def test_get_total_rows(P, bq, rows):
  assert params_lib.get_total_rows(P, bq) == rows


def test_get_indices():
  assert params_lib.get_indices(20, False)[4:] == ((80, 81), (0, 0), (81, 85))
  assert params_lib.get_indices(20, True)[4:] == ((80, 81), (81, 82), (82, 86))
  assert params_lib.get_indices(20, False)[:4] == ((0, 20), (20, 40), (40, 60), (60, 80))


def test_params_json_fixture_roundtrip(tmp_path):
  # the keys the reference fixture testdata/model/params.json carries for the path
  fixture = dict(model_name="transformer_learn_values", max_passes=20, max_length=100, use_ccs_bq=False,
                 per_base_hidden_size=8, pw_hidden_size=8, ip_hidden_size=8, strand_hidden_size=2, sn_hidden_size=8,
                 ccs_bq_hidden_size=8, condense_transformer_input=True, transformer_input_size=280, hidden_size=280,
                 num_heads=2, num_hidden_layers=6, filter_size=2048, attn_win_size=12, rezero=True,
                 add_pos_encoding=True, transformer_model_size="base", dc_calibration="0,1.197654,-0.99781")
  (tmp_path / "params.json").write_text(__import__("json").dumps(fixture))
  p = params_lib.read_params_from_json(str(tmp_path / "checkpoint-1"))
  assert p.total_rows == 85                                             # model_utils_test.py:163-167
  params_lib.modify_params(p)
  assert p.hidden_size == 280 and p.num_heads == 2 and p.filter_size == 2048
  assert params_lib.embedded_width(p) == 560
  assert weights.count_params(p) == 8943775                           


def test_config_derived_hidden_sizes():
  p = params_lib.get_config("transformer_learn_values+test")
  params_lib.modify_params(p, max_length=100)
  assert (p.hidden_size, p.total_rows, p.rezero, p.attn_win_size) == (280, 85, True, 12)
  p = params_lib.get_config("transformer+test")
  params_lib.modify_params(p, max_length=100)
  assert p.hidden_size == 86                                            # 85 rows padded to even (model_utils.py:335-336)
  assert params_lib.embedded_width(params_lib.synthetic_params(20, 100, use_ccs_bq=True)) == 568
  assert params_lib.embedded_width(params_lib.synthetic_params(32, 200)) == 872


# ---- skipped windows (reference: quick_inference.py:567-594 and the skip loop :657-676, executed by
# scripts/make_skipped_golden.py from the reference's own source text)
def test_skipped_windows_against_executed_reference(golden_dir):
  import dataclasses
  from deepconsensus_b200 import calibration, inference
  g = _load(golden_dir, "ref_skipped.json")
  assert len(g["cases"]) >= 40
  n_skipped = 0
  for case in g["cases"]:
    o = case["options"]
    opts = inference.InferenceOptions(
        max_length=case["L"], example_height=4 * o["max_passes"] + 5 + int(o["use_ccs_bq"]), max_passes=o["max_passes"],
        min_quality=0, min_length=0, batch_size=8, use_ccs_bq=o["use_ccs_bq"], cpus=0,
        skip_windows_above=o["skip_windows_above"], use_saved_model=False, max_base_quality=o["max_base_quality"],
        dc_calibration_values=calibration.parse_calibration_string("skip"),
        ccs_calibration_values=calibration.parse_calibration_string(o["ccs_calibration"]))
    P, L = o["max_passes"], case["L"]
    R = 4 * P + 5 + int(o["use_ccs_bq"])
    zmws, cur = [], None
    for w in case["windows"]:
      rows = np.zeros((R, L, 1), np.float32)
      rows[4 * P, :, 0] = w["ccs_row"]
      fd = dict(subreads=rows, ccs_base_quality_scores=np.asarray(w["ccs_q"], dtype=w["ccs_q_dtype"]),
                window_pos=w["window_pos"], name=w["zmw"], ec=w["ec"], np_num_passes=w["np_num_passes"], rq=w["rq"],
                rg=w["rg"], overflow=w["overflow"])
      if cur is None or cur[-1]["name"] != w["zmw"]:
        cur = []
        zmws.append(cur)
      cur.append(fd)
    for_model, skipped = inference.split_skipped_windows(zmws, opts)
    assert [[w["name"], w["window_pos"]] for w in for_model] == case["for_model"]
    assert [dataclasses.asdict(x) for x in skipped] == [dict(s) for s in case["skipped"]]
    n_skipped += len(skipped)
  assert n_skipped >= 50
