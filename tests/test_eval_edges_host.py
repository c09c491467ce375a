"""The evaluation oracle (oracle/losses.py) on the edge cases of tests/golden/ref_eval_edges.npz, which the reference's own
losses_and_metrics.py produced (scripts/make_eval_edge_golden.py): every L = 3 window, 20k tie-prone L = 4 windows,
4000 random L = 24 windows, the window lengths where the GPU kernels' thread mapping changes, degenerate windows, and
the Keras-style aggregation's branches.  Counts, flags and aggregates must be equal; losses agree to relative 1e-6, as
in test_eval_host.py.

The mutation tests show that the cases bite: each runs a copy of oracle/losses.py with one deliberate mistake (the
copy's source is edited in the test; the oracle itself is untouched) and requires it to disagree with the golden on at
least one window.  The two tie-breaking mistakes change no count at L = 3 or 4 (a tie there is resolved into alignments
with the same counts); the L = 24 windows catch them (about 20 and 130 windows)."""
import inspect
import os
import types

import numpy as np
import pytest

from deepconsensus_b200 import evaluate as evaluate_lib
from oracle import losses as ol

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD_PATH = os.path.join(HERE, "golden", "ref_eval_edges.npz")
EDGE_LENGTHS = (1, 2, 31, 32, 33, 127, 128, 129, 255, 256)
GROUPS = ("L3", "L4", "rand24") + tuple("len%d" % L for L in EDGE_LENGTHS) + ("agg0", "agg1", "agg2")
LOSS_RTOL = LOSS_ATOL = 1e-6


@pytest.fixture(scope="module")
def gold():
  return dict(np.load(GOLD_PATH))


def group(g, name):
  p = name + "_"
  return {k[len(p):]: v for k, v in g.items() if k.startswith(p)}


def settings(gr):
  for s, (dc, reg) in enumerate(gr["loss_settings"]):
    yield s, float(dc), None if np.isnan(reg) else float(reg)


def disagreements(lib, gr):
  """Windows of one group on which the losses module `lib` differs from the golden (counts, flag, or any loss)."""
  ev = lib.evaluate_windows(gr["probs"], gr["labels"], gr["ccs"], 10.0, 0.1)
  bad = (ev["pred_counts"] != gr["pred_counts"]).any(-1) | (ev["ccs_counts"] != gr["ccs_counts"]).any(-1)
  bad |= ev["exact"] != gr["exact"]
  for s, dc, reg in settings(gr):
    loss = lib.alignment_loss(gr["probs"], gr["labels"], dc, reg)
    bad |= ~np.isclose(loss, gr["loss"][s], rtol=LOSS_RTOL, atol=LOSS_ATOL)
  return bad


# ---------------------------------------------------------------------------------------------------- the golden itself
def test_golden_covers_the_edges(gold):
  l3 = group(gold, "L3")
  pairs = {(a.tobytes(), b.tobytes()) for a, b in zip(l3["labels"], l3["probs"].argmax(-1).astype(np.uint8))}
  assert len(pairs) == 5 ** 6
  assert len({(a.tobytes(), c.tobytes()) for a, c in zip(l3["labels"], l3["ccs"])}) == 5 ** 6
  assert group(gold, "L4")["labels"].shape == (625 * 32, 4)
  for L in EDGE_LENGTHS:
    gr = group(gold, "len%d" % L)
    assert gr["labels"].shape[1] == L and gr["probs"].shape[1:] == (L, 5)
    assert gr["loss_settings"].shape == (5, 2)
    assert {5, 6, 255} <= set(np.unique(gr["ccs"]).tolist()) or L <= 2
    assert (gr["labels"] == 0).all(-1).any() and (gr["probs"].argmax(-1) == 0).all(-1).any()
    sums = gr["probs"].sum(-1)
    assert (sums > 3).any() and (sums < 1e-2).any()                    # rows that need renormalising
    assert (gr["probs"] == np.float32(0.2)).all(-1).any()              # uniform rows
    assert (gr["probs"] == 1).any()                                    # one-hot rows
  ties = [(gr["pred_counts"][:, 1] > 0) & (gr["pred_counts"][:, 2] > 0)
          for gr in (group(gold, "len%d" % L) for L in EDGE_LENGTHS)]
  assert sum(int(t.sum()) for t in ties) > 0


# ---------------------------------------------------------------------------------------------------- oracle vs reference
@pytest.mark.parametrize("name", GROUPS)
def test_oracle_matches_reference(gold, name):
  gr = group(gold, name)
  ev = ol.evaluate_windows(gr["probs"], gr["labels"], gr["ccs"], 10.0, 0.1)
  np.testing.assert_array_equal(ev["pred_counts"], gr["pred_counts"])
  np.testing.assert_array_equal(ev["ccs_counts"], gr["ccs_counts"])
  np.testing.assert_array_equal(ev["exact"], gr["exact"])
  for s, dc, reg in settings(gr):
    np.testing.assert_allclose(ol.alignment_loss(gr["probs"], gr["labels"], dc, reg), gr["loss"][s], rtol=LOSS_RTOL,
                               atol=LOSS_ATOL, err_msg="%s del_cost=%g loss_reg=%s" % (name, dc, reg))


@pytest.mark.parametrize("name", ["agg0", "agg1", "agg2"])
def test_aggregation_edges(gold, name):
  """evaluate.aggregate on the reference's per-window values gives its batch identities, yield and accuracy: an all-gap
  batch (identity 1.0), no CCS batch at the threshold (divide_no_nan: 0), a last batch of one window."""
  gr = group(gold, name)
  ev = ol.evaluate_windows(gr["probs"], gr["labels"], gr["ccs"], 10.0, 0.1)
  for per in (dict(gr, loss=gr["loss"][0]), ev):
    agg = evaluate_lib.aggregate(per["loss"], per["exact"], per["pred_counts"], per["ccs_counts"],
                                 int(gr["batch_size"]))
    np.testing.assert_array_equal(np.float32(agg["batch_identity_pred"]), gr["batch_identity_pred"])
    np.testing.assert_array_equal(np.float32(agg["batch_identity_ccs"]), gr["batch_identity_ccs"])
    assert np.float32(agg["yield_over_ccs"]) == gr["yield_over_ccs"]
    assert np.float32(agg["per_example_accuracy"]) == gr["accuracy"]
    assert np.float32(agg["identity"]) == gr["identity"]
    assert agg["n_batches"] == len(gr["batch_identity_pred"])


def test_aggregation_edges_are_present(gold):
  a0, a1 = group(gold, "agg0"), group(gold, "agg1")
  assert a0["batch_identity_pred"][0] == 1.0 and a0["ccs_counts"][:int(a0["batch_size"]), 4].sum() == 0
  assert a0["labels"].shape[0] % int(a0["batch_size"]) == 1
  assert (a1["batch_identity_ccs"] < 0.997).all() and (a1["batch_identity_pred"] >= 0.997).any()
  assert a1["yield_over_ccs"] == 0


# ---------------------------------------------------------------------------------------------------- mutations
DEL_BEFORE_INS = """

def _del_before_ins(t):
  return np.array([0, 2, 1])[t[[0, 2, 1]].argmax(0)]
"""
MUTATIONS = {
    # first maximum over [match, del, ins] instead of [match, ins, del], in every state that can pick either
    "ins_del_tie_order_reversed": [
        ("vm, dm = o_match.max(0), o_match.argmax(0)", "vm, dm = o_match.max(0), _del_before_ins(o_match)"),
        ("vd, dd = o_del.max(0), o_del.argmax(0)", "vd, dd = o_del.max(0), _del_before_ins(o_del)"),
        ("col.argmax(0)", "_del_before_ins(col)"),
        ("  return counts\n", "  return counts\n" + DEL_BEFORE_INS),
    ],
    # `>=` in the match-state maximum: the last of tied candidates wins
    "match_state_ge": [("vm, dm = o_match.max(0), o_match.argmax(0)",
                        "vm, dm = o_match.max(0), 2 - o_match[::-1].argmax(0)")],
    "gap_open_5": [("go, ge = F32(5.0 + 4.0), F32(4.0)", "go, ge = F32(5.0), F32(4.0)")],
    "no_left_shift_of_prediction": [
        ("x = left_shift(np.asarray(y_pred_ids).astype(np.int32))", "x = np.asarray(y_pred_ids).astype(np.int32)"),
        ("x = left_shift(np.asarray(probs).argmax(-1).astype(np.int32))", "x = np.asarray(probs).argmax(-1)"),
    ],
    "ccs_ids_above_4_kept": [("ccs = alignment_metric(labels, decode_ccs_ids(ccs_ids))",
                              "ccs = alignment_metric(labels, ccs_ids)")],
    "no_renormalisation": [("p = (p / tot[..., None]).astype(F32)", "p = p")],
}


def _variant(edits):
  """A fresh module made from oracle/losses.py's source with `edits` applied (each must match exactly once)."""
  src = inspect.getsource(ol)
  for old, new in edits:
    assert src.count(old) == 1, old
    src = src.replace(old, new)
  mod = types.ModuleType("losses_variant")
  exec(compile(src, ol.__file__, "exec"), mod.__dict__)
  return mod


def test_unmutated_copy_agrees(gold):
  lib = _variant([])
  for name in ("L3", "len256"):
    assert not disagreements(lib, group(gold, name)).any(), name


@pytest.mark.parametrize("mistake", sorted(MUTATIONS))
def test_mutation_is_caught(gold, mistake):
  lib = _variant(MUTATIONS[mistake])
  found = {name: int(disagreements(lib, group(gold, name)).sum()) for name in GROUPS}
  print("%s: windows that disagree per group %s" % (mistake, {k: v for k, v in found.items() if v}))
  assert sum(found.values()) >= 1
  assert ol.alignment_loss is not lib.alignment_loss
