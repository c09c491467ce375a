"""Generates tests/golden/ref_eval_edges.npz by EXECUTING the reference's own losses_and_metrics.py
(deepconsensus/models/losses_and_metrics.py, unmodified, from the checkout at REF) on the NumPy stand-in for TensorFlow in
scripts/tf_shim.py (install() + install_losses_ops()), on the windows where the evaluation kernels can go wrong: tied
alignments, the lengths where their thread mapping changes, and degenerate inputs.

Groups (checked by tests/test_eval_edges_host.py against oracle/losses.py, and on the GPU by
tests/test_gpu_eval_edges.py).  Every group G stores
  G_labels uint8 [B, L], G_probs float32 [B, L, 5], G_ccs uint8 [B, L]     the windows
  G_pred_counts, G_ccs_counts int32 [B, 5]                                AlignmentMetric.alignment of the argmax
                                                                          prediction and of one_hot(ccs), columns
                                                                          num_matches, num_insertions, num_deletions,
                                                                          num_correct_matches, alignment_length
  G_exact uint8 [B]                                                       PerExampleAccuracy, one window at a time
  G_loss_settings float64 [S, 2], G_loss float32 [S, B]                   AlignmentLoss(del_cost, loss_reg).eval with
                                                                          width=None; loss_reg NaN stands for None
                                                                          (the hard min)
  L3      every label in 5^3 against every prediction in 5^3 (one-hot probabilities), 15,625 windows; the CCS of the
          window with prediction b is sequence PERM[b], so every CCS triple also meets every label.  Losses at
          (10, 0.1) and (10, None).
  L4      all 625 labels, each against 32 predictions drawn (seeded) from shifts by one, single insertions and
          deletions, repeated bases, two-base periods, interleaved gaps and random sequences; one-hot probabilities.
          Losses at (10, 0.1) and (10, None).
  rand24  4000 windows of L = 24 whose label, prediction (one-hot) and CCS are independent random ids 0..4.  At L = 3
          and 4 no tie changes the counts, whichever way it is broken; here about 1 window in 200 (prediction or CCS) has a
          tie between the insertion and deletion states, and about 1 in 30 one among the match state's predecessors,
          whose resolution does.  Losses at (10, 0.1) and (10, None).
  len{L}  L in 1, 2, 31, 32, 33, 127, 128, 129, 255, 256: structured pairs (identical, shifted by one, ATAT.. against
          TATA.., long deletion and insertion runs, all gaps on either side or both, interleaved gaps, one base at
          L - 1, one repeated base, 5 % and 30 % mutations) under sharp and flat softmaxes, one-hot rows, uniform rows,
          rows with a two-way tie at the maximum, and rows scaled by 3.7 or 1e-3; CCS rows carry ids 5, 6 and 255.
          Losses at (10, 0.1), (10, None), (1e9, None), (10, 0.01), (2, 1.0).
  agg{0,1,2}   Keras-style aggregation over batches of agg{i}_batch_size in order, the last batch kept
          (get_batch_identity_ccs_pred, tf.keras.metrics.Mean of the batch identities, YieldOverCCSMetric,
          PerExampleAccuracy): agg{i}_batch_identity_pred / _ccs float32 [n_batches], agg{i}_identity,
          agg{i}_yield_over_ccs, agg{i}_accuracy float32.  agg0 has a batch that is all gaps (alignment length 0,
          identity 1.0) and a last batch of one window; agg1 has no CCS batch identity at or above 0.997 while the
          prediction's is (divide_no_nan gives 0); agg2 has every batch at or above the threshold.
What is NOT pinned: TensorFlow's own kernels (exp / log / sums are NumPy's, in float32, sums in order), the Keras Mean
(restated in tf_shim.py), and tf.argmax's tie rule (NumPy's first maximum, as TensorFlow's CPU kernel does).
Needs a checkout of google/deepconsensus v1.2 at REF and no GPU; the output is committed.  The archive is written with
fixed zip timestamps, so a rerun reproduces it byte for byte.
"""
import io
import itertools
import os
import sys
import zipfile

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "scripts"))
REF = "/root/reference"
OUT = os.path.join(REPO, "tests", "golden", "ref_eval_edges.npz")

import tf_shim  # noqa: E402

F32 = np.float32
EDGE_LENGTHS = (1, 2, 31, 32, 33, 127, 128, 129, 255, 256)
SMALL_SETTINGS = ((10.0, 0.1), (10.0, None))
EDGE_SETTINGS = ((10.0, 0.1), (10.0, None), (1e9, None), (10.0, 0.01), (2.0, 1.0))
COUNT_KEYS = ("num_matches", "num_insertions", "num_deletions", "num_correct_matches", "alignment_length")
PROB_STYLES = ("sharp", "flat", "onehot", "uniform", "tie2", "scale3.7", "scale1e-3")


def import_reference():
  tf = tf_shim.install()
  tf_shim.install_losses_ops(tf)
  sys.path.insert(0, REF)
  from deepconsensus.models import losses_and_metrics
  return losses_and_metrics


def one_hot(ids):
  return np.eye(5, dtype=F32)[np.asarray(ids, np.int64)]


def counts_of(mv):
  return np.stack([np.asarray(mv[k]) for k in COUNT_KEYS], -1).astype(np.int32)


def run_reference(lm, lab, probs, ccs, settings):
  """The stored outputs of one group (module docstring)."""
  y = lab.astype(F32)
  out = {"labels": lab.astype(np.uint8), "probs": probs.astype(F32), "ccs": ccs.astype(np.uint8)}
  _, _, mv = lm.AlignmentMetric().alignment(y, probs)
  out["pred_counts"] = counts_of(mv)
  ccs_one_hot = lm.tf.one_hot(ccs.astype(np.int32), depth=5, dtype=lm.tf.float32)   # ids 5.. give a zero row
  _, _, mv = lm.AlignmentMetric().alignment(y, ccs_one_hot)
  out["ccs_counts"] = counts_of(mv)
  out["exact"] = np.array([exact_flag(lm, y[b:b + 1], probs[b:b + 1]) for b in range(y.shape[0])], np.uint8)
  out["loss_settings"] = np.array([(dc, np.nan if reg is None else reg) for dc, reg in settings], np.float64)
  out["loss"] = np.stack([np.asarray(lm.AlignmentLoss(del_cost=dc, loss_reg=reg, width=None).eval(y, probs), F32)
                          for dc, reg in settings])
  return out


def exact_flag(lm, y, p):
  acc = lm.PerExampleAccuracy()
  acc.update_state(y, p)
  return int(round(float(acc.result())))


# ---------------------------------------------------------------------------------------------------- L = 3 and 4
def all_sequences(L):
  return np.array(list(itertools.product(range(5), repeat=L)), np.uint8)


def exhaustive_l3():
  seqs = all_sequences(3)                                  # 125 x 3
  perm = np.random.default_rng(3).permutation(125)
  a, b = np.meshgrid(np.arange(125), np.arange(125), indexing="ij")
  a, b = a.reshape(-1), b.reshape(-1)
  return seqs[a], one_hot(seqs[b]), seqs[perm[b]]


def tie_prone(rng, lab, L):
  """One prediction for `lab`, chosen among the shapes whose alignments tie."""
  kind = rng.integers(0, 8)
  base = int(rng.integers(1, 5))
  s = list(lab)
  if kind == 0:                                            # shift right by one, the first position filled
    s = [int(rng.integers(0, 5))] + s[:-1]
  elif kind == 1:                                          # shift left by one, the last position filled
    s = s[1:] + [int(rng.integers(0, 5))]
  elif kind == 2:                                          # one deletion
    i = int(rng.integers(0, L))
    s = s[:i] + s[i + 1:] + [0]
  elif kind == 3:                                          # one insertion
    i = int(rng.integers(0, L + 1))
    s = (s[:i] + [base] + s[i:])[:L]
  elif kind == 4:                                          # one repeated base
    s = [base] * L
  elif kind == 5:                                          # a two-base period
    other = int(rng.integers(0, 5))
    s = [base if t % 2 == 0 else other for t in range(L)]
  elif kind == 6:                                          # interleaved gaps
    s = [v if rng.random() < 0.6 else 0 for v in s]
    s = [v for v in s if v] + [0] * L
    out = []
    for v in s:
      if len(out) >= L:
        break
      out.append(v)
      if rng.random() < 0.5:
        out.append(0)
    s = out
  else:
    s = list(rng.integers(0, 5, size=L))
  return np.array(s[:L], np.uint8)


def sampled_l4():
  rng = np.random.default_rng(4)
  seqs = all_sequences(4)
  lab = np.repeat(seqs, 32, axis=0)
  pred = np.stack([tie_prone(rng, lab[w], 4) for w in range(lab.shape[0])])
  ccs = np.roll(pred, 7, axis=0)
  return lab, one_hot(pred), ccs


def random_l24():
  rng = np.random.default_rng(24)
  lab, pred, ccs = (rng.integers(0, 5, size=(4000, 24)).astype(np.uint8) for _ in range(3))
  return lab, one_hot(pred), ccs


# ---------------------------------------------------------------------------------------------------- length edges
def bases(rng, n):
  return rng.integers(1, 5, size=n).astype(np.uint8)


def padded(seq, L):
  out = np.zeros(L, np.uint8)
  seq = np.asarray(seq, np.uint8)[:L]
  out[:len(seq)] = seq
  return out


def mutate(rng, seq, rate):
  s = seq.copy()
  hit = rng.random(s.shape) < rate
  s[hit] = rng.integers(0, 5, size=int(hit.sum()))
  return s


def structured_pairs(rng, L):
  """(label, prediction) id pairs of length L (module docstring)."""
  full = bases(rng, L)
  short = padded(bases(rng, max(1, (3 * L) // 4)), L)       # trailing padding leaves room for insertions
  run = max(1, L // 4)
  cut = L // 3
  pairs = [
      (full, full.copy()),                                                    # identical
      (full, padded(np.concatenate([bases(rng, 1), full[:-1]]), L)),         # shifted right by one
      (short, padded(short[1:], L)),                                          # shifted left by one
      (padded([1 + (t % 2) for t in range(L)], L), padded([2 - (t % 2) for t in range(L)], L)),   # ATAT.. vs TATA..
      (full, padded(np.concatenate([full[:cut], full[cut + run:]]), L)),     # a deletion run
      (short, padded(np.concatenate([short[:cut], bases(rng, run), short[cut:]]), L)),   # an insertion run
      (np.zeros(L, np.uint8), full.copy()),                                   # all-gap label
      (full, np.zeros(L, np.uint8)),                                          # all-gap prediction
      (np.zeros(L, np.uint8), np.zeros(L, np.uint8)),                         # both all gaps
  ]
  spread = np.zeros(L, np.uint8)                                              # interleaved gaps: the label's bases
  spread[::2] = short[:(L + 1) // 2]                                          # with a gap after each
  pairs.append((short, spread))
  pairs.append((spread, short.copy()))
  last = np.zeros(L, np.uint8)
  last[L - 1] = bases(rng, 1)[0]
  pairs.append((last, last.copy()))                                           # one base at L - 1, both sides
  pairs.append((full, last.copy()))
  pairs.append((full, np.full(L, bases(rng, 1)[0], np.uint8)))               # one repeated base
  pairs.append((full, mutate(rng, full, 0.05)))
  pairs.append((short, mutate(rng, short, 0.30)))
  return pairs


def probs_for(rng, pred, style):
  """Probability rows [L, 5] whose argmax is (mostly) `pred`, in one of PROB_STYLES."""
  L = pred.shape[0]
  if style == "onehot":
    return one_hot(pred)
  z = rng.normal(size=(L, 5)).astype(F32)
  z = z * F32(0.3) + F32(0.5) * one_hot(pred) if style == "flat" else z + F32(6.0) * one_hot(pred)
  e = np.exp(z - z.max(-1, keepdims=True))
  p = (e / e.sum(-1, keepdims=True)).astype(F32)
  if style == "uniform":                                   # every third row uniform: the argmax tie goes to 0
    p[::3] = F32(0.2)
  elif style == "tie2":                                    # every second row: two tokens share the maximum
    for j in range(0, L, 2):
      a, b = int(pred[j]), int((pred[j] + 1 + rng.integers(0, 4)) % 5)
      row = np.full(5, F32(0.05), F32)
      row[a] = row[b] = F32(0.4)
      p[j] = row
  elif style == "scale3.7":
    p = (p * F32(3.7)).astype(F32)
  elif style == "scale1e-3":
    p = (p * F32(1e-3)).astype(F32)
  return p


def with_odd_ccs_ids(rng, seq):
  """A CCS row: `seq` at 10 % mutation, with ids 5, 6 and 255 at some positions (they decode as gaps)."""
  c = mutate(rng, seq, 0.10)
  odd = rng.random(c.shape) < 0.15
  c[odd] = rng.choice(np.array([5, 6, 255], np.uint8), size=int(odd.sum()))
  return c


def length_edge(L):
  rng = np.random.default_rng(1000 + L)
  labs, probs, ccs = [], [], []
  for w, (lab, pred) in enumerate(structured_pairs(rng, L)):
    labs.append(lab)
    probs.append(probs_for(rng, pred, PROB_STYLES[w % len(PROB_STYLES)]))
    ccs.append(with_odd_ccs_ids(rng, lab if w % 2 else pred))
  return np.stack(labs), np.stack(probs), np.stack(ccs)


# ---------------------------------------------------------------------------------------------------- aggregation
def aggregation(lm, lab, probs, ccs, bs):
  y = lab.astype(F32)
  acc, yld, mean = lm.PerExampleAccuracy(), lm.YieldOverCCSMetric(), lm.tf.keras.metrics.Mean()
  ident, ident_ccs = [], []
  for b0 in range(0, lab.shape[0], bs):
    sl = slice(b0, b0 + bs)
    acc.update_state(y[sl], probs[sl])
    ic, ip = lm.get_batch_identity_ccs_pred(ccs[sl].astype(F32), probs[sl], y[sl], lm.AlignmentMetric())
    yld.update_state(ic, ip)
    mean.update_state(ip)
    ident.append(float(ip))
    ident_ccs.append(float(ic))
  return dict(batch_size=np.int32(bs), batch_identity_pred=np.array(ident, F32),
              batch_identity_ccs=np.array(ident_ccs, F32), identity=F32(mean.result()),
              yield_over_ccs=F32(yld.result()), accuracy=F32(acc.result()))


def aggregation_cases(rng):
  L = 40
  good = np.stack([padded(bases(rng, 30 + w), L) for w in range(9)])
  cases = []
  # agg0: batch 0 all gaps everywhere, batch 1 mixed, batch 2 a single window
  lab = good.copy()
  lab[:4] = 0
  pred = lab.copy()
  pred[5] = mutate(rng, pred[5], 0.2)
  ccs = lab.copy()
  ccs[6] = mutate(rng, ccs[6], 0.1)
  cases.append((lab, one_hot(pred), ccs, 4))
  # agg1: every CCS batch below 0.997, the prediction exact
  ccs = np.stack([mutate(rng, s, 0.3) for s in good])
  cases.append((good, one_hot(good), ccs, 4))
  # agg2: every batch at or above the threshold on both sides, batch size 2 with a last batch of one
  cases.append((good, one_hot(good), good.copy(), 2))
  return cases


# ---------------------------------------------------------------------------------------------------- output
def save_npz(path, arrays):
  """np.savez_compressed with fixed member timestamps, so that identical arrays give identical bytes."""
  with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as zf:
    for key in sorted(arrays):
      buf = io.BytesIO()
      np.lib.format.write_array(buf, np.asanyarray(arrays[key]), allow_pickle=False)
      info = zipfile.ZipInfo(key + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
      info.compress_type = zipfile.ZIP_DEFLATED
      zf.writestr(info, buf.getvalue())


def main():
  lm = import_reference()
  out = {}

  def put(group, values):
    for k, v in values.items():
      out["%s_%s" % (group, k)] = v

  put("L3", run_reference(lm, *exhaustive_l3(), SMALL_SETTINGS))
  print("L3", out["L3_labels"].shape[0], "windows")
  put("L4", run_reference(lm, *sampled_l4(), SMALL_SETTINGS))
  print("L4", out["L4_labels"].shape[0], "windows")
  put("rand24", run_reference(lm, *random_l24(), SMALL_SETTINGS))
  for L in EDGE_LENGTHS:
    put("len%d" % L, run_reference(lm, *length_edge(L), EDGE_SETTINGS))
    print("len%d" % L, out["len%d_pred_counts" % L][:, 4], out["len%d_loss" % L][0])
  rng = np.random.default_rng(77)
  for i, (lab, probs, ccs, bs) in enumerate(aggregation_cases(rng)):
    put("agg%d" % i, run_reference(lm, lab, probs, ccs, SMALL_SETTINGS[:1]))
    put("agg%d" % i, aggregation(lm, lab, probs, ccs, bs))
    print("agg%d" % i, out["agg%d_batch_identity_pred" % i], out["agg%d_batch_identity_ccs" % i],
          out["agg%d_yield_over_ccs" % i])
  save_npz(OUT, out)
  print("->", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
  main()
