"""Generates tests/golden/ref_distill.npz by EXECUTING the reference's own DistillationLoss
(deepconsensus/models/losses_and_metrics.py, unmodified, from the checkout at REF) on the NumPy stand-in for TensorFlow
in scripts/tf_shim.py (install() + install_losses_ops(): tf.nn.softmax, tf.math.reduce_mean and a tf.keras.losses.get that
resolves the Keras identifiers of the two logit losses).

Cases (checked by tests/test_distill_host.py against oracle/distill.py, and on the GPU by tests/test_gpu_distill.py):
  rand_L{100,120}_{logits_teacher,logits_student}   random logit pairs, 6 windows: students near their teacher at three
                                                    noise levels, an unrelated student, a sharp (scaled x8) pair, and a
                                                    student equal to its teacher (loss exactly 0)
  rand_L{100,120}_{mse,kl}_T{1.0,2.5}               DistillationLoss(temperature=T, logit_loss=tf.keras.losses.get(id))
                                                    .call(teacher, student), float32 [6]
  rand_L100_labels, rand_L100_student_loss          the student term of the distillation loop's compute_loss
                                                    (model_distillation.py:242-270): AlignmentLoss(del_cost 10,
                                                    loss_reg 0.1) of the labels against softmax(student logits)
  rand_L100_total_mse_T1.0                          its per-example total student_alpha * student + distill_alpha *
                                                    distill with the transformer_learn_values_distill config's alphas
                                                    (read from the reference's model_configs.py), and
  rand_L100_batch_total                             tf.nn.compute_average_loss of those totals over batches of 3
What is NOT pinned: TensorFlow's and Keras's own kernels (softmax / exp / log / sums are NumPy's, in float32, sums in
order), nor the Keras losses themselves, which are restated in tf_shim.py.
Needs a checkout of google/deepconsensus v1.2 at REF and no GPU; the output is committed.
"""
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "scripts"))
REF = "/root/reference"
OUT = os.path.join(REPO, "tests", "golden", "ref_distill.npz")

import tf_shim  # noqa: E402

IDS = {"mse": "mean_squared_error", "kl": "kl_divergence"}
TEMPERATURES = (1.0, 2.5)
BATCH = 3


def import_reference():
  tf = tf_shim.install()
  tf_shim.install_losses_ops(tf)
  sys.path.insert(0, REF)
  from deepconsensus.models import losses_and_metrics
  from deepconsensus.models import model_configs
  return tf, losses_and_metrics, model_configs


def logit_pairs(rng, L):
  teacher = (rng.normal(size=(6, L, 5)) * 3.0).astype(np.float32)
  student = np.empty_like(teacher)
  for b, noise in enumerate((0.05, 0.5, 2.0)):
    student[b] = teacher[b] + (rng.normal(size=(L, 5)) * noise).astype(np.float32)
  student[3] = (rng.normal(size=(L, 5)) * 3.0).astype(np.float32)
  teacher[4] *= np.float32(8.0)
  student[4] = teacher[4] + (rng.normal(size=(L, 5)) * 1.0).astype(np.float32)
  student[5] = teacher[5]                                   # identical: the loss is exactly 0
  return teacher, student.astype(np.float32)


def main():
  tf, lm, mc = import_reference()
  cfg = mc.get_config("transformer_learn_values_distill+test")
  student_alpha, distill_alpha = float(cfg.student_alpha), float(cfg.distill_alpha)
  assert cfg.logit_loss_identifier == "mean_squared_error" and float(cfg.temperature) == 1.0
  rng = np.random.default_rng(1170)
  out = dict(student_alpha=np.float64(student_alpha), distill_alpha=np.float64(distill_alpha),
             batch_size=np.int32(BATCH))
  for L in (100, 120):
    key = f"rand_L{L}"
    teacher, student = logit_pairs(rng, L)
    out[key + "_logits_teacher"], out[key + "_logits_student"] = teacher, student
    for short, ident in IDS.items():
      for T in TEMPERATURES:
        loss = lm.DistillationLoss(temperature=T, logit_loss=tf.keras.losses.get(ident),
                                   reduction=tf.keras.losses.Reduction.NONE).call(teacher, student)
        loss = np.asarray(loss, np.float32)
        assert loss[5] == 0.0, (key, short, T, loss)
        out[f"{key}_{short}_T{T}"] = loss
        print(key, short, T, loss)
  # the distillation loop's compute_loss on the L = 100 case, with the distill config's own parameters
  lab = rng.integers(1, 5, size=(6, 100))
  lab[rng.random(lab.shape) < 0.15] = 0
  for b in range(6):
    lab[b, 100 - rng.integers(0, 25):] = 0
  lab = lab.astype(np.uint8)
  teacher, student = out["rand_L100_logits_teacher"], out["rand_L100_logits_student"]
  student_preds = np.asarray(tf.nn.softmax(student), np.float32)
  sl = np.asarray(lm.AlignmentLoss(del_cost=cfg.del_cost, loss_reg=cfg.loss_reg, width=cfg.band_width)
                  .call(lab.astype(np.float32), student_preds), np.float32)
  dl = np.asarray(lm.DistillationLoss(temperature=cfg.temperature,
                                      logit_loss=tf.keras.losses.get(cfg.logit_loss_identifier),
                                      reduction=tf.keras.losses.Reduction.NONE).call(teacher, student), np.float32)
  total = (np.float32(student_alpha) * sl + np.float32(distill_alpha) * dl).astype(np.float32)
  # tf.nn.compute_average_loss(per_example_loss, global_batch_size): reduce_sum / batch size, in float32
  batch_total = np.array([np.asarray(tf.reduce_sum(total[b0:b0 + BATCH])) / np.float32(BATCH)
                          for b0 in range(0, 6, BATCH)], np.float32)
  out.update(rand_L100_labels=lab, rand_L100_student_loss=sl, **{"rand_L100_total_mse_T1.0": total},
             rand_L100_batch_total=batch_total)
  print("compute_loss totals", total, "batches", batch_total)
  np.savez_compressed(OUT, **out)
  print("->", OUT)


if __name__ == "__main__":
  main()
