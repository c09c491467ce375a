"""Device time of the distillation training pieces, with the card's name and power limit read in the same run:
  * dcb_distill_loss_grad (loss + gradient) beside dcb_distill_loss, 1024 windows at L = 100 and 120, both logit losses:
    the median of 20 calls (CUDA events inside the engine, after 3 warm-up calls);
  * one distillation_objective forward + backward on 1024 windows, L = 100 (torch CUDA events around it, median of 20);
  * teacher_logits of a 6-layer teacher on 1024 windows, L = 100, bf16 (torch CUDA events, median of 20).
Seeded random logits, labels and rows; needs a GPU."""
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from deepconsensus_b200 import engine, params as params_lib, synthetic, weights as weights_lib  # noqa: E402


def _median_ms(torch, fn, n=20, warmup=3):
  for _ in range(warmup):
    fn()
  times = []
  for _ in range(n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    times.append(a.elapsed_time(b))
  return float(np.median(times))


def main():
  import torch
  from deepconsensus_b200 import torch_loss
  card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                        text=True).stdout.strip()
  print("card:", card)
  B = 1024
  ps = params_lib.get_config("transformer_learn_values_distill+test")
  ps.batch_size = B
  params_lib.modify_params(ps, max_length=100)
  student = engine.B200Model(ps, weights_lib.init_weights(ps, seed=1), max_batch=B)
  pt = params_lib.synthetic_params(max_passes=20, max_length=100)
  teacher = engine.B200Model(pt, weights_lib.init_weights(pt, seed=2), max_batch=B)
  rng = np.random.default_rng(0)
  try:
    for L in (100, 120):
      t = (rng.normal(size=(B, L, 5)) * 3).astype(np.float32)
      s = (t + rng.normal(size=t.shape)).astype(np.float32)
      for ident in ("mean_squared_error", "kl_divergence"):
        res = {}
        for name, fn in (("loss", lambda: student.distill_loss(t, s, 1.0, ident)["ms"]),
                         ("loss+grad", lambda: student.distill_loss_grad(t, s, 1.0, ident)["ms"])):
          for _ in range(3):
            fn()
          res[name] = float(np.median([fn() for _ in range(20)]))
        print("dcb_distill_loss_grad L=%d B=%d %s: %.4f ms (dcb_distill_loss %.4f ms)" %
              (L, B, ident, res["loss+grad"], res["loss"]))
    dev = torch.device("cuda", 0)
    L = 100
    lab = rng.integers(1, 5, (B, L)).astype(np.uint8)
    lab[rng.random((B, L)) < 0.15] = 0
    y = torch.tensor(lab, device=dev)
    tl = torch.tensor((rng.normal(size=(B, L, 5)) * 3).astype(np.float32), device=dev)
    z = torch.tensor((rng.normal(size=(B, L, 5)) * 3).astype(np.float32), device=dev, requires_grad=True)

    def step():
      z.grad = None
      torch_loss.distillation_objective(student, y, z, tl)["total_loss"].backward()
    print("distillation_objective forward + backward B=%d L=%d: %.3f ms" % (B, L, _median_ms(torch, step)))
    rows = torch.tensor(synthetic.make_rows(pt, B, seed=3)[..., 0], device=dev)
    print("teacher_logits, 6-layer teacher, bf16, B=%d L=%d: %.3f ms" %
          (B, L, _median_ms(torch, lambda: torch_loss.teacher_logits(teacher, rows))))
  finally:
    student.close()
    teacher.close()


if __name__ == "__main__":
  main()
