"""Device time of dcb_alignment_loss_grad (loss + gradient, and loss + gradient + matches) beside dcb_evaluate's, per
1024 windows at L = 100, 120, 200: the median of 20 calls of each (CUDA events inside the engine, after 3 warm-up
calls), with the card's name and power limit.  Random probabilities and labels with 15 % gaps, seeded; needs a GPU."""
import subprocess
import sys
import os

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from deepconsensus_b200 import engine, params as params_lib, weights as weights_lib  # noqa: E402


def main():
  card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                        text=True).stdout.strip()
  print("card:", card)
  B = 1024
  p = params_lib.synthetic_params(max_passes=20, max_length=100)
  m = engine.B200Model(p, weights_lib.init_weights(p, seed=1), max_batch=16)
  rng = np.random.default_rng(0)
  try:
    for L in (100, 120, 200):
      lab = rng.integers(1, 5, (B, L)).astype(np.uint8)
      lab[rng.random((B, L)) < 0.15] = 0
      z = rng.normal(size=(B, L, 5)).astype(np.float32) * 2
      probs = (np.exp(z) / np.exp(z).sum(-1, keepdims=True)).astype(np.float32)
      runs = dict(evaluate=lambda: m.evaluate_windows(probs, lab, lab)["ms"],
                  grad=lambda: m.alignment_loss_grad(probs, lab)["ms"],
                  grad_matches=lambda: m.alignment_loss_grad(probs, lab, want_matches=True)["ms"])
      res = {}
      for name, fn in runs.items():
        for _ in range(3):
          fn()
        res[name] = float(np.median([fn() for _ in range(20)]))
      print("L=%d B=%d: dcb_evaluate %.3f ms, loss+grad %.3f ms, loss+grad+matches %.3f ms; DP scratch %.1f KB per CTA"
            % (L, B, res["evaluate"], res["grad"], res["grad_matches"], (L + 1) ** 2 * 4 / 1024))
  finally:
    m.close()


if __name__ == "__main__":
  main()
