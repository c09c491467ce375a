// Per-token epilogue shared by head_kernel and the strict-fp32 head.
#pragma once
#include <math.h>

#include "common.h"
#include "quality.cuh"

namespace dcb {

// logits (+ fc1 bias) -> softmax -> argmax -> Phred -> calibration -> cap / round -> ASCII, for one token
// (networks.py:238, quick_inference.py:377-414).
__device__ __forceinline__ void head_finish(const HeadParams& p, float (&lg)[kVocab], size_t oidx) {
  float mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < kVocab; ++j) { lg[j] += p.bfc[j]; mx = fmaxf(mx, lg[j]); }
  // softmax (networks.py:238), float32
  float ex[kVocab], sum = 0.f;
#pragma unroll
  for (int j = 0; j < kVocab; ++j) { ex[j] = expf(lg[j] - mx); sum += ex[j]; }
  float pr[kVocab], pmax = -1.f;
  int arg = 0;
#pragma unroll
  for (int j = 0; j < kVocab; ++j) {
    pr[j] = ex[j] / sum;
    if (pr[j] > pmax) { pmax = pr[j]; arg = j; }  // first maximum wins (np.argmax)
  }
  // quick_inference.py:378-389
  const float err = 1.f - pmax;
  // float32 log10, correctly rounded (double log10 rounded once): NumPy's float32 log10 is the platform libm's / SVML's
  // (<= 1 ulp, not always correctly rounded), so "the same float32 value as the reference" is only defined up to
  // that ulp; the correctly rounded value is the one every such library approximates.  err == 0 -> +inf.
  const float qf = -10.f * (float)log10((double)err);
  int qi = head_quality(p, qf);                              // calibration, cap, round (quality.cuh)
  qi = qi < 0 ? 0 : qi;
  const char vocab[kVocab] = {' ', 'A', 'T', 'C', 'G'};
  p.bases[oidx] = (uint8_t)vocab[arg];
  p.quals[oidx] = (uint8_t)(qi + 33);
  if (p.probs) {
#pragma unroll
    for (int j = 0; j < kVocab; ++j) p.probs[oidx * kVocab + j] = pr[j];
  }
  if (p.logits) {
#pragma unroll
    for (int j = 0; j < kVocab; ++j) p.logits[oidx * kVocab + j] = lg[j];
  }
}

}  // namespace dcb
