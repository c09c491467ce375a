// Strict-precision path of the dcb200 engine: the same forward pass in the reference's arithmetic -- float32
// operands, float32 FMA accumulation, float32 softmax / LayerNorm (networks.py:506-507 casts the embedded input to
// float32 and every Keras layer below runs in float32).  Selected per engine (dcb_config.precision =
// DCB_PRECISION_FP32) or per call (DCB_STRICT_FP32).
//
// What it is for: the default path rounds tensor-core operands to bf16, which moves logits by
// 0.02-0.1 and flips the argmax at near-ties.  This path differs from the reference's float32 graph only by summation
// order (measured ~1e-5 on logits), so it produces identical bases wherever the float32 top-2 margin exceeds 1e-3 and
// is the on-device yardstick the default path is compared with at full batch sizes (bench.py "parity", tests).
//
// It runs on the CUDA cores (the tensor cores have no float32-operand mode: tf32 keeps 10 mantissa bits), as
// plain global-memory kernels, row-major [tokens, features] activations, windows packed back to back:
//
//   strict_embed_kernel     format_rows clip + id + gather + sqrt(width) scale + zero-at-id-0 + concat
//                           (data_providers.py:151-162, networks.py:42-63,457-507)
//   strict_gemm_kernel      C = epilogue(A[M,K] . B[K,N]): + bias, ReLU, * scale, + residual, + positional table
//                           (condenser networks.py:509-516; q/k/v/out EinsumDense attention_layer.py:169-171,218;
//                            FFN ffn_layer.py:83-86; ReZero / residual encoder_stack.py:88-92)
//   strict_layernorm_kernel LayerNormalization(eps=1e-6), two-pass mean / biased variance (encoder_stack.py:62-64,79)
//   strict_attention_kernel q k^T, band mask, softmax, . v per (window, head, query) (attention_layer.py:198-214)
//   strict_head_kernel      final LayerNorm, fc1, then the shared head_finish epilogue
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "head_finish.cuh"
#include "kernels.h"

namespace dcb {

// ------------------------------------------------------------------------------------------------- embed
// One CTA per window; thread = position (coalesced along L for every input row).
__global__ void __launch_bounds__(256)
strict_embed_kernel(const float* __restrict__ rows, int R, int L, int E,
                    const StrictEmbedRow* __restrict__ meta, const float* __restrict__ tables,
                    float* __restrict__ emb, int* __restrict__ status) {
  const int b = blockIdx.x;
  int bad = 0;
  for (int l = threadIdx.x; l < L; l += blockDim.x) {
    float* out = emb + ((size_t)b * L + l) * E;
    for (int r = 0; r < R; ++r) {
      const StrictEmbedRow m = meta[r];
      float v = rows[((size_t)b * R + r) * L + l];
      if (m.clip_hi > 0.f) v = fminf(fmaxf(v, 0.f), m.clip_hi);   // format_rows: np.clip(x, 0, MAX)
      v += (float)m.shift;                                        // ccs_bq + 1 (networks.py:495)
      int id = (int)v;                                            // tf.cast(float -> int32): truncation
      if (id < 0 || id >= m.vocab) { bad = 1; id = id < 0 ? 0 : m.vocab - 1; }
      const float* t = tables + m.table_off + (size_t)id * m.width;
      for (int j = 0; j < m.width; ++j) out[m.col0 + j] = t[j];   // pre-scaled by sqrt(width), row 0 zeroed
    }
  }
  if (bad) atomicOr(status, 1);
}

// ------------------------------------------------------------------------------------------------- GEMM
// 128 x 96 tile, 8 x 6 per thread, K step 8, register-staged global loads.  N = 280 / 2048 / 840 waste <= 3 %.
constexpr int kSBM = 128, kSBN = 96, kSBK = 8, kSTM = 8, kSTN = 6;

__global__ void __launch_bounds__(256)
strict_gemm_kernel(const float* __restrict__ A, const float* __restrict__ Bm, float* __restrict__ C, int M, int N, int K,
                   StrictEpi ep) {
  __shared__ float As[kSBK][kSBM + 4];
  __shared__ float Bs[kSBK][kSBN];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.y * kSBM, n0 = blockIdx.x * kSBN;
  const int ty = tid / 16, tx = tid % 16;        // thread tile: rows ty*8.., cols tx*6..
  // A tile loads: 128 x 8 = 1024 values, 4 per thread: row = tid / 2, k = (tid % 2) * 4 + i
  const int a_row = tid >> 1, a_k = (tid & 1) * 4;
  // B tile loads: 8 x 96 = 768 values, 3 per thread: k = tid / 32, col = (tid % 32) * 3 + i
  const int b_k = tid >> 5, b_c = (tid & 31) * 3;
  float ra[4], rb[3];
  auto gload = [&](int k0) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int gm = m0 + a_row, gk = k0 + a_k + i;
      ra[i] = (gm < M && gk < K) ? A[(size_t)gm * K + gk] : 0.f;
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const int gk = k0 + b_k, gn = n0 + b_c + i;
      rb[i] = (gk < K && gn < N) ? Bm[(size_t)gk * N + gn] : 0.f;
    }
  };
  float acc[kSTM][kSTN];
#pragma unroll
  for (int i = 0; i < kSTM; ++i)
#pragma unroll
    for (int j = 0; j < kSTN; ++j) acc[i][j] = 0.f;
  gload(0);
  for (int k0 = 0; k0 < K; k0 += kSBK) {
#pragma unroll
    for (int i = 0; i < 4; ++i) As[a_k + i][a_row] = ra[i];
#pragma unroll
    for (int i = 0; i < 3; ++i) Bs[b_k][b_c + i] = rb[i];
    __syncthreads();
    if (k0 + kSBK < K) gload(k0 + kSBK);
#pragma unroll
    for (int kk = 0; kk < kSBK; ++kk) {
      float a[kSTM], bb[kSTN];
#pragma unroll
      for (int i = 0; i < kSTM; ++i) a[i] = As[kk][ty * kSTM + i];
#pragma unroll
      for (int j = 0; j < kSTN; ++j) bb[j] = Bs[kk][tx * kSTN + j];
#pragma unroll
      for (int i = 0; i < kSTM; ++i)
#pragma unroll
        for (int j = 0; j < kSTN; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < kSTM; ++i) {
    const int gm = m0 + ty * kSTM + i;
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < kSTN; ++j) {
      const int gn = n0 + tx * kSTN + j;
      if (gn >= N) continue;
      float v = acc[i][j];
      if (ep.bias) v += ep.bias[gn];
      if (ep.relu) v = fmaxf(v, 0.f);
      v *= ep.scale;
      if (ep.residual) v = ep.residual[(size_t)gm * N + gn] + v;
      if (ep.pe) v += ep.pe[(size_t)(gm % ep.pe_L) * N + gn];
      C[(size_t)gm * N + gn] = v;
    }
  }
}

// ------------------------------------------------------------------------------------------------- LayerNorm
// One warp per row of kD.
__global__ void __launch_bounds__(256)
strict_layernorm_kernel(const float* __restrict__ x, float* __restrict__ y, int M, const float* __restrict__ g,
                        const float* __restrict__ bta) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= M) return;
  const float* xr = x + (size_t)row * kD;
  float v[(kD + 31) / 32];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < (kD + 31) / 32; ++i) {
    const int c = i * 32 + lane;
    v[i] = c < kD ? xr[c] : 0.f;
    s += v[i];
  }
#pragma unroll
  for (int d = 16; d; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
  const float mean = s * (1.f / kD);
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < (kD + 31) / 32; ++i) {
    const int c = i * 32 + lane;
    const float dlt = c < kD ? v[i] - mean : 0.f;
    ss = fmaf(dlt, dlt, ss);
  }
#pragma unroll
  for (int d = 16; d; d >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, d);
  const float rstd = 1.f / sqrtf(ss * (1.f / kD) + 1e-6f);
#pragma unroll
  for (int i = 0; i < (kD + 31) / 32; ++i) {
    const int c = i * 32 + lane;
    if (c < kD) y[(size_t)row * kD + c] = (v[i] - mean) * rstd * g[c] + bta[c];
  }
}

// ------------------------------------------------------------------------------------------------- attention
// One warp per (window, head, query position).  q is already scaled by depth^-1/2 (attention_layer.py:196-197).
// Keys outside the band get logit -1e9 in the reference (:207); exp(-1e9 - max) is exactly 0 in float32, so they are
// skipped.  win <= 0: full attention.
__global__ void __launch_bounds__(256)
strict_attention_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                        float* __restrict__ o, int nwindows, int L, int win) {
  extern __shared__ float s_p[];                      // [8 warps][L] probabilities, then [8][kDH] the query row
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long gw = (long long)blockIdx.x * 8 + warp;
  const long long total = (long long)nwindows * kHeads * L;
  if (gw >= total) return;
  const int f = (int)(gw % L);
  const int h = (int)((gw / L) % kHeads);
  const int b = (int)(gw / ((long long)L * kHeads));
  float* p = s_p + (size_t)warp * L;
  float* sq = s_p + (size_t)8 * L + (size_t)warp * kDH;
  const size_t base = (size_t)b * L * kD + (size_t)h * kDH;
  for (int c = lane; c < kDH; c += 32) sq[c] = q[base + (size_t)f * kD + c];
  __syncwarp();
  int lo = 0, hi = L - 1;
  if (win > 0) { lo = max(0, f - win); hi = min(L - 1, f + win); }
  float mx = -INFINITY;
  for (int t = lo + lane; t <= hi; t += 32) {
    const float* kr = k + base + (size_t)t * kD;
    float s = 0.f;
    for (int c = 0; c < kDH; ++c) s = fmaf(sq[c], kr[c], s);
    p[t] = s;
    mx = fmaxf(mx, s);
  }
#pragma unroll
  for (int d = 16; d; d >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, d));
  float sum = 0.f;
  for (int t = lo + lane; t <= hi; t += 32) {
    const float e = expf(p[t] - mx);
    p[t] = e;
    sum += e;
  }
#pragma unroll
  for (int d = 16; d; d >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, d);
  __syncwarp();
  const float inv = 1.f / sum;
  for (int c = lane; c < kDH; c += 32) {
    float acc = 0.f;
    for (int t = lo; t <= hi; ++t) acc = fmaf(p[t] * inv, v[base + (size_t)t * kD + c], acc);
    o[base + (size_t)f * kD + c] = acc;
  }
}

// ------------------------------------------------------------------------------------------------- head
// One warp per token: final LayerNorm (encoder_stack.py:197), fc1 (networks.py:342), head_finish.
__global__ void __launch_bounds__(256)
strict_head_kernel(const float* __restrict__ x, int M, HeadParams hp) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= M) return;
  const float* xr = x + (size_t)row * kD;
  float v[(kD + 31) / 32];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < (kD + 31) / 32; ++i) {
    const int c = i * 32 + lane;
    v[i] = c < kD ? xr[c] : 0.f;
    s += v[i];
  }
#pragma unroll
  for (int d = 16; d; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
  const float mean = s * (1.f / kD);
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < (kD + 31) / 32; ++i) {
    const int c = i * 32 + lane;
    const float dlt = c < kD ? v[i] - mean : 0.f;
    ss = fmaf(dlt, dlt, ss);
  }
#pragma unroll
  for (int d = 16; d; d >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, d);
  const float rstd = 1.f / sqrtf(ss * (1.f / kD) + 1e-6f);
  float lg[kVocab];
#pragma unroll
  for (int j = 0; j < kVocab; ++j) lg[j] = 0.f;
#pragma unroll
  for (int i = 0; i < (kD + 31) / 32; ++i) {
    const int c = i * 32 + lane;
    if (c < kD) {
      const float z = (v[i] - mean) * rstd * hp.ln_g[c] + hp.ln_b[c];
#pragma unroll
      for (int j = 0; j < kVocab; ++j) lg[j] = fmaf(z, hp.wfc[c * kVocab + j], lg[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < kVocab; ++j)
#pragma unroll
    for (int d = 16; d; d >>= 1) lg[j] += __shfl_xor_sync(0xffffffffu, lg[j], d);
  if (lane == 0) head_finish(hp, lg, (size_t)row);     // + fc1 bias inside
}

// ------------------------------------------------------------------------------------------------- launchers
void launch_strict_embed(const float* rows, int R, int L, int E, int nwindows, const StrictEmbedRow* meta,
                         const float* tables, float* emb, int* status, cudaStream_t st) {
  if (nwindows > 0) strict_embed_kernel<<<nwindows, 256, 0, st>>>(rows, R, L, E, meta, tables, emb, status);
}

void launch_strict_gemm(const float* A, const float* B, float* C, int M, int N, int K, const StrictEpi& ep,
                        cudaStream_t st) {
  if (M <= 0) return;
  dim3 grid((N + kSBN - 1) / kSBN, (M + kSBM - 1) / kSBM);
  strict_gemm_kernel<<<grid, 256, 0, st>>>(A, B, C, M, N, K, ep);
}

void launch_strict_layernorm(const float* x, float* y, int M, const float* g, const float* b, cudaStream_t st) {
  if (M > 0) strict_layernorm_kernel<<<(M + 7) / 8, 256, 0, st>>>(x, y, M, g, b);
}

void launch_strict_attention(const float* q, const float* k, const float* v, float* o, int nwindows, int L, int win,
                             cudaStream_t st) {
  const long long total = (long long)nwindows * kHeads * L;
  if (total <= 0) return;
  const size_t smem = (size_t)8 * (L + kDH) * sizeof(float);
  strict_attention_kernel<<<(unsigned)((total + 7) / 8), 256, smem, st>>>(q, k, v, o, nwindows, L, win);
}

void launch_strict_head(const float* x, int M, const HeadParams& hp, cudaStream_t st) {
  if (M > 0) strict_head_kernel<<<(M + 7) / 8, 256, 0, st>>>(x, M, hp);
}

}  // namespace dcb
