// dcb200 device kernels (sm_90a).
//
//   embed_rows_kernel   rows f32 [B,R,L] -> concatenated embeddings, bf16 operand image
//                       (format_rows clip + OnDeviceEmbedding gathers + concat + cast;
//                        data_providers.py:151-162, networks.py:42-63,457-507)
//   gemm_kernel         persistent, warp-specialised wgmma GEMM: bulk-copy (TMA) producer warp
//                       feeding two consumer warpgroups through an mbarrier ring.  Used for the
//                       condenser (+pos-enc), fused QKV and attention out-proj.
//   ffn_gemm_kernel     the FFN relu(x W1 + b1) W2 + b2 (ffn_layer.py:83-86) with the hidden
//                       activation kept in registers, half of the tiles per launch.
//   band_attention_kernel  banded multi-head softmax attention (attention_layer.py:198-214)
//   qkv_attention_kernel   the q/k/v projection and the banded attention of one window-aligned tile, with q/k/v
//                       kept on the SM, half of the tiles per launch
//   head_kernel         final LayerNorm -> fc1 -> softmax -> argmax -> Phred -> ASCII
//                       (encoder_stack.py:197, networks.py:342,238, quick_inference.py:377-414)
#include "kernels.h"

#include <cuda_bf16.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>

#include "head_finish.cuh"
#include "sm90.cuh"

namespace dcb {

// =====================================================================================
// tile flow between the forward's launches
// =====================================================================================
// In the window-aligned layout every launch of the forward reads only the tiles the launches before it wrote at the
// same index, so a launch may start tile t as soon as the one before it has finished tile t (TileFlow).  Those launches
// are programmatic dependents of the launch before them (launch below): each one lets the next launch start early
// (pdl_launch_dependents) and, before its threads exit, waits until the launch before it has completed (pdl_wait), so
// a launch never completes before its predecessor and whatever follows the forward in the stream still sees it whole.
// Both instructions do nothing in a plain launch.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.b32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// One thread: wait until tile `tile` carries the stamp of the launch before this one (a gpu-scope acquire, so the
// tile's data is visible to this thread and to the threads it later releases through a barrier).  A wait is bounded:
// after a second it sets kStatusTileWait in the submission's status and goes on, so the host reports an error
// instead of the GPU hanging.  Readers with bulk copies (async proxy) follow it with fence.proxy.async.
__device__ __forceinline__ void tile_wait(const TileFlow& f, int tile) {
  if (!f.flags) return;
  if (ld_acquire_gpu(f.flags + tile) == f.wait) return;
  uint64_t t0, t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  while (ld_acquire_gpu(f.flags + tile) != f.wait) {
    __nanosleep(100);
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    if (t - t0 > 1000000000ull) { atomicOr(f.status, kStatusTileWait); return; }
  }
}

__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

// One thread, after every thread that wrote tile `tile` has met it at a barrier: publish the tile (gpu-scope release,
// cumulative over the writes the barrier ordered before it).
__device__ __forceinline__ void tile_done(const TileFlow& f, int tile) {
  if (f.flags) asm volatile("st.release.gpu.global.b32 [%0], %1;" ::"l"(f.flags + tile), "r"(f.done) : "memory");
}

// The two consumer warpgroups (threads 0-255) of the warp-specialised kernels meet on named barrier 1.
__device__ __forceinline__ void consumer_bar_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// =====================================================================================
// embed
// =====================================================================================
// One CTA per 128-token tile.  Phase 1 turns the tile's R x 128 input values into table ids
// (clip -> shift -> truncate -> range check) in shared memory with coalesced loads along L;
// phase 2 assembles 16-byte K-chunks of the operand image from the shared-memory tables.
__global__ void __launch_bounds__(256)
embed_rows_kernel(const float* __restrict__ rows, const uint8_t* __restrict__ packed, PackedLayout pl, int R, int L,
                  int Lw, int M, int echunks,
                  const EmbedCol* __restrict__ cols, const EmbedRow* __restrict__ rowmeta,
                  const __nv_bfloat16* __restrict__ tables, int table_elems,
                  __nv_bfloat16* __restrict__ emb, int* __restrict__ status, TileFlow flow) {
  extern __shared__ __align__(1024) uint8_t smem[];
  pdl_launch_dependents();
  __nv_bfloat16* s_tab = reinterpret_cast<__nv_bfloat16*>(smem);
  const int tab_bytes = (table_elems * 2 + 15) & ~15;
  EmbedCol* s_cols = reinterpret_cast<EmbedCol*>(smem + tab_bytes);
  const int cols_bytes = (echunks * 8 * (int)sizeof(EmbedCol) + 15) & ~15;
  uint16_t* s_ids = reinterpret_cast<uint16_t*>(smem + tab_bytes + cols_bytes);  // [R][128]
  const int tile = blockIdx.x;
  for (int i = threadIdx.x; i < table_elems; i += blockDim.x) s_tab[i] = tables[i];
  for (int i = threadIdx.x; i < echunks * 8; i += blockDim.x) s_cols[i] = cols[i];
  for (int idx = threadIdx.x; idx < R * kTileM; idx += blockDim.x) {
    const int rr = idx / kTileM, r = idx % kTileM;
    const int tok = tile * kTileM + r;
    int id = 0;
    if (tok < M) {
      const int b = tok / Lw, l = tok - b * Lw;
      const EmbedRow m = rowmeta[rr];
      float f = 0.f;                                                       // window padding rows embed to id 0
      if (l < L) f = packed ? packed_value(pl, packed + (size_t)b * pl.stride, rr, l) : __ldg(rows + ((size_t)b * R + rr) * L + l);
      if (m.clip_hi > 0.f) f = fminf(fmaxf(f, 0.f), m.clip_hi);  // format_rows (data_providers.py:151-162)
      f += (float)m.shift;                                         // networks.py:495
      id = (int)f;  // truncation toward zero == tf.cast(float32 -> int32)
      if (id < 0 || id >= m.vocab) {
        atomicOr(status, 1);  // TF's CPU gather raises here; flag and clamp
        id = id < 0 ? 0 : m.vocab - 1;
      }
    }
    s_ids[idx] = (uint16_t)id;
  }
  __syncthreads();
  const int total = echunks * kTileM;
  for (int idx = threadIdx.x; idx < total; idx += blockDim.x) {
    const int kc = idx / kTileM;
    const int r = idx % kTileM;
    uint4 val;
    const EmbedCol c0 = s_cols[kc * 8];
    if (c0.width == 8 && c0.col == 0 && c0.src_row >= 0) {
      // fast path: the whole 16-byte chunk is one width-8 embedding row (bases/pw/ip/ccs/bq/sn)
      const int id = s_ids[c0.src_row * kTileM + r];
      val = *reinterpret_cast<const uint4*>(s_tab + c0.table_off + id * 8);
    } else {
      uint32_t packed[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        uint32_t pr = 0;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const EmbedCol c = s_cols[kc * 8 + 2 * j + h];
          uint32_t bits = 0;
          if (c.src_row >= 0) {
            const int id = s_ids[c.src_row * kTileM + r];
            bits = __bfloat16_as_ushort(s_tab[c.table_off + id * c.width + c.col]);
          }
          pr |= bits << (16 * h);
        }
        packed[j] = pr;
      }
      val = make_uint4(packed[0], packed[1], packed[2], packed[3]);
    }
    uint4* dst = reinterpret_cast<uint4*>(emb + ((size_t)tile * echunks + kc) * kTileM * 8) + r;
    *dst = val;
  }
  __syncthreads();
  if (threadIdx.x == 0) tile_done(flow, tile);
}

// =====================================================================================
// persistent warp-specialised wgmma GEMM
// =====================================================================================
// D[128 x NI] = A[128 x K] * B^T for one 128-token tile and one n-group of NI = NCH * BN columns; A image
// [tile][K/8][128][8], B image per n-group [K/8][NI][8].  Warps 0-7 are two consumer warpgroups (tile rows 0-63 and
// 64-127, accumulators in registers); one thread of warpgroup 2 streams operands into shared memory with bulk copies
// (TMA) that complete on mbarriers.  setmaxnreg moves the producer warpgroup's registers to the consumers.
//
// kAres (the K = 288 projection with several n-groups: fused QKV): a work item is a pair of
// consecutive tiles (2i, 2i + 1).  Both A tiles are loaded once and stay resident while every n-group streams its B
// k-steps through the stage ring; warpgroup w owns tile 2i + w and issues two m64 wgmmas (tile rows 0-63, 64-127) per B
// k-step, so every weight byte that crosses from L2 feeds 256 tokens.  An odd tile count leaves the last pair with one
// tile: the other warpgroup then waits and arrives on every barrier like its partner but issues no wgmma and stores
// nothing.
//
// kAres epilogues are ordered: the warpgroups take turns, one n-group at a time (WG0 group g, WG1 group g, WG0 group
// g + 1, ...), through two mbarriers (turn[w]: warpgroup w may run its next epilogue).  A warpgroup waits for its turn
// only after it has released every stage of the group, so its partner can always drain the ring; it passes the turn on
// once its stores are issued.  In steady state warpgroup 1 runs about one epilogue behind warpgroup 0, so while one
// converts and stores its accumulators the other keeps the tensor cores busy, and the output stores drain under the
// partner's MMAs.  The idle warpgroup of a one-tile pair takes and passes its turns like a working one.
//
// Otherwise (the row epilogue GEMMs, one n-group covering all 288 columns) warpgroup w owns tile rows
// [64 w, 64 w + 64) of one tile, and A and B k-steps stream together.
//
// Split-bf16 weights: the B image may hold K twice as [W_hi; W_lo] (b_ksteps = 2 * a_ksteps, W_lo = bf16(W - W_hi));
// the A k-steps are then read twice, so the accumulator sums A W_hi + A W_lo and the weights carry ~16 mantissa bits.
//
// EPI_QKV  : bf16 into an operand image (column offset group * NI)
// EPI_ROW  : row epilogue (residual / bias / pos-enc / LayerNorm), NI must be the full 288-wide row
enum { EPI_QKV = 0, EPI_ROW = 1 };

template <int BN, int NCH, bool kAres>
struct GemmCfg {
  static constexpr int kNI = NCH * BN;
  static constexpr int kSK = 2;                                   // k-steps per stage
  static constexpr int kABytesPerK = 2 * kTileM * 16;             // 4096
  static constexpr int kBBytesPerK = 2 * kNI * 16;
  static constexpr int kStageBytes = kSK * ((kAres ? 0 : kABytesPerK) + kBBytesPerK);
  // Ring depth.  kAres: the warpgroups take turns at their epilogues (gemm_kernel), so one runs up to an epilogue ahead
  // of the other over the same B stages; 8 stages hold that offset on top of the prefetch depth.  The row GEMMs keep
  // their epilogues in lockstep (taking turns made the condenser and the out-projection slower) and take 8 stages when
  // an item streams at least kLongK of them (the condenser: 10 % faster on an H100 at 700 W); the out-projection (18
  // stages per item) keeps 4.
  static constexpr int kStages = 8;
  static constexpr int kShortStages = 4;
  static constexpr int kLongK = 32;
  __host__ __device__ static constexpr int stages(int kstages) {
    return kAres || kstages >= kLongK ? kStages : kShortStages;
  }
  static constexpr int kMH = kAres ? 2 : 1;                       // m64 row blocks per consumer warpgroup
  static constexpr int kATileBytes = (kDP / 16) * kABytesPerK;    // kAres: one resident A tile, K = 288
  static constexpr int kAresBytes = kAres ? 2 * kATileBytes : 0;  // kAres: the item's two tiles
  static constexpr int kThreads = 384;                            // 2 consumer warpgroups + 1 producer warpgroup
  static constexpr int kVecBytes = kAres ? 0 : 3 * kDP * 4;       // row epilogue: bias, LayerNorm gamma, beta (fp32)
  // ring of nst stages, then 256 bytes of mbarriers, then the row epilogue's vectors
  __host__ __device__ static constexpr int smem_bytes(int nst) { return kAresBytes + nst * kStageBytes + 256 + kVecBytes; }
  static constexpr int kSmemBytes = smem_bytes(kStages);          // the most any launch asks for
  static_assert(kSmemBytes <= 232448, "over the sm_90 opt-in shared memory per block");
  static_assert((2 * kStages + 4) * 8 <= 256, "the mbarriers (full, empty, a_full, a_empty, turn[2]) fill 256 bytes");
};

template <int BN>
__device__ __forceinline__ void wgmma_bn(float (&d)[BN / 2], uint64_t a, uint64_t b, int acc);
template <>
__device__ __forceinline__ void wgmma_bn<144>(float (&d)[72], uint64_t a, uint64_t b, int acc) { wgmma_m64n144k16(d, a, b, acc); }
template <>
__device__ __forceinline__ void wgmma_bn<128>(float (&d)[64], uint64_t a, uint64_t b, int acc) { wgmma_m64n128k16(d, a, b, acc); }

// Sum over the four lanes of a quad (the lanes that share an accumulator row).
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  return v;
}

// The row epilogue's per-column vectors in shared memory: bias, LayerNorm gamma, beta (fp32 [3][kDP]).
__device__ __forceinline__ void row_vectors_to_smem(float* s_vec, const RowEpi& epi) {
  for (int i = threadIdx.x; i < kDP; i += blockDim.x) {
    if (epi.bias) s_vec[i] = epi.bias[i];
    if (epi.ln_g) { s_vec[kDP + i] = epi.ln_g[i]; s_vec[2 * kDP + i] = epi.ln_b[i]; }
  }
}

// Row epilogue of one consumer warpgroup's 64 rows of a tile (accumulator fragment: row, 2 adjacent columns; the
// thread's rows are row0 and row0 + 8): x_new = acc (+ x_old) (+ bias) (+ pos-enc) into the residual image, and the next
// sub-layer's bf16 operand (identity or LayerNorm) into epi.xb unless it is null.  Ends the accumulators' live range.
// kPe false: the caller never adds the positional encoding (epi.pe is ignored), which leaves the epilogue the
// registers its address arithmetic would take.
template <int BN, int NCH, bool kPe = true>
__device__ __forceinline__ void row_epilogue(float (&acc)[NCH][BN / 2], int tile, int row0, int q, const float* s_vec,
                                             const RowEpi& epi) {
  // x is updated in place, so the compiler keeps each x_old load behind every store that precedes it in source
  // order.  Each pass (row half h, accumulator chunk j) therefore issues all of its global loads before its first
  // store: four batches of 18 loads per tile instead of a load -> store round trip per fragment.  The per-column
  // vectors come from shared memory (s_vec).  Fragment (j, jj) holds columns c0 + 2q, c0 + 2q + 1 with
  // c0 = j * BN + jj * 8; in the residual image (and pe_img) it sits c0 * kTileM floats past this thread's xr.
  // (Prefetching the residual tile into L2 from the producer when it starts the item was measured ~3 % slower
  // per step on an H100 SXM at 400 W than these batched loads alone.)
  float* xt = epi.x + (size_t)tile * x_image_elems();
  const int xoff = ((q >> 1) * kTileM + row0) * 4 + 2 * (q & 1);
  const bool ln = epi.ln_g != nullptr;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row0 + 8 * h;
    const int l = (tile * kTileM + row) % epi.L;
    float* xr = xt + xoff + 32 * h;
    const float* per = epi.pe_img ? epi.pe_img + xoff + 32 * h : epi.pe + (size_t)l * kDP + 2 * q;
    const int pe_stride = epi.pe_img ? kTileM : 1;   // floats per column step of c0
    float s1 = 0.f;
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
      float2 ld[BN / 8];
      if (epi.has_xold) {
#pragma unroll
        for (int jj = 0; jj < BN / 8; ++jj)
          ld[jj] = *reinterpret_cast<const float2*>(xr + (j * BN + jj * 8) * kTileM);
#pragma unroll
        for (int jj = 0; jj < BN / 8; ++jj) {
          acc[j][jj * 4 + 2 * h] += ld[jj].x;
          acc[j][jj * 4 + 2 * h + 1] += ld[jj].y;
        }
      }
      if (kPe && epi.pe) {
#pragma unroll
        for (int jj = 0; jj < BN / 8; ++jj)
          ld[jj] = __ldg(reinterpret_cast<const float2*>(per + (size_t)(j * BN + jj * 8) * pe_stride));
      }
#pragma unroll
      for (int jj = 0; jj < BN / 8; ++jj) {
        const int col = j * BN + jj * 8 + 2 * q;
        float2 v = make_float2(acc[j][jj * 4 + 2 * h], acc[j][jj * 4 + 2 * h + 1]);
        if (epi.bias) {
          const float2 b = *reinterpret_cast<const float2*>(s_vec + col);
          v.x += b.x; v.y += b.y;
        }
        if (kPe && epi.pe) { v.x += ld[jj].x; v.y += ld[jj].y; }
        v.x = col < kD ? v.x : 0.f;
        v.y = col + 1 < kD ? v.y : 0.f;
        *reinterpret_cast<float2*>(xr + (j * BN + jj * 8) * kTileM) = v;
        acc[j][jj * 4 + 2 * h] = v.x;
        acc[j][jj * 4 + 2 * h + 1] = v.y;
        s1 += v.x + v.y;
      }
    }
    if (!epi.xb) continue;
    float mean = 0.f, rstd = 1.f;
    if (ln) {   // LayerNorm, eps = 1e-6, biased variance (two passes over the registers)
      mean = quad_sum(s1) * (1.f / kD);
      float s2 = 0.f;
#pragma unroll
      for (int j = 0; j < NCH; ++j)
#pragma unroll
        for (int jj = 0; jj < BN / 8; ++jj) {
          const int col = j * BN + jj * 8 + 2 * q;
          const float d0 = col < kD ? acc[j][jj * 4 + 2 * h] - mean : 0.f;
          const float d1 = col + 1 < kD ? acc[j][jj * 4 + 2 * h + 1] - mean : 0.f;
          s2 += d0 * d0 + d1 * d1;
        }
      rstd = rsqrtf(quad_sum(s2) * (1.f / kD) + 1e-6f);
    }
    __nv_bfloat16* xb = epi.xb + (size_t)tile * act_image_elems(kDP) + row * 8 + 2 * q;
#pragma unroll
    for (int j = 0; j < NCH; ++j)
#pragma unroll
      for (int jj = 0; jj < BN / 8; ++jj) {
        const int col = j * BN + jj * 8 + 2 * q;
        float v0 = acc[j][jj * 4 + 2 * h], v1 = acc[j][jj * 4 + 2 * h + 1];
        if (ln) {
          v0 = col < kD ? (v0 - mean) * rstd * s_vec[kDP + col] + s_vec[2 * kDP + col] : 0.f;
          v1 = col + 1 < kD ? (v1 - mean) * rstd * s_vec[kDP + col + 1] + s_vec[2 * kDP + col + 1] : 0.f;
        }
        *reinterpret_cast<uint32_t*>(xb + (j * BN + jj * 8) * kTileM) = pack_bf16x2(v0, v1);
      }
  }
  // The next item's first wgmma does not read the accumulators (scale-d 0), but the register fences before it
  // do.  Redefining them here ends each half's live range after its last use above, which leaves the second
  // half the registers its batched loads need (without this ptxas spills).
#pragma unroll
  for (int j = 0; j < NCH; ++j)
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[j][i] = 0.f;
}

template <int BN, int NCH, int EPI, bool kAres>
__global__ void __launch_bounds__(384, 1)
gemm_kernel(const __nv_bfloat16* __restrict__ a_img, const __nv_bfloat16* __restrict__ b_img, int a_ksteps, int ksteps,
            int ntiles,
            int ngroups, __nv_bfloat16* __restrict__ out_img, int out_chunks, RowEpi epi, TileFlow flow) {
  using Cfg = GemmCfg<BN, NCH, kAres>;
  static_assert(EPI != EPI_ROW || (Cfg::kNI == kDP && !kAres), "row epilogue needs the full 288-wide row");
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* a_res = smem;
  const int kstages = ksteps / Cfg::kSK;   // ksteps % kSK == 0 (launchers): every stage holds exactly kSK k-steps, so
                                           // its wgmma run is straight-line code with no register moves in between
  const int nst = Cfg::stages(kstages);   // ring depth; the launch asks for Cfg::smem_bytes(nst)
  uint8_t* stage_base = smem + Cfg::kAresBytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(stage_base + nst * Cfg::kStageBytes);
  uint64_t* empty = full + nst;
  uint64_t* a_full = empty + nst;
  uint64_t* a_empty = a_full + 1;
  uint64_t* turn = a_empty + 1;   // [2], kAres: ordered epilogues
  float* s_vec = reinterpret_cast<float*>(stage_base + nst * Cfg::kStageBytes + 256);   // [3][kDP]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if constexpr (EPI == EPI_ROW) row_vectors_to_smem(s_vec, epi);
  if (threadIdx.x == 0) {
    for (int i = 0; i < nst; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 256);   // every consumer thread (no lane-divergent code between the wgmma)
    }
    mbar_init(a_full, 1);
    mbar_init(a_empty, 256);
    mbar_init(&turn[0], 128);   // the other warpgroup's threads, once per epilogue
    mbar_init(&turn[1], 128);
    mbar_fence_init();
  }
  __syncthreads();
  pdl_launch_dependents();

  // kAres: a work item is a tile pair (its n-groups run back to back on the resident A); otherwise a (tile, n-group) pair
  const int nitems = kAres ? (ntiles + 1) / 2 : ntiles * ngroups;
  const int gper = kAres ? ngroups : 1;
  const size_t a_tile_bytes = (size_t)a_ksteps * Cfg::kABytesPerK;
  const size_t b_group_bytes = (size_t)ksteps * Cfg::kBBytesPerK;

  if (warp >= 8) {
    // ------------------------------------------------------------- producer
    setmaxnreg_dec<40>();
    if (warp == 8 && lane == 0) {
      uint32_t slot = 0, phase = 0, it = 0;
      for (int item = blockIdx.x; item < nitems; item += gridDim.x, ++it) {
        const int tile = kAres ? 2 * item : item / ngroups;
        const uint8_t* a_src = reinterpret_cast<const uint8_t*>(a_img) + tile * a_tile_bytes;
        // (flags are set for the row GEMM only, whose items are tiles) the tile is in place before its A copies; the
        // row epilogue's residual loads follow this acquire through the stage barriers (arrive.expect_tx here, then
        // the consumers' wait on `full`)
        tile_wait(flow, tile);
        fence_proxy_async();
        if constexpr (kAres) {   // the pair's A images are contiguous: one copy of one or two tiles
          const uint32_t a_bytes = (uint32_t)((tile + 1 < ntiles ? 2 : 1) * a_tile_bytes);
          mbar_wait(a_empty, (it & 1) ^ 1);
          mbar_arrive_expect_tx(a_full, a_bytes);
          bulk_g2s(a_res, a_src, a_bytes, a_full);
        }
        for (int gi = 0; gi < gper; ++gi) {
          const int grp = kAres ? gi : item % ngroups;
          const uint8_t* b_src = reinterpret_cast<const uint8_t*>(b_img) + grp * b_group_bytes;
          for (int s = 0; s < kstages; ++s) {
            constexpr int kh = Cfg::kSK;
            mbar_wait(&empty[slot], phase ^ 1);
            uint8_t* st = stage_base + slot * Cfg::kStageBytes;
            if constexpr (kAres) {
              mbar_arrive_expect_tx(&full[slot], kh * Cfg::kBBytesPerK);
            } else {
              mbar_arrive_expect_tx(&full[slot], kh * (Cfg::kABytesPerK + Cfg::kBBytesPerK));
#pragma unroll
              for (int kk = 0; kk < kh; ++kk)
                bulk_g2s(st + kk * Cfg::kABytesPerK, a_src + (size_t)((s * Cfg::kSK + kk) % a_ksteps) * Cfg::kABytesPerK,
                         Cfg::kABytesPerK, &full[slot]);
              st += Cfg::kSK * Cfg::kABytesPerK;
            }
            bulk_g2s(st, b_src + (size_t)s * Cfg::kSK * Cfg::kBBytesPerK, kh * Cfg::kBBytesPerK, &full[slot]);
            if (++slot == nst) { slot = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }

  // --------------------------------------------------------------- consumers (2 warpgroups)
  setmaxnreg_inc<232>();
  const int wg = warp >> 2;
  const int g = lane >> 2, q = lane & 3;
  // this thread's accumulator rows in its tile: row0 + 64 mh and row0 + 64 mh + 8 for m64 block mh < kMH
  const int row0 = (kAres ? 0 : wg * 64) + (warp & 3) * 16 + g;
  float accm[Cfg::kMH][NCH][BN / 2];
  uint32_t slot = 0, phase = 0, it = 0;
  // kAres: this warpgroup's n-th epilogue waits until the partner has passed the turn n - wg times (warpgroup 0 starts)
  uint32_t epis = 0;
  auto wait_turn = [&]() { mbar_wait(&turn[wg], (epis & 1) ^ (wg ^ 1)); };
  auto pass_turn = [&]() { mbar_arrive(&turn[wg ^ 1]); ++epis; };
  for (int item = blockIdx.x; item < nitems; item += gridDim.x, ++it) {
    const int tile = kAres ? 2 * item + wg : item / ngroups;
    if constexpr (kAres) {
      mbar_wait(a_full, it & 1);
      if (tile >= ntiles) {
        // the pair has one tile: step through the same barrier phases as the partner warpgroup without MMAs or stores
        // (waiting on `full` keeps these arrivals from running ahead into the slot's next phase)
        for (int gi = 0; gi < gper; ++gi) {
          for (int s = 0; s < kstages; ++s) {
            mbar_wait(&full[slot], phase);
            mbar_arrive(&empty[slot]);
            if (++slot == nst) { slot = 0; phase ^= 1; }
          }
          wait_turn();
          pass_turn();
        }
        mbar_arrive(a_empty);
        continue;
      }
    }
    for (int gi = 0; gi < gper; ++gi) {
      const int grp = kAres ? gi : item % ngroups;
      uint32_t prev = 0;
      for (int s = 0; s < kstages; ++s) {
        mbar_wait(&full[slot], phase);
        const uint32_t st = smem_u32(stage_base + slot * Cfg::kStageBytes);
        const uint32_t sb = kAres ? st : st + Cfg::kSK * Cfg::kABytesPerK;
#pragma unroll
        for (int mh = 0; mh < Cfg::kMH; ++mh)
#pragma unroll
          for (int j = 0; j < NCH; ++j) wgmma_fence_regs(accm[mh][j]);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < Cfg::kSK; ++kk) {
          const uint32_t sa = kAres ? smem_u32(a_res) + wg * Cfg::kATileBytes +
                                          ((s * Cfg::kSK + kk) % a_ksteps) * Cfg::kABytesPerK
                                    : st + kk * Cfg::kABytesPerK;
#pragma unroll
          for (int mh = 0; mh < Cfg::kMH; ++mh) {
            const uint64_t adesc = make_kc16_desc(sa + (kAres ? 64 * mh : 64 * wg) * 16, kTileM * 16, 128);
#pragma unroll
            for (int j = 0; j < NCH; ++j) {
              const uint64_t bdesc = make_kc16_desc(sb + kk * Cfg::kBBytesPerK + j * BN * 16, Cfg::kNI * 16, 128);
              wgmma_bn<BN>(accm[mh][j], adesc, bdesc, (s | kk) != 0);
            }
          }
        }
        wgmma_commit();
#pragma unroll
        for (int mh = 0; mh < Cfg::kMH; ++mh)
#pragma unroll
          for (int j = 0; j < NCH; ++j) wgmma_fence_regs(accm[mh][j]);
        // the previous stage's MMAs are complete once at most this stage's group is in flight: hand it back
        wgmma_wait<1>();
        if (s > 0) mbar_arrive(&empty[prev]);
        prev = slot;
        if (++slot == nst) { slot = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int mh = 0; mh < Cfg::kMH; ++mh)
#pragma unroll
        for (int j = 0; j < NCH; ++j) wgmma_fence_regs(accm[mh][j]);
      mbar_arrive(&empty[prev]);
      if (kAres && gi + 1 == gper) mbar_arrive(a_empty);   // the last group's MMAs have read A

      // ----------------------------------------------------------- epilogue (fragment: row, 2 adjacent columns)
      if constexpr (kAres) wait_turn();
      if constexpr (EPI == EPI_QKV) {
        __nv_bfloat16* obase = out_img + (size_t)tile * kTileM * out_chunks * 8;
#pragma unroll
        for (int mh = 0; mh < Cfg::kMH; ++mh)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = row0 + 64 * mh + 8 * h;
#pragma unroll
            for (int j = 0; j < NCH; ++j)
#pragma unroll
              for (int jj = 0; jj < BN / 8; ++jj) {
                const int col = grp * Cfg::kNI + j * BN + jj * 8 + 2 * q;
                *reinterpret_cast<uint32_t*>(obase + ((size_t)(col >> 3) * kTileM + row) * 8 + (col & 7)) =
                    pack_bf16x2(accm[mh][j][jj * 4 + 2 * h], accm[mh][j][jj * 4 + 2 * h + 1]);
              }
          }
        if constexpr (kAres) pass_turn();   // the stores are issued; they drain under the partner's MMAs
      } else {
        row_epilogue<BN, NCH>(accm[0], tile, row0, q, s_vec, epi);   // one m64 block per warpgroup
      }
    }
    if (flow.flags) {   // the tile's stores are done
      consumer_bar_sync();
      if (threadIdx.x == 0) tile_done(flow, item);
    }
  }
  pdl_wait();
}

// =====================================================================================
// FFN with the hidden activation on the SM
// =====================================================================================
// out = relu(xb W1 + b1) W2 + b2 + x for one 128-token tile per work item, over all of the filter's 128-unit chunks.
// The tile's xb (A) image is loaded once and stays resident; warpgroup w owns tile rows [64 w, 64 w + 64).  Per chunk
// c each consumer warpgroup
//   1. computes H = xb W1[:, c] with m64n128k16 wgmmas over the 18 k-steps (the W1 image holds chunk c as one
//      contiguous [36][128][8] group),
//   2. turns H into bf16(relu(H + b1)) in registers, packed straight into the A fragments of the next step (for
//      hidden k-step kk: pack(d[8kk + 0..1]), pack(d[8kk + 2..3]), pack(d[8kk + 4..5]), pack(d[8kk + 6..7])),
//   3. accumulates that times W2's rows of chunk c (k-steps [8c, 8c + 8) of the [ff/8][288][8] image) with register-A
//      m64n144k16 wgmmas into the 288-wide fp32 accumulators,
// and the tile ends with the row epilogue.  The producer streams W1 group c and then W2's k-steps of c through one
// ring of 9216-byte stages (two W1 k-steps or one W2 k-step each).  A W1 stage leaves 1 KB free: the chunk's last W1
// stage also brings the chunk's 128 b1 values there, and the consumers hand that stage back only after step 2 has
// read them.  (Held in the first W1 stage, b1 would stall the producer before this chunk's last W2 stage, which
// reuses that slot; the last W1 stage's slot is not needed again until the next chunk.)
//
// The forward launches the kernel twice per layer, over the first and the second half of the tiles, because each of
// the forward's five launches per layer ends on a captured stage.  Each tile runs the whole filter once; its first
// MMA starts from zero, so every output element sees the same k16 MMAs in the same order on one fp32 accumulator
// wherever the tiles are split, and the hidden values come from the same instruction shape, K order, bias, ReLU and
// rounding as a separate up-projection would give.  kHid: the hidden activation is also stored to `hid` as a bf16
// operand image [tile][ff/8][128][8] (debug capture).
struct FfnCfg {
  static constexpr int kUpK = kDP / 16;                   // up-projection k-steps per chunk
  static constexpr int kDownK = kFFChunk / 16;            // down-projection k-steps per chunk
  static constexpr int kABytesPerK = 2 * kTileM * 16;     // 4096
  static constexpr int kW1Bytes = 2 * kFFChunk * 16;      // one W1 k-step: 4096
  static constexpr int kW2Bytes = 2 * kDP * 16;           // one W2 k-step: 9216
  static constexpr int kStageBytes = kW2Bytes;            // two W1 k-steps or one W2 k-step
  static constexpr int kB1Off = 2 * kW1Bytes;             // a chunk's b1 in its last W1 stage
  static constexpr int kB1Bytes = kFFChunk * 4;
  static constexpr int kStages = 16;
  static constexpr int kATileBytes = kUpK * kABytesPerK;  // the resident xb tile
  static constexpr int kBarBytes = 512;
  static constexpr int kVecBytes = 3 * kDP * 4;           // row epilogue: bias, LayerNorm gamma, beta (fp32)
  // the xb tile, the ring, the mbarriers, the row vectors
  static constexpr int kSmemBytes = kATileBytes + kStages * kStageBytes + kBarBytes + kVecBytes;
  static constexpr int kThreads = 384;
  static_assert(kSmemBytes <= 232448, "over the sm_90 opt-in shared memory per block");
  static_assert((2 * kStages + 2) * 8 <= kBarBytes, "the mbarriers (full, empty, a_full, a_empty) fit");
  static_assert(kB1Off + kB1Bytes <= kStageBytes && kUpK % 2 == 0, "a stage holds two W1 k-steps and b1");
};

template <bool kHid>
__global__ void __launch_bounds__(384, 1)
ffn_gemm_kernel(const __nv_bfloat16* __restrict__ xb_img, const __nv_bfloat16* __restrict__ w1_img,
                const float* __restrict__ b1, const __nv_bfloat16* __restrict__ w2_img, int ff, int tile_begin,
                int tile_end, __nv_bfloat16* __restrict__ hid, RowEpi epi, TileFlow flow) {
  using Cfg = FfnCfg;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* a_res = smem;
  uint8_t* stage_base = smem + Cfg::kATileBytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(stage_base + Cfg::kStages * Cfg::kStageBytes);
  uint64_t* empty = full + Cfg::kStages;
  uint64_t* a_full = empty + Cfg::kStages;
  uint64_t* a_empty = a_full + 1;
  float* s_vec = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(full) + Cfg::kBarBytes);   // [3][kDP]
  const int nch = ff / kFFChunk;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  row_vectors_to_smem(s_vec, epi);
  if (threadIdx.x == 0) {
    for (int i = 0; i < Cfg::kStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 256);   // every consumer thread
    }
    mbar_init(a_full, 1);
    mbar_init(a_empty, 256);
    mbar_fence_init();
  }
  __syncthreads();
  pdl_launch_dependents();

  if (warp >= 8) {
    // ------------------------------------------------------------- producer
    setmaxnreg_dec<24>();
    if (warp == 8 && lane == 0) {
      uint32_t slot = 0, phase = 0, it = 0;
      // one stage: `bytes` from src, and b1_bytes (0 or the chunk's b1) from b1_src behind them
      auto stage = [&](const uint8_t* src, uint32_t bytes, const float* b1_src, uint32_t b1_bytes) {
        mbar_wait(&empty[slot], phase ^ 1);
        uint8_t* st = stage_base + slot * Cfg::kStageBytes;
        mbar_arrive_expect_tx(&full[slot], bytes + b1_bytes);
        bulk_g2s(st, src, bytes, &full[slot]);
        if (b1_bytes) bulk_g2s(st + Cfg::kB1Off, b1_src, b1_bytes, &full[slot]);
        if (++slot == Cfg::kStages) { slot = 0; phase ^= 1; }
      };
      for (int tile = tile_begin + blockIdx.x; tile < tile_end; tile += gridDim.x, ++it) {
        // the tile is in place before its xb copy; the row epilogue's residual loads follow this acquire through
        // a_full (arrive.expect_tx here, the consumers' wait there)
        tile_wait(flow, tile);
        fence_proxy_async();
        mbar_wait(a_empty, (it & 1) ^ 1);
        mbar_arrive_expect_tx(a_full, Cfg::kATileBytes);
        bulk_g2s(a_res, reinterpret_cast<const uint8_t*>(xb_img) + (size_t)tile * Cfg::kATileBytes, Cfg::kATileBytes,
                 a_full);
        for (int c = 0; c < nch; ++c) {
          const uint8_t* w1 = reinterpret_cast<const uint8_t*>(w1_img) + (size_t)c * Cfg::kUpK * Cfg::kW1Bytes;
          for (int s = 0; s < Cfg::kUpK / 2; ++s)
            stage(w1 + (size_t)s * 2 * Cfg::kW1Bytes, 2 * Cfg::kW1Bytes, b1 + c * kFFChunk,
                  s + 1 == Cfg::kUpK / 2 ? Cfg::kB1Bytes : 0);
          const uint8_t* w2 = reinterpret_cast<const uint8_t*>(w2_img) + (size_t)c * Cfg::kDownK * Cfg::kW2Bytes;
          for (int kk = 0; kk < Cfg::kDownK; ++kk) stage(w2 + (size_t)kk * Cfg::kW2Bytes, Cfg::kW2Bytes, nullptr, 0);
        }
      }
    }
    return;
  }

  // --------------------------------------------------------------- consumers (2 warpgroups)
  setmaxnreg_inc<240>();
  const int wg = warp >> 2;
  const int g = lane >> 2, q = lane & 3;
  const int row0 = wg * 64 + (warp & 3) * 16 + g;   // this thread's accumulator rows: row0, row0 + 8
  const uint32_t a_base = smem_u32(a_res) + wg * 64 * 16;
  float acc[2][kNC / 2];          // out[:, 0..287]
  float hacc[kFFChunk / 2];       // H of the current chunk
  uint32_t slot = 0, phase = 0, it = 0;
  auto next_slot = [&]() { if (++slot == Cfg::kStages) { slot = 0; phase ^= 1; } };
  for (int tile = tile_begin + blockIdx.x; tile < tile_end; tile += gridDim.x, ++it) {
    mbar_wait(a_full, it & 1);
    for (int c = 0; c < nch; ++c) {
      // ---- 1. H = xb W1[:, c]
      uint32_t prev = 0;
#pragma unroll
      for (int s = 0; s < Cfg::kUpK / 2; ++s) {
        mbar_wait(&full[slot], phase);
        const uint32_t st = smem_u32(stage_base + slot * Cfg::kStageBytes);
        // H starts at the chunk's first wgmma (scale-d 0, written only), so it is not live between chunks
        if (s > 0) wgmma_fence_regs(hacc);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 2; ++kk) {
          const uint64_t adesc = make_kc16_desc(a_base + (2 * s + kk) * Cfg::kABytesPerK, kTileM * 16, 128);
          const uint64_t bdesc = make_kc16_desc(st + kk * Cfg::kW1Bytes, kFFChunk * 16, 128);
          if (s == 0 && kk == 0) wgmma_m64n128k16_first(hacc, adesc, bdesc);
          else wgmma_m64n128k16(hacc, adesc, bdesc, 1);
        }
        wgmma_commit();
        wgmma_fence_regs(hacc);
        wgmma_wait<1>();
        if (s > 0) mbar_arrive(&empty[prev]);
        prev = slot;
        next_slot();
      }
      wgmma_wait<0>();
      wgmma_fence_regs(hacc);
      if (c + 1 == nch) mbar_arrive(a_empty);   // the item's last MMAs on xb have completed

      // ---- 2. bf16(relu(H + b1)) as A fragments: fragment (kk, i) holds hidden columns 16 kk + 8 (i >> 1) + 2q, +1
      // of row row0 + 8 (i & 1), i.e. accumulator elements 8 kk + 2 i, + 1.  b1 is in the last W1 stage (prev).
      uint32_t af[Cfg::kDownK][4];
      const float* bc = reinterpret_cast<const float*>(stage_base + prev * Cfg::kStageBytes + Cfg::kB1Off) + 2 * q;
#pragma unroll
      for (int kk = 0; kk < Cfg::kDownK; ++kk)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 b = *reinterpret_cast<const float2*>(bc + 16 * kk + 8 * (i >> 1));
          af[kk][i] = pack_bf16x2(fmaxf(hacc[8 * kk + 2 * i] + b.x, 0.f), fmaxf(hacc[8 * kk + 2 * i + 1] + b.y, 0.f));
        }
      mbar_arrive(&empty[prev]);
      if constexpr (kHid) {
        __nv_bfloat16* hb = hid + (size_t)tile * kTileM * ff + (size_t)row0 * 8 + 2 * q;
#pragma unroll
        for (int kk = 0; kk < Cfg::kDownK; ++kk)
#pragma unroll
          for (int i = 0; i < 4; ++i)
            *reinterpret_cast<uint32_t*>(hb + ((size_t)(c * 16 + 2 * kk + (i >> 1)) * kTileM + 8 * (i & 1)) * 8) =
                af[kk][i];
      }

      // ---- 3. acc += bf16(H) W2[c rows, :]
#pragma unroll
      for (int kk = 0; kk < Cfg::kDownK; ++kk) {
        mbar_wait(&full[slot], phase);
        const uint32_t st = smem_u32(stage_base + slot * Cfg::kStageBytes);
        wgmma_fence_regs(acc[0]);
        wgmma_fence_regs(acc[1]);
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < 2; ++j)
          wgmma_m64n144k16_rs(acc[j], af[kk], make_kc16_desc(st + j * kNC * 16, kDP * 16, 128), c != 0 || kk != 0);
        wgmma_commit();
        wgmma_fence_regs(acc[0]);
        wgmma_fence_regs(acc[1]);
        wgmma_wait<1>();
        if (kk > 0) {
          wgmma_fence_regs(af[kk - 1]);   // read by the group that just completed
          mbar_arrive(&empty[prev]);
        }
        prev = slot;
        next_slot();
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc[0]);
      wgmma_fence_regs(acc[1]);
      wgmma_fence_regs(af[Cfg::kDownK - 1]);
      mbar_arrive(&empty[prev]);
    }

    row_epilogue<kNC, 2, false>(acc, tile, row0, q, s_vec, epi);
    if (flow.flags) {
      consumer_bar_sync();
      if (threadIdx.x == 0) tile_done(flow, tile);
    }
  }
  pdl_wait();
}

// =====================================================================================
// banded attention (mma.sync m16n8k16 bf16, online softmax over 16-key tiles)
// =====================================================================================
// One CTA per (window, head).  K and V rows of the window are staged in shared memory
// (row stride 152 bf16 = 304 B: conflict-free for the 32-bit K-fragment loads and for
// ldmatrix.trans on V); Q fragments are read straight from the global operand image.
// FLOP share of this kernel is ~1-4 % of the model, so the legacy warp-level MMA path
// is used here on purpose.
constexpr int kAttStride = 144;              // dense rows; 16-byte chunks are rotated by the row index
constexpr int kAttChunks = kDHP / 8;         // 18 chunks per row

__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0,
                                               uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void ldmatrix_x2_trans(uint32_t& r0, uint32_t& r1, uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0, %1}, [%2];"
               : "=r"(r0), "=r"(r1)
               : "r"(addr));
}

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr)
               : "memory");
}

// element (token, col) of a bf16 operand image with `chunks` 8-wide chunks per row
__device__ __forceinline__ size_t img_off(int tok, int col, int chunks) {
  const int tile = tok / kTileM, r = tok % kTileM;
  return (((size_t)tile * chunks + (col >> 3)) * kTileM + r) * 8 + (col & 7);
}

// Shared-memory K/V rows are dense (288 B) with the 18 16-byte chunks of row r rotated by r
// (physical chunk = (c + r) mod 18): 8 consecutive rows then hit 8 distinct 16-byte bank groups
// (48 r mod 128 is a permutation of the multiples of 16), which keeps both the 32-bit K-fragment
// loads and ldmatrix.trans on V conflict-free without padding -- 73.7 KB per CTA, 3 CTAs per SM.
__device__ __forceinline__ int att_rot(int chunk, int rowmod) {
  const int t = chunk + rowmod;
  return t >= kAttChunks ? t - kAttChunks : t;
}

// The banded online-softmax attention of one 16-row query block [i0, i0 + 16) of a window against its K and V rows in
// shared memory (the rotated layout above, zero beyond L up to a multiple of 16), called by a whole warp.  qa holds the
// block's Q as mma.sync A fragments, one per 16-column k-step (zero for rows >= L).  The bf16 output of the rows < L
// goes to columns [head * kDHP, head * kDHP + kDHP) of the attention image, whose window starts at token tok0.  A
// block's arithmetic does not depend on which warp runs it, so both attention kernels give the same bits.
__device__ __forceinline__ void attend_block(const uint32_t (&qa)[kDHP / 16][4], const __nv_bfloat16* sK,
                                             const __nv_bfloat16* sV, int i0, int L, int band,
                                             __nv_bfloat16* __restrict__ att, int tok0, int head) {
  const int lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  constexpr float kLog2e = 1.4426950408889634f;
  constexpr int kChunkElems = kTileM * 8;
  const int r0 = i0 + g, r1 = i0 + g + 8;
  float o[kDHP / 8][4];
#pragma unroll
  for (int nt = 0; nt < kDHP / 8; ++nt) { o[nt][0] = o[nt][1] = o[nt][2] = o[nt][3] = 0.f; }
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

  int jlo = i0 - band; if (jlo < 0) jlo = 0; jlo &= ~15;
  int jhi = i0 + 15 + band + 1; if (jhi > L) jhi = L;
  for (int j0 = jlo; j0 < jhi; j0 += 16) {
    // S tile 16 x 16 = two n-tiles of 8 keys; two partial accumulators per n-tile shorten the
    // dependent HMMA chains (4 independent chains instead of 2)
    float s[2][4], s2[2][4];
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
      s2[nt][0] = s2[nt][1] = s2[nt][2] = s2[nt][3] = 0.f;
    }
    const int krow0 = j0 + g, krow1 = j0 + 8 + g;
    const __nv_bfloat16* kr0 = sK + (size_t)krow0 * kAttStride + 2 * t;
    const __nv_bfloat16* kr1 = sK + (size_t)krow1 * kAttStride + 2 * t;
    const int km0 = krow0 % kAttChunks, km1 = krow1 % kAttChunks;
#pragma unroll
    for (int ks = 0; ks < kDHP / 16; ++ks) {
      const uint32_t a0 = *reinterpret_cast<const uint32_t*>(kr0 + att_rot(2 * ks, km0) * 8);
      const uint32_t a1 = *reinterpret_cast<const uint32_t*>(kr0 + att_rot(2 * ks + 1, km0) * 8);
      const uint32_t c0 = *reinterpret_cast<const uint32_t*>(kr1 + att_rot(2 * ks, km1) * 8);
      const uint32_t c1 = *reinterpret_cast<const uint32_t*>(kr1 + att_rot(2 * ks + 1, km1) * 8);
      if (ks & 1) {
        mma_bf16_16816(s2[0], qa[ks], a0, a1);
        mma_bf16_16816(s2[1], qa[ks], c0, c1);
      } else {
        mma_bf16_16816(s[0], qa[ks], a0, a1);
        mma_bf16_16816(s[1], qa[ks], c0, c1);
      }
    }
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) s[nt][e] += s2[nt][e];
    // mask: |i - j| <= band and j < L  (tf.where(mask, logits, -1e9): exp underflows to 0)
    float tmax0 = -INFINITY, tmax1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = (e < 2) ? r0 : r1;
        const int j = j0 + nt * 8 + 2 * t + (e & 1);
        const int dlt = i - j;
        const bool ok = (j < L) && (dlt <= band) && (dlt >= -band);
        s[nt][e] = ok ? s[nt][e] : -INFINITY;
      }
      tmax0 = fmaxf(tmax0, fmaxf(s[nt][0], s[nt][1]));
      tmax1 = fmaxf(tmax1, fmaxf(s[nt][2], s[nt][3]));
    }
    tmax0 = fmaxf(tmax0, __shfl_xor_sync(0xffffffffu, tmax0, 1));
    tmax0 = fmaxf(tmax0, __shfl_xor_sync(0xffffffffu, tmax0, 2));
    tmax1 = fmaxf(tmax1, __shfl_xor_sync(0xffffffffu, tmax1, 1));
    tmax1 = fmaxf(tmax1, __shfl_xor_sync(0xffffffffu, tmax1, 2));
    const float mn0 = fmaxf(m0, tmax0), mn1 = fmaxf(m1, tmax1);
    // rows with no valid key yet keep m = -inf; use 0 as the subtraction base there
    const float base0 = mn0 == -INFINITY ? 0.f : mn0, base1 = mn1 == -INFINITY ? 0.f : mn1;
    const float sc0 = exp2f((m0 - base0) * kLog2e), sc1 = exp2f((m1 - base1) * kLog2e);
    m0 = mn0; m1 = mn1;
    float ps0 = 0.f, ps1 = 0.f;
    uint32_t pa[4];
    {
      float p[2][4];
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) {
        p[nt][0] = exp2f((s[nt][0] - base0) * kLog2e);
        p[nt][1] = exp2f((s[nt][1] - base0) * kLog2e);
        p[nt][2] = exp2f((s[nt][2] - base1) * kLog2e);
        p[nt][3] = exp2f((s[nt][3] - base1) * kLog2e);
        ps0 += p[nt][0] + p[nt][1];
        ps1 += p[nt][2] + p[nt][3];
      }
      // C fragments of the two n-tiles form the A fragment of one 16-key k-step
      pa[0] = pack_bf16x2(p[0][0], p[0][1]);
      pa[1] = pack_bf16x2(p[0][2], p[0][3]);
      pa[2] = pack_bf16x2(p[1][0], p[1][1]);
      pa[3] = pack_bf16x2(p[1][2], p[1][3]);
    }
    l0 = l0 * sc0 + ps0;
    l1 = l1 * sc1 + ps1;
    // O = O * scale + P V
    const int vrow = j0 + (lane & 15);
    const int vm = vrow % kAttChunks;
    const uint32_t vbase = smem_u32(sV + (size_t)vrow * kAttStride);
#pragma unroll
    for (int nt = 0; nt < kDHP / 8; ++nt) {
      o[nt][0] *= sc0; o[nt][1] *= sc0; o[nt][2] *= sc1; o[nt][3] *= sc1;
      uint32_t b0, b1;
      ldmatrix_x2_trans(b0, b1, vbase + att_rot(nt, vm) * 16);
      mma_bf16_16816(o[nt], pa, b0, b1);
    }
  }
  // normalise (row sums live in the quad) and store bf16 to the attention operand image
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float inv0 = 1.f / l0, inv1 = 1.f / l1;
  __nv_bfloat16* o0 = att + img_off(tok0 + (r0 < L ? r0 : 0), head * kDHP + 2 * t, kDP / 8);
  __nv_bfloat16* o1 = att + img_off(tok0 + (r1 < L ? r1 : 0), head * kDHP + 2 * t, kDP / 8);
#pragma unroll
  for (int nt = 0; nt < kDHP / 8; ++nt) {
    if (r0 < L)
      *reinterpret_cast<uint32_t*>(o0 + nt * kChunkElems) = pack_bf16x2(o[nt][0] * inv0, o[nt][1] * inv0);
    if (r1 < L)
      *reinterpret_cast<uint32_t*>(o1 + nt * kChunkElems) = pack_bf16x2(o[nt][2] * inv1, o[nt][3] * inv1);
  }
}

__global__ void __launch_bounds__(128, 3)
band_attention_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ att,
                      int L, int Lw, int win, int nwindows) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int w = blockIdx.x >> 1;
  const int head = blockIdx.x & 1;
  if (w >= nwindows) return;
  const int Lp = (L + 15) & ~15;  // key rows padded to a multiple of 16 (zero filled)
  __nv_bfloat16* sK = reinterpret_cast<__nv_bfloat16*>(smem);
  __nv_bfloat16* sV = sK + (size_t)Lp * kAttStride;
  constexpr int qkv_chunks = kQKVN / 8;  // 108
  const int kcol = (2 + head) * kDHP, vcol = (4 + head) * kDHP, qcol = head * kDHP;
  const int tok0 = w * Lw;   // windows start every Lw tokens in the flattened layout (Lw >= L)

  // stage K, V with cp.async: thread = row (coalesced 16 B chunks across the warp), no divisions
  for (int row = threadIdx.x; row < Lp; row += blockDim.x) {
    const int rm = row % kAttChunks;
    __nv_bfloat16* dk = sK + (size_t)row * kAttStride;
    __nv_bfloat16* dv = sV + (size_t)row * kAttStride;
    if (row < L) {
      const int tok = tok0 + row;
      const size_t base = ((size_t)(tok / kTileM) * qkv_chunks) * kTileM * 8 + (size_t)(tok % kTileM) * 8;
      const __nv_bfloat16* gk = qkv + base + (size_t)(kcol >> 3) * kTileM * 8;
      const __nv_bfloat16* gv = qkv + base + (size_t)(vcol >> 3) * kTileM * 8;
#pragma unroll
      for (int ch = 0; ch < kAttChunks; ++ch) {
        const int pc = att_rot(ch, rm) * 8;
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dk + pc)),
                     "l"(gk + (size_t)ch * kTileM * 8) : "memory");
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dv + pc)),
                     "l"(gv + (size_t)ch * kTileM * 8) : "memory");
      }
    } else {
#pragma unroll
      for (int ch = 0; ch < kAttChunks; ++ch) {
        *reinterpret_cast<uint4*>(dk + ch * 8) = make_uint4(0, 0, 0, 0);
        *reinterpret_cast<uint4*>(dv + ch * 8) = make_uint4(0, 0, 0, 0);
      }
    }
  }
  asm volatile("cp.async.commit_group;" ::: "memory");

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int band = win > 0 ? win : L;  // attn_win_size None/0 => full attention

  // Q fragments for 9 k-steps: rows i0+g, i0+g+8 (zero beyond L), straight from global.
  // In the operand image a row's k-chunks are kTileM*8 elements apart, so every fragment address is
  // the row base plus a compile-time constant (no per-load index arithmetic).
  constexpr int kChunkElems = kTileM * 8;
  uint32_t qa[kDHP / 16][4];
  auto load_q = [&](int qb) {
    const int r0 = qb * 16 + g, r1 = r0 + 8;
    const __nv_bfloat16* q0 = qkv + img_off(tok0 + (r0 < L ? r0 : 0), qcol + 2 * t, qkv_chunks);
    const __nv_bfloat16* q1 = qkv + img_off(tok0 + (r1 < L ? r1 : 0), qcol + 2 * t, qkv_chunks);
#pragma unroll
    for (int ks = 0; ks < kDHP / 16; ++ks) {
      const uint32_t v0 = __ldg(reinterpret_cast<const uint32_t*>(q0 + (2 * ks) * kChunkElems));
      const uint32_t v1 = __ldg(reinterpret_cast<const uint32_t*>(q1 + (2 * ks) * kChunkElems));
      const uint32_t v2 = __ldg(reinterpret_cast<const uint32_t*>(q0 + (2 * ks + 1) * kChunkElems));
      const uint32_t v3 = __ldg(reinterpret_cast<const uint32_t*>(q1 + (2 * ks + 1) * kChunkElems));
      qa[ks][0] = r0 < L ? v0 : 0u;
      qa[ks][1] = r1 < L ? v1 : 0u;
      qa[ks][2] = r0 < L ? v2 : 0u;
      qa[ks][3] = r1 < L ? v3 : 0u;
    }
  };
  if (warp * 16 < L) load_q(warp);
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();

  for (int qb = warp; qb * 16 < L; qb += 4) {
    if (qb != warp) load_q(qb);
    attend_block(qa, sK, sV, qb * 16, L, band, att, tok0, head);
  }
}

// =====================================================================================
// q/k/v projection and attention of one window-aligned tile on the SM
// =====================================================================================
// In the window-aligned layout (Lw == kTileM, L <= 128) a tile is one window, and the band never leaves it, so the
// attention of a tile needs only that tile's q/k/v.  One work item is one tile in [tile_begin, tile_end).  Its xb (A)
// image is loaded once and stays resident; warpgroup w owns tile rows [64 w, 64 w + 64).  Per head h each consumer
// warpgroup
//   1. runs the k_h and then the v_h n-group of the q/k/v weights (split-bf16, 36 k-steps: W_hi then W_lo, A k-step
//      (s * kSK + kk) % 18, as gemm_kernel's EPI_QKV) and stores each, rounded to bf16, into sK / sV in the attention's
//      rotated layout, zero for rows >= L.  A comes from registers: at the start of each group every warp loads its
//      16 rows of the 18 A k-steps from the resident xb tile with ldmatrix, in the m16n8k16 A layout the register-A
//      wgmma takes, and the group's 36 wgmmas read B alone from shared memory.  Shared-memory A operands were read
//      once per wgmma, twice per group (W_hi and W_lo); register A halves the group's A reads from shared memory, and
//      the wgmma arithmetic does not depend on where A comes from,
//   2. runs the q_h n-group and keeps it in registers as mma.sync A fragments (the m64n144 accumulator of warp w & 3
//      covers its 16 rows in the m16n8k16 C layout: k-step ks is pack(d[8ks..+1]), pack(d[8ks+2..+3]),
//      pack(d[8ks+4..+5]), pack(d[8ks+6..+7]), the mapping the FFN uses for its hidden activation),
//   3. meets its partner on named barrier 1 (the band crosses row 64, so both halves of K and V must be in place),
//   4. runs attend_block for the warp's own 16-row query block.
// Before a warpgroup next writes sK / sV it meets its partner again, so no warp still reads the previous head's K and
// V; the wgmmas of the next group are already under way by then.  The producer streams the groups in the order k_h0,
// v_h0, q_h0, k_h1, v_h1, q_h1 (groups 2, 4, 0, 3, 5, 1 of the [q_h0|q_h1|k_h0|k_h1|v_h0|v_h1] weight image) through
// a ring of four 18432-byte stages (four k-steps of one group), and the next tile's xb loads once q_h1's MMAs have read
// it, under head 1's attention.
//
// Every q/k/v value is the accumulator gemm_kernel<144, 1, EPI_QKV, true> computes (same wgmma shape, same K order)
// rounded the same way, and attend_block is band_attention_kernel's, so the attention image is the same bit for bit.
// kQkv: the q/k/v accumulators are also stored to the q/k/v operand image as the EPI_QKV epilogue does (debug capture).
struct QkvAttCfg {
  static constexpr int kAK = kDP / 16;                    // A k-steps: 18
  // Ring shape: the same 72 KB as eight stages of two k-steps, but each stage's wgmma run, commit, wait and release
  // covers four k-steps, so a warpgroup synchronises half as often per weight byte.  On an H100 SXM at 700 W that
  // made the kernel (A still from shared memory) about 3 % faster at the bench workload; six k-steps in three stages
  // and a second stage group in flight per warpgroup (wait_group 2) were not faster.
  static constexpr int kSK = 4;                           // k-steps per stage
  static constexpr int kGroupStages = 2 * kAK / kSK;      // split-bf16 weights: 36 k-steps per group, 9 stages
  static constexpr int kABytesPerK = 2 * kTileM * 16;     // 4096
  static constexpr int kBBytesPerK = 2 * kQKVGroup * 16;  // 4608
  static constexpr int kStageBytes = kSK * kBBytesPerK;   // 18432
  static constexpr int kGroupBytes = 2 * kAK * kBBytesPerK;
  static constexpr int kStages = 4;
  static constexpr int kATileBytes = kAK * kABytesPerK;   // the resident xb tile: 72 KB
  static constexpr int kKVBytes = kTileM * kAttStride * 2;  // K or V of one head: 36 KB
  static constexpr int kBarBytes = 256;
  // the xb tile, sK, sV, the ring, the mbarriers
  static constexpr int kSmemBytes = kATileBytes + 2 * kKVBytes + kStages * kStageBytes + kBarBytes;
  static constexpr int kThreads = 384;
  static_assert(kSmemBytes <= 232448, "over the sm_90 opt-in shared memory per block");
  static_assert((2 * kStages + 2) * 8 <= kBarBytes, "the mbarriers (full, empty, a_full, a_empty) fit");
  static_assert((2 * kAK) % kSK == 0, "every stage holds kSK k-steps of one group");
  static_assert(kQKVGroup == kDHP && kQKVN == 6 * kQKVGroup, "one n-group is one head's q, k or v");
};

// the n-group of the q/k/v weight image that item step i (0..5) of a tile runs: k_h0, v_h0, q_h0, k_h1, v_h1, q_h1
__device__ __forceinline__ int qkv_att_group(int i) {
  const int h = i / 3, part = i % 3;
  return part == 0 ? 2 + h : part == 1 ? 4 + h : h;
}

template <bool kQkv>
__global__ void __launch_bounds__(384, 1)
qkv_attention_kernel(const __nv_bfloat16* __restrict__ xb_img, const __nv_bfloat16* __restrict__ b_img, int L,
                     int win, int tile_begin, int tile_end, __nv_bfloat16* __restrict__ qkv_img,
                     __nv_bfloat16* __restrict__ att, TileFlow flow) {
  using Cfg = QkvAttCfg;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* a_res = smem;
  __nv_bfloat16* sK = reinterpret_cast<__nv_bfloat16*>(smem + Cfg::kATileBytes);
  __nv_bfloat16* sV = reinterpret_cast<__nv_bfloat16*>(smem + Cfg::kATileBytes + Cfg::kKVBytes);
  uint8_t* stage_base = smem + Cfg::kATileBytes + 2 * Cfg::kKVBytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(stage_base + Cfg::kStages * Cfg::kStageBytes);
  uint64_t* empty = full + Cfg::kStages;
  uint64_t* a_full = empty + Cfg::kStages;
  uint64_t* a_empty = a_full + 1;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < Cfg::kStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 256);   // every consumer thread
    }
    mbar_init(a_full, 1);
    mbar_init(a_empty, 256);
    mbar_fence_init();
  }
  __syncthreads();
  pdl_launch_dependents();

  if (warp >= 8) {
    // ------------------------------------------------------------- producer
    setmaxnreg_dec<24>();
    if (warp == 8 && lane == 0) {
      uint32_t slot = 0, phase = 0, it = 0;
      for (int tile = tile_begin + blockIdx.x; tile < tile_end; tile += gridDim.x, ++it) {
        tile_wait(flow, tile);   // the tile's xb is in place before its copy
        fence_proxy_async();
        mbar_wait(a_empty, (it & 1) ^ 1);
        mbar_arrive_expect_tx(a_full, Cfg::kATileBytes);
        bulk_g2s(a_res, reinterpret_cast<const uint8_t*>(xb_img) + (size_t)tile * Cfg::kATileBytes, Cfg::kATileBytes,
                 a_full);
        for (int i = 0; i < 6; ++i) {
          const uint8_t* b_src = reinterpret_cast<const uint8_t*>(b_img) + (size_t)qkv_att_group(i) * Cfg::kGroupBytes;
          for (int s = 0; s < Cfg::kGroupStages; ++s) {
            mbar_wait(&empty[slot], phase ^ 1);
            mbar_arrive_expect_tx(&full[slot], Cfg::kStageBytes);
            bulk_g2s(stage_base + slot * Cfg::kStageBytes, b_src + (size_t)s * Cfg::kStageBytes, Cfg::kStageBytes,
                     &full[slot]);
            if (++slot == Cfg::kStages) { slot = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }

  // --------------------------------------------------------------- consumers (2 warpgroups)
  setmaxnreg_inc<240>();
  const int wg = warp >> 2;
  const int g = lane >> 2, q = lane & 3;
  const int row0 = wg * 64 + (warp & 3) * 16 + g;   // this thread's accumulator rows: row0, row0 + 8
  // ldmatrix.x4 row address of this lane for A k-step 0: matrices (rows 0-7, chunk 0), (rows 8-15, chunk 0),
  // (rows 0-7, chunk 1), (rows 8-15, chunk 1) of the warp's 16 rows, i.e. the m16n8k16 A fragment a0..a3
  const uint32_t a_frag = smem_u32(a_res) +
                          ((lane >> 4) * kTileM + wg * 64 + (warp & 3) * 16 + ((lane >> 3) & 1) * 8 + (lane & 7)) * 16;
  const int band = win > 0 ? win : L;   // attn_win_size None/0 => full attention
  float acc[kQKVGroup / 2];
  uint32_t slot = 0, phase = 0, it = 0;
  for (int tile = tile_begin + blockIdx.x; tile < tile_end; tile += gridDim.x, ++it) {
    mbar_wait(a_full, it & 1);
#pragma unroll 1
    for (int h = 0; h < kHeads; ++h) {
      uint32_t qa[kDHP / 16][4];
#pragma unroll
      for (int part = 0; part < 3; ++part) {
        // ---- acc = xb W[:, group], A from registers: this warp's 16 rows of the 18 A k-steps (each used by the
        // W_hi and the W_lo half of the group)
        uint32_t af[Cfg::kAK][4];
#pragma unroll
        for (int k = 0; k < Cfg::kAK; ++k) ldmatrix_x4(af[k], a_frag + k * Cfg::kABytesPerK);
        uint32_t prev = 0;
#pragma unroll
        for (int s = 0; s < Cfg::kGroupStages; ++s) {
          mbar_wait(&full[slot], phase);
          const uint32_t st = smem_u32(stage_base + slot * Cfg::kStageBytes);
          wgmma_fence_regs(acc);
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < Cfg::kSK; ++kk) {
            const uint64_t bdesc = make_kc16_desc(st + kk * Cfg::kBBytesPerK, kQKVGroup * 16, 128);
            wgmma_m64n144k16_rs(acc, af[(s * Cfg::kSK + kk) % Cfg::kAK], bdesc, (s | kk) != 0);
          }
          wgmma_commit();
          wgmma_fence_regs(acc);
          // the previous stage's MMAs are complete once at most this stage's group is in flight: hand it back
          wgmma_wait<1>();
          if (s > 0) mbar_arrive(&empty[prev]);
          prev = slot;
          if (++slot == Cfg::kStages) { slot = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
#pragma unroll
        for (int k = 0; k < Cfg::kAK; ++k) wgmma_fence_regs(af[k]);   // read by MMAs up to the one just completed
        mbar_arrive(&empty[prev]);
        if (h + 1 == kHeads && part == 2) mbar_arrive(a_empty);   // the item's last reads of xb are done

        const int grp = part == 0 ? 2 + h : part == 1 ? 4 + h : h;   // qkv_att_group(3 h + part)
        if constexpr (kQkv) {   // the EPI_QKV epilogue's stores
          __nv_bfloat16* obase = qkv_img + (size_t)tile * kTileM * (kQKVN / 8) * 8;
#pragma unroll
          for (int hr = 0; hr < 2; ++hr)
#pragma unroll
            for (int jj = 0; jj < kQKVGroup / 8; ++jj) {
              const int col = grp * kQKVGroup + jj * 8 + 2 * q;
              *reinterpret_cast<uint32_t*>(obase + ((size_t)(col >> 3) * kTileM + row0 + 8 * hr) * 8 + (col & 7)) =
                  pack_bf16x2(acc[jj * 4 + 2 * hr], acc[jj * 4 + 2 * hr + 1]);
            }
        }
        if (part < 2) {
          // ---- K or V into shared memory; before K, every warp is done with the previous head's K and V
          if (part == 0) consumer_bar_sync();
          __nv_bfloat16* dst = part == 0 ? sK : sV;
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            const int r = row0 + 8 * hr;
            const int rm = r % kAttChunks;
            __nv_bfloat16* drow = dst + (size_t)r * kAttStride + 2 * q;
#pragma unroll
            for (int jj = 0; jj < kDHP / 8; ++jj)
              *reinterpret_cast<uint32_t*>(drow + att_rot(jj, rm) * 8) =
                  r < L ? pack_bf16x2(acc[jj * 4 + 2 * hr], acc[jj * 4 + 2 * hr + 1]) : 0u;
          }
        } else {
          // ---- Q as A fragments (zero for rows >= L)
          const bool v0 = row0 < L, v1 = row0 + 8 < L;
#pragma unroll
          for (int ks = 0; ks < kDHP / 16; ++ks) {
            qa[ks][0] = v0 ? pack_bf16x2(acc[8 * ks + 0], acc[8 * ks + 1]) : 0u;
            qa[ks][1] = v1 ? pack_bf16x2(acc[8 * ks + 2], acc[8 * ks + 3]) : 0u;
            qa[ks][2] = v0 ? pack_bf16x2(acc[8 * ks + 4], acc[8 * ks + 5]) : 0u;
            qa[ks][3] = v1 ? pack_bf16x2(acc[8 * ks + 6], acc[8 * ks + 7]) : 0u;
          }
        }
      }
      // ---- attention of this warp's query block once both halves of K and V are in place
      consumer_bar_sync();
      const int i0 = warp * 16;
      if (i0 < L) attend_block(qa, sK, sV, i0, L, band, att, tile * kTileM, h);
    }
    if (flow.flags) {
      consumer_bar_sync();
      if (threadIdx.x == 0) tile_done(flow, tile);
    }
  }
  pdl_wait();
}

// =====================================================================================
// head: final LayerNorm -> fc1 -> softmax -> argmax / Phred / ASCII
// =====================================================================================
// Token tile * kTileM + r of head_kernel; sGW, sA, sBj: its shared-memory copies of p.gw8 and p.ab.
__device__ __forceinline__ void head_row(const HeadParams& p, const float* sGW, const float* sA, const float* sBj,
                                         int tile, int r) {
  // logits_j = sum_c ((x_c - mean) * rstd * g_c + b_c) * W_cj + bfc_j
  //          = rstd * (sum_c y_c * (g_c W_cj) - mean_y * A_j) + B_j + bfc_j,   y = x - shift, A_j = sum_c g_c W_cj,
  //            B_j = sum_c b_c W_cj
  // so ONE pass over the row accumulates sum y, sum y^2 and the five sums y * gW_j (the residual image is read once).
  const int tok = tile * kTileM + r;
  if (tok >= p.M) return;
  const int wdw = tok / p.Lw, pos = tok - wdw * p.Lw;
  if (pos >= p.L) return;                       // layout padding row
  const size_t oidx = (size_t)wdw * p.L + pos;  // outputs are dense [B, L]
  const float4* xrow = reinterpret_cast<const float4*>(p.x + (size_t)tile * x_image_elems()) + r;
  // mean / variance are biased, eps = 1e-6 (encoder_stack.py:131-133); 10 loads in flight per batch
  float s1 = 0.f, s2 = 0.f;
  float t[kVocab];
#pragma unroll
  for (int j = 0; j < kVocab; ++j) t[j] = 0.f;
  const float shift = xrow[0].x;
  constexpr int kHB = 10;
  static_assert((kD / 4) % kHB == 0, "head batch");
#pragma unroll 1
  for (int c0 = 0; c0 < kD / 4; c0 += kHB) {
    float4 v[kHB];
#pragma unroll
    for (int u = 0; u < kHB; ++u) v[u] = xrow[(size_t)(c0 + u) * kTileM];
#pragma unroll
    for (int u = 0; u < kHB; ++u) {
      const float ys[4] = {v[u].x - shift, v[u].y - shift, v[u].z - shift, v[u].w - shift};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int col = (c0 + u) * 4 + i;
        s1 += ys[i];
        s2 = fmaf(ys[i], ys[i], s2);
        const float4 w0 = *reinterpret_cast<const float4*>(&sGW[col * 8]);       // two 16-byte broadcast reads per element
        const float w4 = sGW[col * 8 + 4];
        t[0] = fmaf(ys[i], w0.x, t[0]); t[1] = fmaf(ys[i], w0.y, t[1]); t[2] = fmaf(ys[i], w0.z, t[2]);
        t[3] = fmaf(ys[i], w0.w, t[3]); t[4] = fmaf(ys[i], w4, t[4]);
      }
    }
  }
  const float m1 = s1 * (1.f / kD);             // mean of y
  const float rstd = rsqrtf(fmaxf(s2 * (1.f / kD) - m1 * m1, 0.f) + 1e-6f);
  float lg[kVocab];
#pragma unroll
  for (int j = 0; j < kVocab; ++j) lg[j] = rstd * (t[j] - m1 * sA[j]) + sBj[j];   // + fc1 bias in head_finish (networks.py:342)
  head_finish(p, lg, oidx);
}

__global__ void __launch_bounds__(128)
head_kernel(HeadParams p, TileFlow flow) {
  __shared__ __align__(16) float sGW[kD * 8];
  __shared__ float sA[kVocab], sBj[kVocab];
  for (int i = threadIdx.x; i < kD * 2; i += blockDim.x)
    reinterpret_cast<float4*>(sGW)[i] = __ldg(reinterpret_cast<const float4*>(p.gw8) + i);
  if (threadIdx.x < kVocab) { sA[threadIdx.x] = p.ab[threadIdx.x]; sBj[threadIdx.x] = p.ab[8 + threadIdx.x]; }
  if (threadIdx.x == 0) tile_wait(flow, blockIdx.x);   // every thread's residual loads follow it through the barrier
  __syncthreads();
  head_row(p, sGW, sA, sBj, blockIdx.x, threadIdx.x);
  pdl_wait();
}

// =====================================================================================
// launchers
// =====================================================================================
static int g_num_sms = 0;
static int num_sms() {
  if (!g_num_sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_num_sms <= 0) g_num_sms = 132;
  }
  return g_num_sms;
}


template <int BN, int NCH, int EPI, bool kAres>
static cudaError_t gemm_init() {
  return cudaFuncSetAttribute(gemm_kernel<BN, NCH, EPI, kAres>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              GemmCfg<BN, NCH, kAres>::kSmemBytes);
}

cudaError_t kernels_init() {
  cudaError_t e;
  if ((e = gemm_init<kNC, 2, EPI_ROW, false>()) != cudaSuccess) return e;
  if ((e = gemm_init<kNC, 1, EPI_QKV, true>()) != cudaSuccess) return e;
  for (auto fn : {ffn_gemm_kernel<false>, ffn_gemm_kernel<true>})
    if ((e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, FfnCfg::kSmemBytes)) != cudaSuccess)
      return e;
  for (auto fn : {qkv_attention_kernel<false>, qkv_attention_kernel<true>})
    if ((e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, QkvAttCfg::kSmemBytes)) !=
        cudaSuccess)
      return e;
  e = cudaFuncSetAttribute(embed_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(band_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           2 * 256 * kAttStride * 2);
  return e;
}

// kernel<<<grid, threads, smem, st>>>(args...), as a programmatic dependent of the launch before it in the stream when
// `flow` carries flags (the tile flow above).  Such a launch may start before the one it depends on has finished; it
// cannot deadlock on it: a dependent launch starts only once every CTA of the launch before it has issued
// launch_dependents, i.e. is resident or finished, and so every tile a CTA waits for belongs to a CTA that is running
// or done (the chain's launches wait only on the launch just before them).
template <typename... P, typename... A>
static void launch(const TileFlow& flow, void (*kernel)(P...), int grid, int threads, size_t smem, cudaStream_t st,
                   A... args) {
  cudaLaunchAttribute attr{};
  attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr.val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cfg.attrs = flow.flags ? &attr : nullptr;
  cfg.numAttrs = flow.flags ? 1 : 0;
  cudaLaunchKernelEx(&cfg, kernel, args...);   // an error is left for the submission's cudaGetLastError
}

size_t embed_smem_bytes(int R, int echunks, int table_elems) {
  return (size_t)((table_elems * 2 + 15) & ~15) + ((echunks * 8 * sizeof(EmbedCol) + 15) & ~(size_t)15) +
         (size_t)R * kTileM * 2;
}

void launch_embed(const float* rows, const uint8_t* packed, const PackedLayout& pl, int R, int L, int Lw, int M, int ntiles, int echunks,
                  const EmbedCol* cols, const EmbedRow* rowmeta, const __nv_bfloat16* tables,
                  int table_elems, __nv_bfloat16* emb, int* status, const TileFlow& flow, cudaStream_t st) {
  embed_rows_kernel<<<ntiles, 256, embed_smem_bytes(R, echunks, table_elems), st>>>(
      rows, packed, pl, R, L, Lw, M, echunks, cols, rowmeta, tables, table_elems, emb, status, flow);
}

void launch_gemm_row(const __nv_bfloat16* a_img, const __nv_bfloat16* b_img, int a_ksteps, int b_ksteps, int ntiles,
                     const RowEpi& epi, const TileFlow& flow, cudaStream_t st) {
  using Cfg = GemmCfg<kNC, 2, false>;
  const int grid = ntiles < num_sms() ? ntiles : num_sms();
  const int smem = Cfg::smem_bytes(Cfg::stages(b_ksteps / Cfg::kSK));
  launch(flow, gemm_kernel<kNC, 2, EPI_ROW, false>, grid, Cfg::kThreads, smem, st, a_img, b_img, a_ksteps, b_ksteps,
         ntiles, 1, (__nv_bfloat16*)nullptr, 0, epi, flow);
}

void launch_gemm_qkv(const __nv_bfloat16* a_img, const __nv_bfloat16* b_img, int ntiles,
                     __nv_bfloat16* qkv_img, cudaStream_t st) {
  using Cfg = GemmCfg<kNC, 1, true>;
  const int npairs = (ntiles + 1) / 2;
  const int grid = npairs < num_sms() ? npairs : num_sms();
  RowEpi none{};
  gemm_kernel<kNC, 1, EPI_QKV, true><<<grid, Cfg::kThreads, Cfg::kSmemBytes, st>>>(
      a_img, b_img, kDP / 16, 2 * (kDP / 16), ntiles, kQKVN / kQKVGroup, qkv_img, kQKVN / 8, none, TileFlow{});
}

void launch_ffn(int half, const __nv_bfloat16* xb_img, const __nv_bfloat16* w1_img, const float* b1,
                const __nv_bfloat16* w2_img, int ff, int ntiles, __nv_bfloat16* hid_img, const RowEpi& epi,
                const TileFlow& flow, cudaStream_t st) {
  const int split = (ntiles + 1) / 2;
  const int t0 = half ? split : 0, t1 = half ? ntiles : split;
  // a half without tiles still launches (one CTA that finds no work), so the forward's launch count does not depend
  // on the chunk size
  const int n = t1 - t0;
  const int grid = n < 1 ? 1 : n < num_sms() ? n : num_sms();
  launch(flow, hid_img ? ffn_gemm_kernel<true> : ffn_gemm_kernel<false>, grid, FfnCfg::kThreads, FfnCfg::kSmemBytes,
         st, xb_img, w1_img, b1, w2_img, ff, t0, t1, hid_img, epi, flow);
}

// packed rows -> the float32 [B, R, L] rows they stand for (the strict-fp32 path reads float32 rows)
__global__ void __launch_bounds__(256)
unpack_rows_kernel(const uint8_t* __restrict__ packed, PackedLayout pl, int nwindows, float* __restrict__ rows) {
  const int b = blockIdx.x;
  const uint8_t* w = packed + (size_t)b * pl.stride;
  float* out = rows + (size_t)b * pl.R * pl.L;
  for (int i = threadIdx.x; i < pl.R * pl.L; i += blockDim.x) {
    const int r = i / pl.L, l = i - r * pl.L;
    out[i] = packed_value(pl, w, r, l);
  }
}

void launch_unpack_rows(const uint8_t* packed, const PackedLayout& pl, int nwindows, float* rows, cudaStream_t st) {
  if (nwindows > 0) unpack_rows_kernel<<<nwindows, 256, 0, st>>>(packed, pl, nwindows, rows);
}


void launch_attention(const __nv_bfloat16* qkv, __nv_bfloat16* att, int L, int Lw, int win, int nwindows,
                      cudaStream_t st) {
  const int Lp = (L + 15) & ~15;
  const size_t smem = (size_t)2 * Lp * kAttStride * 2;
  band_attention_kernel<<<nwindows * 2, 128, smem, st>>>(qkv, att, L, Lw, win, nwindows);
}

void launch_qkv_attention(int half, const __nv_bfloat16* xb_img, const __nv_bfloat16* wqkv, int L, int win,
                          int ntiles, __nv_bfloat16* qkv_img, __nv_bfloat16* att, const TileFlow& flow,
                          cudaStream_t st) {
  const int split = (ntiles + 1) / 2;
  const int t0 = half ? split : 0, t1 = half ? ntiles : split;
  // a half without tiles still launches (one CTA that finds no work), as launch_ffn's
  const int n = t1 - t0;
  const int grid = n < 1 ? 1 : n < num_sms() ? n : num_sms();
  launch(flow, qkv_img ? qkv_attention_kernel<true> : qkv_attention_kernel<false>, grid, QkvAttCfg::kThreads,
         QkvAttCfg::kSmemBytes, st, xb_img, wqkv, L, win, t0, t1, qkv_img, att, flow);
}



// =====================================================================================
// stitch: per-read concatenation of windows + gap compaction (stitch_utils.py:51-98)
// =====================================================================================
// One CTA per read (ZMW).  Its windows are contiguous in the batch, so the read's input is one span of `bases` /
// `quals`: window w starts at win_off[w] (windows of any width, win_off [n_windows + 1]) or, with win_off NULL, at
// w * L.  The gap character ' ' and the quality character under it are dropped (order preserving: ballot-free block
// prefix sum over 1024-character tiles) and the compacted read is written at the same offset of seq_out / qual_out.
// Integer / byte work only: bit-exact against the reference's string loops.
__global__ void __launch_bounds__(256)
stitch_kernel(const uint8_t* __restrict__ bases, const uint8_t* __restrict__ quals, int L,
              const int64_t* __restrict__ win_off, const int32_t* __restrict__ zmw_start, uint8_t* __restrict__ seq_out,
              uint8_t* __restrict__ qual_out, int32_t* __restrict__ len_out) {
  __shared__ int s_warp[8];
  __shared__ int s_total;
  const int z = blockIdx.x;
  const size_t off = (size_t)window_offset(win_off, zmw_start[z], L);
  const int n = (int)(window_offset(win_off, zmw_start[z + 1], L) - (int64_t)off);
  const uint8_t* in_b = bases + off;
  const uint8_t* in_q = quals + off;
  uint8_t* out_b = seq_out + off;
  uint8_t* out_q = qual_out + off;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int running = 0;
  for (int t0 = 0; t0 < n; t0 += 1024) {
    uint8_t b[4], q[4];
    int cnt = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int idx = t0 + threadIdx.x * 4 + k;
      b[k] = idx < n ? in_b[idx] : (uint8_t)' ';
      q[k] = idx < n ? in_q[idx] : (uint8_t)0;
      cnt += b[k] != (uint8_t)' ';
    }
    // inclusive scan inside the warp, then across the 8 warps
    int incl = cnt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += v;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (threadIdx.x == 0) {
      int acc = 0;
      for (int w = 0; w < 8; ++w) { const int v = s_warp[w]; s_warp[w] = acc; acc += v; }
      s_total = acc;
    }
    __syncthreads();
    int pos = running + s_warp[warp] + incl - cnt;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (b[k] != (uint8_t)' ') {
        out_b[pos] = b[k];
        out_q[pos] = q[k];
        ++pos;
      }
    }
    running += s_total;
    __syncthreads();
  }
  if (threadIdx.x == 0) len_out[z] = running;
}

void launch_stitch(const uint8_t* bases, const uint8_t* quals, int L, const int64_t* win_off, const int32_t* zmw_start,
                   int n_zmw, uint8_t* seq_out, uint8_t* qual_out, int32_t* len_out, cudaStream_t st) {
  if (n_zmw > 0) stitch_kernel<<<n_zmw, 256, 0, st>>>(bases, quals, L, win_off, zmw_start, seq_out, qual_out, len_out);
}

void launch_head(const HeadParams& p, int ntiles, const TileFlow& flow, cudaStream_t st) {
  launch(flow, head_kernel, ntiles, 128, 0, st, p, flow);
}

}  // namespace dcb
