// Shared host/device definitions of the dcb200 engine: model constants, HBM image
// layouts and kernel parameter blocks.
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

namespace dcb {

// ------------------------------------------------------------------ model geometry
// The released DeepConsensus transformers all use hidden_size=280, 2 heads
// (model_configs.py:84,139); the engine fixes these at compile time and validates
// params.json against them in dcb_create().  Everything else (max_passes,
// max_length, layers, filter_size, ReZero vs LayerNorm, ccs_bq, band) is runtime.
constexpr int kTileM = 128;     // tokens per tile (two wgmma M=64 warpgroups)
constexpr int kD = 280;         // hidden_size
constexpr int kDP = 288;        // hidden_size padded to a multiple of 16 (wgmma K granularity)
constexpr int kHeads = 2;
constexpr int kDH = 140;        // size per head
constexpr int kDHP = 144;       // padded per-head size (multiple of 16)
constexpr int kQKVN = 3 * kHeads * kDHP;  // 864: [q_h0|q_h1|k_h0|k_h1|v_h0|v_h1]
constexpr int kQKVGroup = 144;  // q/k/v columns per GEMM n-group (6 groups: one accumulator chunk per consumer)
constexpr int kNC = 144;        // wgmma N per instruction for the d-wide GEMMs (288 = 2 x 144)
constexpr int kVocab = 5;       // ' ATCG' (dc_constants.py:39-42)
constexpr int kFFChunk = 128;   // filter_size is processed in chunks of 128 hidden units

// ------------------------------------------------------------------ HBM images
// bf16 activation image ("A operand image"): [tile][K/8][128][8]  -> 16 B per (chunk,row)
// fp32 residual image:                        [tile][288/4][128][4] -> 16 B per (chunk,row)
// Both make a warp's accesses (lane == row) 512 B contiguous.
constexpr int kXChunks = kDP / 4;  // 72
__host__ __device__ inline size_t act_image_elems(int k) { return (size_t)kTileM * k; }
__host__ __device__ inline size_t x_image_elems() { return (size_t)kTileM * kDP; }

// ------------------------------------------------------------------ embed descriptor
// One entry per column e of the concatenated embedding (networks.py:457-506).
struct EmbedCol {
  int16_t src_row;    // input row r
  int16_t width;      // embedding width of that row's table
  int16_t col;        // column within the embedding vector
  int16_t shift;      // +1 for the ccs_bq row (networks.py:495)
  int32_t table_off;  // element offset of the table in the packed bf16 table blob
  int32_t vocab;      // rows of the table
  float clip_hi;      // > 0: clip value to [0, clip_hi] first (data_providers.py:151-162)
};

// Per input row: how a raw value becomes a table id.
struct EmbedRow {
  float clip_hi;   // > 0: clip to [0, clip_hi] (format_rows)
  int32_t shift;   // +1 for ccs_bq
  int32_t vocab;   // table rows
};

// ------------------------------------------------------------------ packed input rows (include/dcb200.h)
// Per window: u8 [P][L] base|strand<<3, u8 [P][L] pw, u8 [P][L] ip, u8 [L] ccs, (u8 [L] ccs_bq + 1), pad to 16 B,
// f32 [4] SN.  Reference row r of the float32 layout (data_providers.py:81-113) maps to:
struct PackedLayout {
  int P, L, bq;
  int R;          // reference rows: 4P + 5 + bq
  int sn_off;     // byte offset of the four SN floats
  int stride;     // bytes per window (multiple of 16)
};
__host__ __device__ inline PackedLayout make_packed_layout(int P, int L, int bq) {
  PackedLayout pl;
  pl.P = P; pl.L = L; pl.bq = bq; pl.R = 4 * P + 5 + bq;
  pl.sn_off = ((3 * P + 1 + bq) * L + 15) & ~15;
  pl.stride = pl.sn_off + 16;
  return pl;
}
// The float32 value row r of the reference layout holds at position l (ccs_bq: the stored byte is value + 1).
__host__ __device__ inline float packed_value(const PackedLayout& pl, const uint8_t* w, int r, int l) {
  const int P = pl.P, L = pl.L;
  if (r < P) return (float)(w[r * L + l] & 7);
  if (r < 3 * P) return (float)w[r * L + l];
  if (r < 4 * P) return (float)((w[(r - 3 * P) * L + l] >> 3) & 3);
  if (r == 4 * P) return (float)w[3 * P * L + l];
  if (pl.bq && r == 4 * P + 1) return (float)w[(3 * P + 1) * L + l] - 1.f;
  return reinterpret_cast<const float*>(w + pl.sn_off)[r - (pl.R - 4)];
}

// ------------------------------------------------------------------ strict-fp32 path (strict_kernels.cu)
// Per input row: clip / shift / vocabulary as EmbedRow, plus where its embedding lands in the concatenated vector and
// which float32 table (pre-scaled by sqrt(width), row 0 zeroed) it reads.
struct StrictEmbedRow {
  float clip_hi;
  int32_t shift;
  int32_t vocab;
  int32_t width;
  int32_t col0;        // first column in the [E] embedding vector
  int32_t table_off;   // element offset in the float32 table blob
};
// v = acc (+ bias[n]) -> (ReLU) -> * scale -> (+ residual[m, n]) -> (+ pe[m % pe_L, n])
struct StrictEpi {
  const float* bias = nullptr;
  const float* residual = nullptr;
  const float* pe = nullptr;
  int pe_L = 1;
  int relu = 0;
  float scale = 1.f;
};

// ------------------------------------------------------------------ row epilogue
// Shared tail of every d-wide GEMM: x_new = acc (+ x_old) (+ bias) (+ pos-enc);
// write x_new (fp32 image) and the next sub-layer's bf16 operand image
// (identity for ReZero, LayerNorm(eps=1e-6) otherwise).
struct RowEpi {
  float* x;              // fp32 residual image of the chunk (read when has_xold, always written)
  __nv_bfloat16* xb;     // bf16 operand image for the next GEMM (may be null: skip)
  const float* bias;     // [288] or null
  const float* pe;       // [Lw][288] or null (rows >= max_length are zero)
  const float* pe_img;   // the same table as a residual image [72][128][4] (tile == window), or null
  const float* ln_g;     // [288] or null  (null => xb = bf16(x_new))
  const float* ln_b;     // [288]
  int has_xold;
  int L;                 // tokens per window in the flattened layout (Lw): position = token % L
};

// ------------------------------------------------------------------ tile flow
// How one launch of the window-aligned forward meets the launches around it tile by tile (kernels.cu, tile_wait and
// tile_done): before it reads tile t it waits until flags[t] == wait, and once tile t's outputs are visible it stores
// `done` there.  flags null: the launch is serialized behind the one before it and neither waits nor stores.
struct TileFlow {
  int* flags;            // [tiles of a chunk]
  int wait, done;
  int* status;           // the submission's status word: kStatusTileWait is set when a wait times out
};
constexpr int kStatusTileWait = 2;

struct HeadParams {
  const float* x;        // fp32 residual image
  const float* ln_g;     // final LayerNorm gamma/beta [288]
  const float* ln_b;
  const float* wfc;      // [280][5]
  const float* bfc;      // [5]
  const float* gw8;      // [280][8]: gamma_c * Wfc[c][j] for j < 5, zero padded
  const float* ab;       // [16]: A_j = sum_c gamma_c Wfc[c][j] at 0..4, B_j = sum_c beta_c Wfc[c][j] at 8..12
  uint8_t* bases;        // [M] ASCII ' ATCG'
  uint8_t* quals;        // [M] Phred+33
  float* probs;          // [M][5] or null
  float* logits;         // [M][5] or null
  int M;                 // tokens in the layout (windows * Lw)
  int L, Lw;             // window length / tokens per window in the layout (Lw >= L: padding rows are skipped)
  int calib_enabled;
  float calib_thr, calib_w, calib_b;
  double calib_w64, calib_b64, calib_thr64;
  float max_q;
};

}  // namespace dcb
