// tf32x3 path of the dcb200 engine: the strict-fp32 forward (strict_kernels.cu) with its GEMMs on the tensor cores.
// Selected per engine (dcb_config.precision = DCB_PRECISION_TF32X3); embed, LayerNorm, attention and head are the
// strict path's own kernels.
//
// 3xTF32: every float32 operand x is split into big = tf32(x) and small = tf32(x - big) (cvt.rna, ties away from
// zero; 10 + 10 mantissa bits), and the product is accumulated in float32 as small.big + big.small + big.big.  Only
// small.small and the rounding of small (~2^-22 relative) are lost, so the logits stay within float32 tolerance of the
// strict path at tensor-core speed.
//
//   tf32x3_gemm_kernel  C = epilogue(A[M,K] . W[K,N]), StrictEpi's epilogue in the same order
//     - persistent CTAs over 128 x 144 output tiles, n fastest (the CTAs in flight share their A rows in L2)
//     - one producer warp: W's big / small k-slabs by one bulk copy (TMA) per stage, A's rows by cp.async (16 B
//       when the row pitch allows it, 4 B otherwise) with rows >= M and columns >= K zero-filled; both complete on
//       the stage's mbarrier
//     - two consumer warpgroups, 64 rows each: A from shared memory into registers, split there (no second activation
//       image), then wgmma m64n144k8 tf32 with A in registers and W's images in shared memory; each stage's products
//       (32 of K) are summed on the tensor cores and added to a float32 register accumulator
//     - no split-K and no atomics: an output's bits depend only on its row of A and on W
//
// W's image (tf32x3_image, built once per weight load): [N / 144 tiles][K / 32 stages][big, small][8][144][4] floats,
// the K-major no-swizzle core-matrix layout of sm90.cuh with 4-float (16 B) K-chunks.  Within each 16-wide K block the
// K order is permuted so that a thread's four consecutive A floats are its fragments of two k8 steps: slot j of the
// first / second core matrix of k8 step s holds k = 4j + 2s / 4j + 2s + 1.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "kernels.h"
#include "sm90.cuh"

namespace dcb {

namespace {

constexpr int kBM = 128, kBN = 144, kBK = 32, kStages = 4;
constexpr int kAPitch = kBK + 4;                   // floats per A row in shared memory (16-byte aligned, fewer conflicts)
constexpr int kABytes = kBM * kAPitch * 4;         // 18 KB
constexpr int kBSlab = kBK * kBN;                  // floats of one k-slab of W (big or small)
constexpr int kBBytes = 2 * kBSlab * 4;            // 36 KB: big, then small
constexpr int kStageBytes = kABytes + kBBytes;
constexpr size_t kSmemBytes = (size_t)kStages * kStageBytes + 2 * kStages * sizeof(uint64_t);
constexpr int kThreads = 384;                      // two consumer warpgroups + the producer warpgroup (one warp copies)

__device__ __forceinline__ uint32_t tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}

__device__ __forceinline__ void cp_async16(void* dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async4(void* dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(src_bytes) : "memory");
}
// one arrival on `bar` once every cp.async this thread has issued so far has landed (counted in the barrier's init)
__device__ __forceinline__ void cp_async_mbar_arrive(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// D[64 x 144] (+)= A[64 x 8] * B[144 x 8]^T, tf32 operands, A in registers (the m16n8k8 tf32 A layout: a0 row g k q,
// a1 row g + 8 k q, a2 row g k q + 4, a3 row g + 8 k q + 4; g = lane / 4, q = lane % 4), B K-major in shared memory.
__device__ __forceinline__ void wgmma_m64n144k8_tf32(float (&d)[72], const uint32_t (&a)[4], uint64_t b_desc,
                                                     int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %77, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n144k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71}, {%72, %73, %74, %75}, %76, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate));
}

__global__ void __launch_bounds__(kThreads, 1)
tf32x3_gemm_kernel(const float* __restrict__ A, const float* __restrict__ Wimg, float* C, int M, int N, int K,
                   StrictEpi ep) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes);
  uint64_t* empty = full + kStages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full[i], 1 + 32);   // the producer's expect_tx arrival + one cp.async arrival per producer lane
      mbar_init(&empty[i], 256);     // every consumer thread
    }
    mbar_fence_init();
  }
  __syncthreads();

  const int ntn = (N + kBN - 1) / kBN, nk = (K + kBK - 1) / kBK;
  const int ntiles = ((M + kBM - 1) / kBM) * ntn;

  if (warp >= 8) {
    // ------------------------------------------------------------- producer
    setmaxnreg_dec<40>();   // its registers go to the consumers' two accumulators
    if (warp != 8) return;
    const bool vec = (K & 3) == 0 && (reinterpret_cast<uintptr_t>(A) & 15) == 0;
    uint32_t slot = 0, phase = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      const int m0 = (tile / ntn) * kBM, nt = tile % ntn;
      for (int kc = 0; kc < nk; ++kc) {
        mbar_wait(&empty[slot], phase ^ 1);
        uint8_t* st = smem + slot * kStageBytes;
        if (lane == 0) {
          mbar_arrive_expect_tx(&full[slot], kBBytes);
          bulk_g2s(st + kABytes, Wimg + ((size_t)nt * nk + kc) * 2 * kBSlab, kBBytes, &full[slot]);
        }
        float* as = reinterpret_cast<float*>(st);
        const int k0 = kc * kBK;
        if (vec) {
#pragma unroll 4
          for (int i = 0; i < kBM * kBK / 4 / 32; ++i) {
            const int idx = i * 32 + lane, r = idx >> 3, c = (idx & 7) * 4;
            const int gm = m0 + r, gk = k0 + c;
            const bool ok = gm < M && gk < K;
            cp_async16(as + r * kAPitch + c, ok ? A + (size_t)gm * K + gk : A, ok ? 16 : 0);
          }
        } else {
#pragma unroll 4
          for (int i = 0; i < kBM * kBK / 32; ++i) {
            const int r = i, c = lane;
            const int gm = m0 + r, gk = k0 + c;
            const bool ok = gm < M && gk < K;
            cp_async4(as + r * kAPitch + c, ok ? A + (size_t)gm * K + gk : A, ok ? 4 : 0);
          }
        }
        cp_async_mbar_arrive(&full[slot]);
        if (++slot == kStages) { slot = 0; phase ^= 1; }
      }
    }
    return;
  }

  // --------------------------------------------------------------- consumers
  setmaxnreg_inc<232>();
  const int wg = warp >> 2, wl = warp & 3;
  const int g = lane >> 2, q = lane & 3;
  const int row0 = wg * 64 + wl * 16 + g;   // this thread's rows in the tile: row0, row0 + 8
  uint32_t slot = 0, phase = 0;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int m0 = (tile / ntn) * kBM, n0 = (tile % ntn) * kBN;
    // The tensor cores' float32 accumulation is not IEEE round-to-nearest (measured: 10-20x the error of exact
    // products over K = 2048), so each stage's 96 products are summed there into `part` and the stages here.
    float acc[72], part[72];
#pragma unroll
    for (int i = 0; i < 72; ++i) acc[i] = 0.f;
    for (int kc = 0; kc < nk; ++kc) {
      mbar_wait(&full[slot], phase);
      const uint8_t* st = smem + slot * kStageBytes;
      const float* as = reinterpret_cast<const float*>(st) + row0 * kAPitch + 4 * q;
      uint32_t big[4][4], sml[4][4];   // per k8 step: a0..a3
#pragma unroll
      for (int kb = 0; kb < 2; ++kb) {
        const float4 x0 = *reinterpret_cast<const float4*>(as + kb * 16);
        const float4 x1 = *reinterpret_cast<const float4*>(as + 8 * kAPitch + kb * 16);
        const float v[2][4] = {{x0.x, x1.x, x0.y, x1.y}, {x0.z, x1.z, x0.w, x1.w}};
#pragma unroll
        for (int s = 0; s < 2; ++s)
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            big[2 * kb + s][i] = tf32_rna(v[s][i]);
            sml[2 * kb + s][i] = tf32_rna(v[s][i] - __uint_as_float(big[2 * kb + s][i]));
          }
      }
      const uint32_t wb = smem_u32(st + kABytes), ws = wb + kBSlab * 4;
      wgmma_fence();
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        const uint64_t db = make_kc16_desc(wb + s * 2 * kBN * 16, kBN * 16, 128);
        const uint64_t ds = make_kc16_desc(ws + s * 2 * kBN * 16, kBN * 16, 128);
        wgmma_m64n144k8_tf32(part, sml[s], db, s);
        wgmma_m64n144k8_tf32(part, big[s], ds, 1);
        wgmma_m64n144k8_tf32(part, big[s], db, 1);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(part);
#pragma unroll
      for (int i = 0; i < 72; ++i) acc[i] += part[i];
      mbar_arrive(&empty[slot]);
      if (++slot == kStages) { slot = 0; phase ^= 1; }
    }
    // epilogue (strict_gemm_kernel's order): + bias, ReLU, * scale, + residual (may alias C), + positional table
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int gm = m0 + row0 + 8 * h;
      if (gm >= M) continue;
      const float* pe_row = ep.pe ? ep.pe + (size_t)(gm % ep.pe_L) * N : nullptr;
#pragma unroll
      for (int j = 0; j < 18; ++j)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int gn = n0 + 8 * j + 2 * q + c;
          if (gn >= N) continue;
          float v = acc[4 * j + 2 * h + c];
          if (ep.bias) v += ep.bias[gn];
          if (ep.relu) v = fmaxf(v, 0.f);
          v *= ep.scale;
          if (ep.residual) v = ep.residual[(size_t)gm * N + gn] + v;
          if (pe_row) v += pe_row[gn];
          C[(size_t)gm * N + gn] = v;
        }
    }
  }
}

float tf32_rna_host(float x) {   // cvt.rna.tf32.f32 on finite values
  uint32_t u;
  memcpy(&u, &x, 4);
  if ((u & 0x7f800000u) != 0x7f800000u) u += 0x1000u;
  u &= 0xffffe000u;
  memcpy(&x, &u, 4);
  return x;
}

}  // namespace

size_t tf32x3_image_elems(int K, int N) {
  return (size_t)((N + kBN - 1) / kBN) * ((K + kBK - 1) / kBK) * 2 * kBSlab;
}

std::vector<float> tf32x3_image(const float* W, int K, int N) {
  const int ntn = (N + kBN - 1) / kBN, nk = (K + kBK - 1) / kBK;
  std::vector<float> img(tf32x3_image_elems(K, N), 0.f);
  for (int nt = 0; nt < ntn; ++nt)
    for (int kc = 0; kc < nk; ++kc)
      for (int kch = 0; kch < kBK / 4; ++kch)
        for (int n = 0; n < kBN; ++n)
          for (int j = 0; j < 4; ++j) {
            const int st = kch >> 1, c = kch & 1;   // k8 step in the stage, first / second core matrix
            const int k = kc * kBK + (st >> 1) * 16 + 4 * j + 2 * (st & 1) + c, gn = nt * kBN + n;
            if (k >= K || gn >= N) continue;
            const float w = W[(size_t)k * N + gn];
            const float big = tf32_rna_host(w);
            const size_t at = ((((size_t)nt * nk + kc) * 2) * (kBK / 4) + kch) * kBN * 4 + (size_t)n * 4 + j;
            img[at] = big;
            img[at + kBSlab] = tf32_rna_host(w - big);
          }
  return img;
}

cudaError_t tf32x3_init() {
  return cudaFuncSetAttribute(tf32x3_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes);
}

void launch_tf32x3_gemm(const float* A, const float* Wimg, float* C, int M, int N, int K, const StrictEpi& ep,
                        cudaStream_t st) {
  if (M <= 0) return;
  const int ntiles = ((M + kBM - 1) / kBM) * ((N + kBN - 1) / kBN);
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  tf32x3_gemm_kernel<<<ntiles < sms ? ntiles : sms, kThreads, kSmemBytes, st>>>(A, Wimg, C, M, N, K, ep);
}

}  // namespace dcb
