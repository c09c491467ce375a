// L2 -> shared-memory streaming ceiling of the GEMM's operand ring (used by profile_gemms.py; not product code).
//
// Every CTA (one per SM, 384 threads like gemm_kernel) streams the same L2-resident weight image -- 16 n-groups of
// [18 k-steps][128 columns][16 B], the FFN up-projection's 1.18 MB -- through the GEMM's ring: kStages slots of
// kSK k-steps, one bulk copy per slot completing on its `full` mbarrier.  The 256 consumer threads do no MMA; they
// wait on `full` and arrive on `empty`.  The rate this reaches is what the producer side of the GEMM can deliver.
//
//   l2_stream <reps> [bytes_per_kstep]     prints one JSON line
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../deepconsensus_b200/csrc/sm90.cuh"

using namespace dcb;

constexpr int kStages = 4;
constexpr int kSK = 2;
constexpr int kKsteps = 18;
constexpr int kGroups = 16;

__global__ void __launch_bounds__(384, 1) l2_stream_kernel(const uint8_t* __restrict__ img, int kstep_bytes, int reps) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int stage_bytes = kSK * kstep_bytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kStages * stage_bytes);
  uint64_t* empty = full + kStages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 256);
    }
    mbar_fence_init();
  }
  __syncthreads();
  const int nstages = reps * kGroups * (kKsteps / kSK);
  uint32_t slot = 0, phase = 0;
  if (warp >= 8) {
    if (warp == 8 && lane == 0) {
      for (int s = 0, src = 0; s < nstages; ++s) {
        mbar_wait(&empty[slot], phase ^ 1);
        mbar_arrive_expect_tx(&full[slot], stage_bytes);
        bulk_g2s(smem + slot * stage_bytes, img + (size_t)src * stage_bytes, stage_bytes, &full[slot]);
        if (++src == kGroups * (kKsteps / kSK)) src = 0;
        if (++slot == kStages) { slot = 0; phase ^= 1; }
      }
    }
    return;
  }
  for (int s = 0; s < nstages; ++s) {
    mbar_wait(&full[slot], phase);
    mbar_arrive(&empty[slot]);
    if (++slot == kStages) { slot = 0; phase ^= 1; }
  }
}

#define CK(x)                                                                      \
  do {                                                                             \
    cudaError_t e_ = (x);                                                          \
    if (e_ != cudaSuccess) {                                                       \
      fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_));                     \
      return 1;                                                                    \
    }                                                                              \
  } while (0)

int main(int argc, char** argv) {
  const int reps = argc > 1 ? atoi(argv[1]) : 20;
  const int kstep_bytes = argc > 2 ? atoi(argv[2]) : 2 * 128 * 16;
  const size_t img_bytes = (size_t)kGroups * kKsteps * kstep_bytes;
  int dev = 0, sms = 0;
  CK(cudaGetDevice(&dev));
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, dev));
  uint8_t* img = nullptr;
  CK(cudaMalloc(&img, img_bytes));
  CK(cudaMemset(img, 1, img_bytes));
  // as much shared memory as the GEMM asks for, so that one CTA runs per SM
  const int smem = 180 * 1024;
  CK(cudaFuncSetAttribute(l2_stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  cudaEvent_t a, b;
  CK(cudaEventCreate(&a));
  CK(cudaEventCreate(&b));
  for (int i = 0; i < 3; ++i) l2_stream_kernel<<<sms, 384, smem>>>(img, kstep_bytes, reps);
  CK(cudaGetLastError());
  CK(cudaDeviceSynchronize());
  const int iters = 10;
  std::vector<float> ms(iters);
  for (int i = 0; i < iters; ++i) {
    CK(cudaEventRecord(a));
    l2_stream_kernel<<<sms, 384, smem>>>(img, kstep_bytes, reps);
    CK(cudaEventRecord(b));
    CK(cudaEventSynchronize(b));
    CK(cudaEventElapsedTime(&ms[i], a, b));
  }
  float best = ms[0], sum = 0.f;
  for (float m : ms) { best = m < best ? m : best; sum += m; }
  const double bytes = (double)sms * reps * img_bytes;
  printf("{\"device\": \"%s\", \"sms\": %d, \"image_bytes\": %zu, \"stage_bytes\": %d, \"stages\": %d, \"reps\": %d, "
         "\"bytes_per_launch\": %.0f, \"best_ms\": %.4f, \"mean_ms\": %.4f, \"best_tbps\": %.3f, \"mean_tbps\": %.3f}\n",
         prop.name, sms, img_bytes, kSK * kstep_bytes, kStages, reps, bytes, best, sum / iters, bytes / (best * 1e-3) / 1e12,
         bytes / (sum / iters * 1e-3) / 1e12);
  CK(cudaFree(img));
  return 0;
}
