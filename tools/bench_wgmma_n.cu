// bench_wgmma_n.cu — does one wide wgmma (m64n64k8 / m64n128k8, tf32, A from registers) retire the work of two or
// four m64n32k8 in less time?  (`make build/bench_wgmma_n && build/bench_wgmma_n`; needs an sm_90a GPU)
//
// One CTA per SM, two warpgroups, as in the Linear GEMMs.  Each "block" is what the dW kernel issues per 32 vertices
// and warpgroup: 4 k8 steps x 3 operand pairs (3xTF32) over N = 32 NC output columns, either as NC m64n32k8 per pair
// or as one m64n(32 NC)k8.  B sits in shared memory (K-major, 128-byte swizzle); the loop commits one group per
// block and retires with wait_group 1, so the tensor pipe always has the next block queued.  No global traffic in
// the loop: this is the tensor pipe's own rate.  Prints one JSON line per variant.
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "tc_common.cuh"

using namespace roc::tc;

template <int NC, bool WIDE>
__global__ void __launch_bounds__(256, 1) k_mma_rate(float* out, int iters, long long* cycles) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* b = reinterpret_cast<float*>(smem);
  for (int i = threadIdx.x; i < 2 * NC * 32 * 32; i += blockDim.x) b[i] = (float)((i * 7) % 13) * 0.125f;
  fence_proxy_async_smem();
  __syncthreads();
  const uint32_t dHi = smem_u32(b), dLo = dHi + NC * 32 * 32 * 4;
  uint32_t fr[4][2][4];
#pragma unroll
  for (int kk = 0; kk < 4; kk++)
#pragma unroll
    for (int i = 0; i < 4; i++) split_tf32((float)((threadIdx.x + kk * 5 + i) % 11) * 0.25f, fr[kk][0][i], fr[kk][1][i]);
  float acc[NC][16];
#pragma unroll
  for (int c = 0; c < NC; c++)
#pragma unroll
    for (int i = 0; i < 16; i++) acc[c][i] = 0.f;
  const long long t0 = clock64();
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int kk = 0; kk < 4; kk++) {
      wgmma_fence();
      const uint32_t off = (uint32_t)kk * 32u;
      if constexpr (WIDE) {
        wgmma_m64nNk8_tf32<NC>(acc, fr[kk][1], make_sdesc_sw128(dHi + off));
        wgmma_m64nNk8_tf32<NC>(acc, fr[kk][0], make_sdesc_sw128(dLo + off));
        wgmma_m64nNk8_tf32<NC>(acc, fr[kk][0], make_sdesc_sw128(dHi + off));
      } else {
#pragma unroll
        for (int c = 0; c < NC; c++) {
          const uint32_t o = off + (uint32_t)c * 32u * 128u;
          wgmma_m64n32k8_tf32(acc[c], fr[kk][1], make_sdesc_sw128(dHi + o));
          wgmma_m64n32k8_tf32(acc[c], fr[kk][0], make_sdesc_sw128(dLo + o));
          wgmma_m64n32k8_tf32(acc[c], fr[kk][0], make_sdesc_sw128(dHi + o));
        }
      }
    }
    wgmma_commit();
    asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
  }
  wgmma_wait_all();
#pragma unroll
  for (int c = 0; c < NC; c++) wgmma_fence_acc(acc[c]);
  const long long t1 = clock64();
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < NC; c++)
#pragma unroll
    for (int i = 0; i < 16; i++) s += acc[c][i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

#define CK(x)                                                                        \
  do {                                                                               \
    cudaError_t e_ = (x);                                                            \
    if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); return 1; } \
  } while (0)

template <int NC, bool WIDE>
static int run(int sms, int iters) {
  const size_t smem = 1024 + 2 * NC * 32 * 32 * 4;
  CK(cudaFuncSetAttribute(k_mma_rate<NC, WIDE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  float* out; long long* cyc;
  CK(cudaMalloc(&out, (size_t)sms * 256 * sizeof(float)));
  CK(cudaMalloc(&cyc, (size_t)sms * sizeof(long long)));
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  k_mma_rate<NC, WIDE><<<sms, 256, smem>>>(out, iters / 10, cyc);   // warm-up
  CK(cudaEventRecord(e0));
  k_mma_rate<NC, WIDE><<<sms, 256, smem>>>(out, iters, cyc);
  CK(cudaEventRecord(e1));
  CK(cudaEventSynchronize(e1));
  CK(cudaGetLastError());
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, e0, e1));
  std::vector<long long> c(sms);
  CK(cudaMemcpy(c.data(), cyc, sms * sizeof(long long), cudaMemcpyDeviceToHost));
  double cycles = 0;
  for (long long v : c) cycles += (double)v;
  cycles /= sms;
  // per block and CTA: 2 warpgroups x 4 k8 x 3 pairs x 64 x 32 NC x 8 multiply-adds
  const double flops = 2.0 * (double)sms * iters * 2 * 4 * 3 * 64.0 * 32 * NC * 8;
  printf("{\"n\": %d, \"mma\": \"%s\", \"mmas_per_block_per_wg\": %d, \"ns_per_block\": %.1f, "
         "\"cycles_per_block\": %.1f, \"sm_mhz\": %.0f, \"tflops_tf32\": %.1f}\n",
         32 * NC, WIDE ? "wide" : "n32", WIDE ? 12 : 12 * NC, ms * 1e6 / iters, cycles / iters,
         cycles / (ms * 1e3), flops / (ms * 1e9));
  CK(cudaFree(out)); CK(cudaFree(cyc));
  return 0;
}

int main(int argc, char** argv) {
  int dev = 0, sms = 0;
  CK(cudaSetDevice(dev));
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int iters = argc > 1 ? atoi(argv[1]) : 20000;
  int rc = 0;
  rc |= run<1, false>(sms, iters);
  rc |= run<2, false>(sms, iters);
  rc |= run<2, true>(sms, iters);
  rc |= run<4, false>(sms, iters);
  rc |= run<4, true>(sms, iters);
  return rc;
}
