// Profiling aid (not on the product path): SM -> L2 store throughput (scripts/store_rate.py).
#include <stdlib.h>

#include "common.cuh"

namespace aldm {

// Store-path probe: every CTA (8 warps, like the GEMM epilogue) writes `iters` tiles of 64 KB to its own region of `dst`
// (L2-resident when the regions are small), either with STG.128 full-line stores (mode 0: lane l of warp w writes 16 bytes,
// 8 lanes per 128-byte row, 4 rows per instruction -- the epilogue's pattern) or with one cp.async.bulk (TMA) store of 4 KB
// per warp from shared memory (mode 1).  out[cta] = cycles.  Run with all SMs and with a few CTAs to separate a per-SM
// limit from a chip-level one.
__global__ void __launch_bounds__(256, 1) store_rate_kernel(float4* dst, int iters, int mode, long long region_bytes, long long* out) {
  extern __shared__ __align__(1024) uint8_t sm_store[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  uint8_t* base = reinterpret_cast<uint8_t*>(dst) + (long long)blockIdx.x * region_bytes;
  const int tiles_in_region = (int)(region_bytes / 65536);
  for (int i = tid; i < 65536 / 16; i += 256) reinterpret_cast<float4*>(sm_store)[i] = make_float4(1.f, 2.f, 3.f, 4.f);
  fence_proxy_async();
  __syncthreads();
  const long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
    uint8_t* tile = base + (long long)(it % tiles_in_region) * 65536;
    if (mode == 0) {
#pragma unroll
      for (int ch = 0; ch < 2; ++ch) {
        uint8_t* p = tile + (warp * 2 + ch) * 4096;      // 32 rows x 128 B
#pragma unroll
        for (int r = 0; r < 8; ++r)
          *reinterpret_cast<float4*>(p + (r * 4 + (lane >> 3)) * 128 + (lane & 7) * 16) = make_float4((float)it, 1.f, 2.f, 3.f);
      }
    } else {
      if (elect_one()) {
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(tile + warp * 8192), "r"(smem_u32(sm_store) + warp * 8192), "n"(8192) : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
      }
      __syncwarp();
    }
  }
  if (mode == 1 && elect_one()) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  __threadfence();
  __syncthreads();
  if (tid == 0) out[blockIdx.x] = clock64() - t0;
}

}  // namespace aldm

extern "C" int aldm_debug_store_rate(int32_t n_cta, int32_t iters, int32_t mode, long long region_bytes, long long* host_out) {
  using namespace aldm;
  ALDM_REQUIRE(host_out && n_cta > 0 && iters > 0 && (mode == 0 || mode == 1) && region_bytes >= 65536 && region_bytes % 65536 == 0, ALDM_E_ARG,
               "debug_store_rate: bad arguments");
  float4* dst = nullptr;
  long long* dev = nullptr;
  ALDM_CHECK_CUDA(cudaMalloc(&dst, (size_t)n_cta * region_bytes));
  ALDM_CHECK_CUDA(cudaMalloc(&dev, sizeof(long long) * n_cta));
  ALDM_CHECK_CUDA(cudaFuncSetAttribute(store_rate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  for (int rep = 0; rep < 2; ++rep) store_rate_kernel<<<n_cta, 256, 200 * 1024>>>(dst, iters, mode, region_bytes, dev);      // 200 KB: one CTA per SM
  ALDM_CHECK_CUDA(cudaGetLastError());
  ALDM_CHECK_CUDA(cudaDeviceSynchronize());
  ALDM_CHECK_CUDA(cudaMemcpy(host_out, dev, sizeof(long long) * n_cta, cudaMemcpyDeviceToHost));
  cudaFree(dst);
  cudaFree(dev);
  return ALDM_OK;
}
