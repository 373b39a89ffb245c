// DDIMSampler.stochastic_encode (latent_diffusion/models/ddim.py:434-449) for style transfer, next to K6's DDIM step
// (elementwise.cu): out = sqrt(ddim_alphas)[t] * x0' + ddim_sqrt_one_minus_alphas[t] * noise, float4, one HBM-bound
// pass.  x0' is x0, or clip(x0, -10, 10) when the device-side guard word says so (AudioLDM 1's latent guard), so that
// the decision made on the device from the encoder's output needs no host synchronisation before the first UNet step.
#include "../common.cuh"

namespace aldm {

__device__ __forceinline__ float guard_clip(float v) {
  // torch.clip(v, -10, 10); NaN passes through (fminf / fmaxf would replace it by the bound)
  return v != v ? v : fminf(fmaxf(v, -10.0f), 10.0f);
}

// The two products and the sum are rounded one by one (no FMA contraction), in the order of the reference's torch
// expression, so the result equals it bit for bit.  Algorithmic traffic: read x0, noise; write out = 12 B / element.
__global__ void __launch_bounds__(256) stochastic_encode_kernel(const float4* __restrict__ x0,
                                                                const float4* __restrict__ nz,
                                                                float4* __restrict__ out,
                                                                const int* __restrict__ clip_flag, long long n4,
                                                                float c0, float c1) {
  pdl_wait();
  const bool clip = clip_flag != nullptr && *clip_flag != 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 X = __ldcs(x0 + i);
    const float4 Z = __ldcs(nz + i);
    if (clip) {
      X.x = guard_clip(X.x);
      X.y = guard_clip(X.y);
      X.z = guard_clip(X.z);
      X.w = guard_clip(X.w);
    }
    float4 O;
    O.x = __fadd_rn(__fmul_rn(c0, X.x), __fmul_rn(c1, Z.x));
    O.y = __fadd_rn(__fmul_rn(c0, X.y), __fmul_rn(c1, Z.y));
    O.z = __fadd_rn(__fmul_rn(c0, X.z), __fmul_rn(c1, Z.z));
    O.w = __fadd_rn(__fmul_rn(c0, X.w), __fmul_rn(c1, Z.w));
    out[i] = O;
  }
}

// [a, a + na) and [b, b + nb) share a byte
inline bool overlaps(const void* a, long long na, const void* b, long long nb) {
  const uintptr_t pa = reinterpret_cast<uintptr_t>(a), pb = reinterpret_cast<uintptr_t>(b);
  return pa < pb + (uintptr_t)nb && pb < pa + (uintptr_t)na;
}

}  // namespace aldm

using namespace aldm;

extern "C" int aldm_stochastic_encode(const float* x0, const float* noise, float* out, int64_t n_total, float c0,
                                      float c1, const int32_t* clip_flag, void* stream) {
  ALDM_REQUIRE(x0 && noise && out, ALDM_E_ARG, "stochastic_encode: null pointer");
  ALDM_REQUIRE(n_total > 0 && n_total % 4 == 0, ALDM_E_SHAPE,
               "stochastic_encode: n_total=%lld must be a positive multiple of 4", (long long)n_total);
  ALDM_REQUIRE(aligned16(x0) && aligned16(noise) && aligned16(out), ALDM_E_ALIGN,
               "stochastic_encode: x0, noise and out must be 16B aligned");
  ALDM_REQUIRE(!clip_flag || (reinterpret_cast<uintptr_t>(clip_flag) & 3u) == 0, ALDM_E_ALIGN,
               "stochastic_encode: clip_flag must be 4B aligned");
  const long long bytes = (long long)n_total * 4;
  ALDM_REQUIRE(!overlaps(out, bytes, x0, bytes) && !overlaps(out, bytes, noise, bytes), ALDM_E_ARG,
               "stochastic_encode: out must not overlap x0 or noise");
  ALDM_REQUIRE(!clip_flag || !overlaps(out, bytes, clip_flag, 4), ALDM_E_ARG,
               "stochastic_encode: clip_flag must not lie inside out");
  const long long n4 = n_total / 4;
  long long blocks = (n4 + 255) / 256;
  if (blocks > num_sms() * 8) blocks = num_sms() * 8;
  stochastic_encode_kernel<<<(unsigned)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float4*>(x0), reinterpret_cast<const float4*>(noise), reinterpret_cast<float4*>(out),
      reinterpret_cast<const int*>(clip_flag), n4, c0, c1);
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}
