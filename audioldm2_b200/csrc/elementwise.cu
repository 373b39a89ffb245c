// K6 and friends: the HBM-bound elementwise kernels of the sampler loop.
//   ddim_step_kernel      CFG combine + DDIM x_{t-1} update (ddim.py:298-300,339-354), float4, one pass
//   masked_blend_kernel   q_sample + mask blend (ddim.py:226-231, ddpm.py:430-436)
//   temb_kernel           sinusoidal timestep embedding (util.py:172-196) -> operand planes
//   transpose_kernel      [B,C,HW] <-> [B,HW,C]
//   posterior_kernel      DiagonalGaussianDistribution.sample with caller noise (distributions.py:24-41)
#include "common.cuh"

namespace aldm {

struct DdimCoef {
  float inv_sqrt_at, s1m, sqrt_aprev, dir, sigma, g;
};

// Algorithmic traffic: read x, e_u, e_c, noise; write x_prev (+pred_x0) = 20 (24) bytes / element.
__global__ void __launch_bounds__(256) ddim_step_kernel(const float4* __restrict__ x, const float4* __restrict__ eu,
                                                        const float4* __restrict__ ec, const float4* __restrict__ nz,
                                                        float4* __restrict__ xp, float4* __restrict__ px0,
                                                        long long n4, DdimCoef c) {
  pdl_wait();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 X = __ldcs(x + i), U = __ldcs(eu + i), Cn = __ldcs(ec + i), Z = __ldcs(nz + i);
    float4 P, O;
#define ALDM_DDIM1(f)                                          \
    {                                                          \
      const float e = U.f + c.g * (Cn.f - U.f);                \
      const float p0 = (X.f - c.s1m * e) / c.inv_sqrt_at;      \
      P.f = p0;                                                \
      O.f = c.sqrt_aprev * p0 + c.dir * e + c.sigma * Z.f;     \
    }
    ALDM_DDIM1(x) ALDM_DDIM1(y) ALDM_DDIM1(z) ALDM_DDIM1(w)
#undef ALDM_DDIM1
    xp[i] = O;
    if (px0) px0[i] = P;
  }
}

__global__ void masked_blend_kernel(float* __restrict__ img, const float* __restrict__ x0,
                                    const float* __restrict__ mask, const float* __restrict__ qn, int C, int TF,
                                    long long n, float sa, float sb) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long b = i / ((long long)C * TF);
  const float m = mask[b * TF + (i % TF)];
  const float orig = sa * x0[i] + sb * qn[i];
  img[i] = orig * m + (1.0f - m) * img[i];
}

__global__ void temb_kernel(const long long* __restrict__ t, int B, int dim, const float* __restrict__ freqs,
                            aldm_plane_t* __restrict__ hi, aldm_plane_t* __restrict__ lo) {
  pdl_wait();
  const int half = dim >> 1;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * half) return;
  const int b = idx / half, i = idx % half;
  // freqs[i] = exp(-ln(max_period) * i / half) is tabulated by the host exactly as util.py:183-187
  // does (a 1-ulp difference in exp() would be amplified by t ~ 1000 in the argument);
  // args = t.float() * freqs (util.py:188) is an exact fp32 product.
  const float arg = (float)t[b] * __ldg(freqs + i);
  const float cv = cosf(arg), sv = sinf(arg);
  store_split1(hi, lo, (long long)b * dim + i, cv);
  store_split1(hi, lo, (long long)b * dim + half + i, sv);
}

__global__ void transpose_kernel(const float* __restrict__ src, float* __restrict__ dst, int C, int HW, int to_nhwc,
                                 long long n) {
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  // i indexes dst
  if (to_nhwc) {
    const int c = (int)(i % C);
    const long long p = (i / C) % HW, b = i / ((long long)C * HW);
    dst[i] = src[(b * C + c) * HW + p];
  } else {
    const long long p = i % HW;
    const int c = (int)((i / HW) % C);
    const long long b = i / ((long long)C * HW);
    dst[i] = src[(b * HW + p) * C + c];
  }
}

__global__ void posterior_kernel(const float* __restrict__ mom, const float* __restrict__ noise, float* __restrict__ z,
                                 int zc, int HW, long long n, float scale) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // over NCHW output
  if (i >= n) return;
  const long long p = i % HW;
  const int c = (int)((i / HW) % zc);
  const long long b = i / ((long long)zc * HW);
  const float* mp = mom + (b * HW + p) * (2 * zc);
  const float mean = mp[c];
  float lv = mp[zc + c];
  lv = fminf(fmaxf(lv, -30.0f), 20.0f);
  z[i] = scale * (mean + expf(0.5f * lv) * noise[i]);
}

}  // namespace aldm

using namespace aldm;

extern "C" int aldm_ddim_step(const float* x, const float* eps_uncond, const float* eps_cond, const float* noise,
                              float* x_prev, float* pred_x0, int64_t n_total, float a_t, float a_prev, float sigma_t,
                              float sqrt_one_minus_at, float guidance, void* stream) {
  ALDM_REQUIRE(x && eps_uncond && eps_cond && noise && x_prev, ALDM_E_ARG, "ddim_step: null pointer");
  ALDM_REQUIRE(n_total > 0 && n_total % 4 == 0, ALDM_E_SHAPE, "ddim_step: n_total=%lld must be a positive multiple of 4",
               (long long)n_total);
  ALDM_REQUIRE(aligned16(x) && aligned16(eps_uncond) && aligned16(eps_cond) && aligned16(noise) && aligned16(x_prev) &&
                   (!pred_x0 || aligned16(pred_x0)),
               ALDM_E_ALIGN, "ddim_step: pointers must be 16B aligned");
  DdimCoef c;
  // same fp32 evaluation order as the reference: a_t.sqrt(), (1 - a_prev - sigma^2).sqrt(), a_prev.sqrt()
  c.inv_sqrt_at = sqrtf(a_t);              // used as a divisor, exactly as `/ a_t.sqrt()` (ddim.py:339)
  c.s1m = sqrt_one_minus_at;
  c.sqrt_aprev = sqrtf(a_prev);
  c.dir = sqrtf(1.0f - a_prev - sigma_t * sigma_t);
  c.sigma = sigma_t;
  c.g = guidance;
  const long long n4 = n_total / 4;
  long long blocks = (n4 + 255) / 256;
  if (blocks > num_sms() * 8) blocks = num_sms() * 8;
  ddim_step_kernel<<<(unsigned)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float4*>(x), reinterpret_cast<const float4*>(eps_uncond),
      reinterpret_cast<const float4*>(eps_cond), reinterpret_cast<const float4*>(noise),
      reinterpret_cast<float4*>(x_prev), reinterpret_cast<float4*>(pred_x0), n4, c);
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}

extern "C" int aldm_masked_blend(float* img, const float* x0, const float* mask, const float* q_noise, int32_t B,
                                 int32_t C, int32_t TF, float sqrt_acp, float sqrt_1m_acp, void* stream) {
  ALDM_REQUIRE(img && x0 && mask && q_noise, ALDM_E_ARG, "masked_blend: null pointer");
  ALDM_REQUIRE(B > 0 && C > 0 && TF > 0, ALDM_E_SHAPE, "masked_blend: bad shape");
  const long long n = (long long)B * C * TF;
  masked_blend_kernel<<<(unsigned)((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      img, x0, mask, q_noise, C, TF, n, sqrt_acp, sqrt_1m_acp);
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}

extern "C" int aldm_timestep_embedding(const int64_t* t, int32_t B, int32_t dim, const float* freqs, void* out_hi,
                                       void* out_lo, void* stream) {
  ALDM_REQUIRE(t && freqs && out_hi, ALDM_E_ARG, "timestep_embedding: null pointer");      // out_lo == NULL: hi plane only
  ALDM_REQUIRE(B > 0 && dim > 0 && dim % 8 == 0, ALDM_E_SHAPE, "timestep_embedding: B=%d dim=%d", B, dim);
  const int n = B * (dim / 2);
  temb_kernel<<<(n + 127) / 128, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const long long*>(t), B, dim, freqs, reinterpret_cast<aldm_plane_t*>(out_hi),
      reinterpret_cast<aldm_plane_t*>(out_lo));
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}

extern "C" int aldm_transpose_chw(const float* src, float* dst, int32_t B, int32_t C, int32_t HW, int32_t to_nhwc,
                                  void* stream) {
  ALDM_REQUIRE(src && dst && B > 0 && C > 0 && HW > 0, ALDM_E_ARG, "transpose: bad arguments");
  const long long n = (long long)B * C * HW;
  transpose_kernel<<<(unsigned)((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(src, dst, C, HW,
                                                                                                     to_nhwc, n);
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}

extern "C" int aldm_posterior_sample(const float* moments, const float* noise_nchw, float* z_nchw, int32_t B, int32_t zc,
                                     int32_t HW, float scale, void* stream) {
  ALDM_REQUIRE(moments && noise_nchw && z_nchw && B > 0 && zc > 0 && HW > 0, ALDM_E_ARG, "posterior_sample: bad arguments");
  const long long n = (long long)B * zc * HW;
  posterior_kernel<<<(unsigned)((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      moments, noise_nchw, z_nchw, zc, HW, n, scale);
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}
