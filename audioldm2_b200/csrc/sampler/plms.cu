// The PLMS sampler's per-evaluation update (latent_diffusion/models/plms.py), next to K6's DDIM step
// (elementwise.cu): CFG combine + e' (first-step average or Adams-Bashforth order 1-4) + x_{t-1} update, float4, one
// HBM-bound pass.
#include "../common.cuh"

namespace aldm {

struct PlmsCoef {
  float sqrt_at, s1m, sqrt_aprev, dir, g;
};

// PLMS e' (plms.py:341-356) + x_{t-1} update with sigma = 0 (plms.py:30,319-338).  order 1..4: e' from e_t and the
// order - 1 held values h1 (most recent), h2, h3; order 0: the first step's average (h1 + e_t) / 2, h1 = the e_t of
// that step's first evaluation.  Multiplications, sums and the final division are rounded one by one in the reference's
// order (no contraction into FMAs), the CFG combine and the update included: the AB coefficients sum to up to 160 / 24
// in absolute value.
// Algorithmic traffic: read x, e_u, e_c, order - 1 held values; write x_prev (+ e_t, + pred_x0) = 32 B / element at
// order 4 with e_t stored.
__global__ void __launch_bounds__(256) plms_step_kernel(const float4* __restrict__ x, const float4* __restrict__ eu,
                                                        const float4* __restrict__ ec, const float4* __restrict__ h1,
                                                        const float4* __restrict__ h2, const float4* __restrict__ h3,
                                                        float4* __restrict__ et_out, float4* __restrict__ xp,
                                                        float4* __restrict__ px0, long long n4, int order, PlmsCoef c) {
  pdl_wait();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 X = __ldcs(x + i), U = __ldcs(eu + i), Cn = __ldcs(ec + i);
    float4 E, A = {}, B = {}, D = {}, P, O;
    if (order == 0 || order >= 2) A = __ldcs(h1 + i);
    if (order >= 3) B = __ldcs(h2 + i);
    if (order >= 4) D = __ldcs(h3 + i);
#define ALDM_PLMS1(f)                                                                                          \
    {                                                                                                          \
      const float e = __fadd_rn(U.f, __fmul_rn(c.g, __fsub_rn(Cn.f, U.f)));                                    \
      E.f = e;                                                                                                 \
      float ep;                                                                                                \
      if (order == 0)                                                                                          \
        ep = __fdiv_rn(__fadd_rn(A.f, e), 2.0f);                                                               \
      else if (order == 1)                                                                                     \
        ep = e;                                                                                                \
      else if (order == 2)                                                                                     \
        ep = __fdiv_rn(__fsub_rn(__fmul_rn(3.0f, e), A.f), 2.0f);                                              \
      else if (order == 3)                                                                                     \
        ep = __fdiv_rn(__fadd_rn(__fsub_rn(__fmul_rn(23.0f, e), __fmul_rn(16.0f, A.f)), __fmul_rn(5.0f, B.f)), \
                       12.0f);                                                                                 \
      else                                                                                                     \
        ep = __fdiv_rn(__fsub_rn(__fadd_rn(__fsub_rn(__fmul_rn(55.0f, e), __fmul_rn(59.0f, A.f)),              \
                                           __fmul_rn(37.0f, B.f)),                                             \
                                 __fmul_rn(9.0f, D.f)),                                                        \
                       24.0f);                                                                                 \
      const float p0 = __fdiv_rn(__fsub_rn(X.f, __fmul_rn(c.s1m, ep)), c.sqrt_at);                             \
      P.f = p0;                                                                                                \
      O.f = __fadd_rn(__fmul_rn(c.sqrt_aprev, p0), __fmul_rn(c.dir, ep));                                      \
    }
    ALDM_PLMS1(x) ALDM_PLMS1(y) ALDM_PLMS1(z) ALDM_PLMS1(w)
#undef ALDM_PLMS1
    if (et_out) et_out[i] = E;
    xp[i] = O;
    if (px0) px0[i] = P;
  }
}

}  // namespace aldm

using namespace aldm;

extern "C" int aldm_plms_step(const float* x, const float* eps_uncond, const float* eps_cond, const float* held1,
                              const float* held2, const float* held3, int32_t order, float* e_t_out, float* x_prev,
                              float* pred_x0, int64_t n_total, float a_t, float a_prev, float sqrt_one_minus_at,
                              float guidance, void* stream) {
  ALDM_REQUIRE(x && eps_uncond && eps_cond && x_prev, ALDM_E_ARG, "plms_step: null pointer");
  ALDM_REQUIRE(order >= ALDM_PLMS_AVERAGE && order <= 4, ALDM_E_ARG, "plms_step: order=%d (0 = first-step average, 1..4)",
               order);
  ALDM_REQUIRE((order != ALDM_PLMS_AVERAGE && order < 2) || held1, ALDM_E_ARG, "plms_step: order %d needs held1", order);
  ALDM_REQUIRE(order < 3 || held2, ALDM_E_ARG, "plms_step: order %d needs held2", order);
  ALDM_REQUIRE(order < 4 || held3, ALDM_E_ARG, "plms_step: order 4 needs held3");
  ALDM_REQUIRE(order != ALDM_PLMS_AVERAGE || !e_t_out, ALDM_E_ARG,
               "plms_step: the first-step average stores nothing (e_t_out must be NULL)");
  ALDM_REQUIRE(n_total > 0 && n_total % 4 == 0, ALDM_E_SHAPE, "plms_step: n_total=%lld must be a positive multiple of 4",
               (long long)n_total);
  ALDM_REQUIRE(aligned16(x) && aligned16(eps_uncond) && aligned16(eps_cond) && aligned16(x_prev) &&
                   (!held1 || aligned16(held1)) && (!held2 || aligned16(held2)) && (!held3 || aligned16(held3)) &&
                   (!e_t_out || aligned16(e_t_out)) && (!pred_x0 || aligned16(pred_x0)),
               ALDM_E_ALIGN, "plms_step: pointers must be 16B aligned");
  PlmsCoef c;
  // the fp32 evaluation order of get_x_prev_and_pred_x0 with sigma = 0: a_t.sqrt(), (1 - a_prev - 0^2).sqrt(), a_prev.sqrt()
  c.sqrt_at = sqrtf(a_t);                  // a divisor, as `/ a_t.sqrt()` (plms.py:329)
  c.s1m = sqrt_one_minus_at;
  c.sqrt_aprev = sqrtf(a_prev);
  c.dir = sqrtf(1.0f - a_prev);
  c.g = guidance;
  const long long n4 = n_total / 4;
  long long blocks = (n4 + 255) / 256;
  if (blocks > num_sms() * 8) blocks = num_sms() * 8;
  plms_step_kernel<<<(unsigned)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float4*>(x), reinterpret_cast<const float4*>(eps_uncond),
      reinterpret_cast<const float4*>(eps_cond), reinterpret_cast<const float4*>(held1),
      reinterpret_cast<const float4*>(held2), reinterpret_cast<const float4*>(held3), reinterpret_cast<float4*>(e_t_out),
      reinterpret_cast<float4*>(x_prev), reinterpret_cast<float4*>(pred_x0), n4, order, c);
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}
