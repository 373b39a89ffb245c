// Shared device helpers for the sm_90a kernels: PTX wrappers (mbarrier, cp.async, bulk copy,
// wgmma), fp16 hi/lo splitting, error plumbing.
#pragma once

#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/aldm_b200.h"

namespace aldm {

void set_error(const char* fmt, ...);

#define ALDM_CHECK_CUDA(expr)                                                        \
  do {                                                                               \
    cudaError_t _e = (expr);                                                         \
    if (_e != cudaSuccess) {                                                         \
      ::aldm::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return ALDM_E_CUDA;                                                            \
    }                                                                                \
  } while (0)

#define ALDM_REQUIRE(cond, code, ...)                                                \
  do {                                                                               \
    if (!(cond)) {                                                                   \
      ::aldm::set_error(__VA_ARGS__);                                                \
      return (code);                                                                 \
    }                                                                                \
  } while (0)

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
inline int cdiv(int a, int b) { return (a + b - 1) / b; }

// ---- programmatic dependent launch (PDL) ----------------------------------------------------
// Every kernel of the per-step programs is launched with programmatic stream serialisation: it may
// start (block scheduling, barrier init, index set-up) while its predecessor drains, and calls pdl_wait()
// before its first global-memory access, which blocks until the predecessor has completed and flushed.
// Because every such kernel waits, completion stays transitive along the stream (kernel k+2 cannot pass
// its wait before kernel k is done).  pdl_launch() is issued LATE (last MMA issued / last loads done), so
// that dependent blocks are co-resident with the primary only for its tail rather than its whole run.
// ALDM_PDL=0 in the environment disables the launch attribute (the device instructions are then no-ops).
bool pdl_enabled();
// streaming multiprocessors of the current device (grid sizing of the persistent and grid-stride kernels)
int num_sms();
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// ------------------------------------------------------------------------------------------
// fp16 operand planes.  hi = fp16(x) carries 11 significand bits; lo = fp16(x - hi) adds 11 more (|x - hi - lo| <=
// 2^-22 |x| while lo stays normal, <= 2^-25 absolute once it is subnormal).  Two-plane operands feed three tensor-core
// passes (hi*hi + hi*lo + lo*hi), single-plane activations two (hi*w_hi + hi*w_lo).  Inputs saturate at the fp16 range
// (+-65504) so that x - hi can never be inf - inf; activations behind a normalisation / gating stay far inside it.
// ------------------------------------------------------------------------------------------
typedef __half aldm_plane_t;
__device__ __forceinline__ float sat_f16(float x) { return fminf(fmaxf(x, -65504.0f), 65504.0f); }
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
  a = sat_f16(a);
  b = sat_f16(b);
  const __half2 h = __floats2half2_rn(a, b);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn(a - hf.x, b - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}
__device__ __forceinline__ uint32_t pack2_hi(float a, float b) {       // hi plane only
  const __half2 h = __floats2half2_rn(sat_f16(a), sat_f16(b));
  return *reinterpret_cast<const uint32_t*>(&h);
}
__device__ __forceinline__ float2 unpack2(uint32_t v) { return __half22float2(*reinterpret_cast<const __half2*>(&v)); }
__device__ __forceinline__ float plane_to_f(aldm_plane_t v) { return __half2float(v); }
// scalar element store: hi (and lo when the operand has a second plane)
__device__ __forceinline__ void store_split1(aldm_plane_t* hp, aldm_plane_t* lp, long long i, float v) {
  v = sat_f16(v);
  const __half h = __float2half_rn(v);
  hp[i] = h;
  if (lp) lp[i] = __float2half_rn(v - __half2float(h));
}

// 8 consecutive floats -> one 16-byte chunk of hi and one of lo
__device__ __forceinline__ void split8(const float* v, uint4& hi, uint4& lo) {
  split2(v[0], v[1], hi.x, lo.x);
  split2(v[2], v[3], hi.y, lo.y);
  split2(v[4], v[5], hi.z, lo.z);
  split2(v[6], v[7], hi.w, lo.w);
}
// same without the fp16-range clamp, for values known to lie in [0, 1] (softmax probabilities): the clamp is two FMNMX per
// element, a fifth of the attention softmax loop's instructions
__device__ __forceinline__ uint4 pack8_hi_unit(const float* v) {
  uint4 r;
  __half2 h;
  h = __floats2half2_rn(v[0], v[1]); r.x = *reinterpret_cast<const uint32_t*>(&h);
  h = __floats2half2_rn(v[2], v[3]); r.y = *reinterpret_cast<const uint32_t*>(&h);
  h = __floats2half2_rn(v[4], v[5]); r.z = *reinterpret_cast<const uint32_t*>(&h);
  h = __floats2half2_rn(v[6], v[7]); r.w = *reinterpret_cast<const uint32_t*>(&h);
  return r;
}
__device__ __forceinline__ uint4 pack8_hi(const float* v) {
  return make_uint4(pack2_hi(v[0], v[1]), pack2_hi(v[2], v[3]), pack2_hi(v[4], v[5]), pack2_hi(v[6], v[7]));
}

// x * sigmoid(x) with approximate reciprocal (the IEEE division expands to ~20 instructions with a guarded slow path;
// the GroupNorm+SiLU apply kernel is issue-bound on it).  ~2 ulp, far below the 2^-17 operand split that follows.
__device__ __forceinline__ float silu_f(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
// erf GELU as F.gelu default (attention.py:44).  erf via Abramowitz-Stegun 7.1.26 (|err| < 5e-7 in fp32,
// i.e. at fp32 round-off of the GELU output): 1 RCP + 1 EX2 + 8 FMA-class instructions instead of the
// ~40-instruction erff -- the GEGLU epilogue is issue-bound.
__device__ __forceinline__ float gelu_f(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  float t;      // rcp.approx (1 MUFU, ~1 ulp): __frcp_rn expands to MUFU + Newton step + a guarded slow-path CALL per element
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  p *= t;
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-z * z * 1.4426950408889634f));
  const float erf_abs = fmaf(-p, e, 1.0f);
  return 0.5f * x + 0.5f * fabsf(x) * erf_abs;     // 0.5 x (1 + sign(x) erf(|x|/sqrt2))
}

// GPT-2's gelu_new (activations.py NewGELUActivation): 0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3))) with the accurate
// tanhf, in the order of the module's expression.
__device__ __forceinline__ float gelu_tanh_f(float x) {
  return 0.5f * x * (1.0f + tanhf(0.7978845608028654f * (x + 0.044715f * (x * x * x))));
}

// v[i] *= gelu(g[i]) for NB values at once, written stage by stage so that NB independent dependency chains are in
// flight: the GEGLU epilogue runs two warps per scheduler, and with the elements evaluated one or two at a time
// (what the compiler produces from the scalar form under the 128-register cap) the dependency chain of each element
// (two MUFU round trips) is fully exposed.
template <int NB>
__device__ __forceinline__ void geglu_mul(float* __restrict__ v, const float* __restrict__ g) {
  float z[NB], t[NB], e[NB], p[NB];
#pragma unroll
  for (int j = 0; j < NB; ++j) z[j] = fabsf(g[j]) * 0.70710678118654752440f;
#pragma unroll
  for (int j = 0; j < NB; ++j) asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t[j]) : "f"(fmaf(0.3275911f, z[j], 1.0f)));
#pragma unroll
  for (int j = 0; j < NB; ++j) asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e[j]) : "f"(-z[j] * z[j] * 1.4426950408889634f));
#pragma unroll
  for (int j = 0; j < NB; ++j) p[j] = fmaf(1.061405429f, t[j], -1.453152027f);
#pragma unroll
  for (int j = 0; j < NB; ++j) p[j] = fmaf(p[j], t[j], 1.421413741f);
#pragma unroll
  for (int j = 0; j < NB; ++j) p[j] = fmaf(p[j], t[j], -0.284496736f);
#pragma unroll
  for (int j = 0; j < NB; ++j) p[j] = fmaf(p[j], t[j], 0.254829592f);
#pragma unroll
  for (int j = 0; j < NB; ++j) p[j] *= t[j] * e[j];
#pragma unroll
  for (int j = 0; j < NB; ++j) {
    const float erf_abs = 1.0f - p[j];
    v[j] *= fmaf(0.5f * fabsf(g[j]), erf_abs, 0.5f * g[j]);      // 0.5 g (1 + sign(g) erf(|g| / sqrt 2))
  }
}

// ------------------------------------------------------------------------------------------
// shared-memory address + mbarrier
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// Bounded wait: a protocol bug must become a CUDA error (a trap after 4 s), never a hung GPU.  The timer is
// only consulted every 4096 failed probes (try_wait itself suspends the thread in hardware), so the hot path
// is a bare try_wait loop.  No printf here: a call inside the wgmma consumer loops makes ptxas serialise the
// asynchronous MMAs across it.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  uint64_t t0 = 0;
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 4095u) == 0) {
      const uint64_t now = globaltimer_ns();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 4000000000ull) __trap();   // 4 s
    }
  }
}

// non-blocking probe (mbarrier.test_wait never suspends the thread)
__device__ __forceinline__ bool mbar_test_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// pure spin variant for latency-critical single-thread waits
__device__ __forceinline__ void mbar_wait_spin(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_test_wait(bar, parity)) {
    if (++spins > (1u << 28)) __trap();
  }
}

// ------------------------------------------------------------------------------------------
// cp.async (LDGSTS) 16-byte with zero fill, completion signalled on an mbarrier
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void cp_async_16(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
// same with an immediate destination offset (one base register for the eight rows a producer thread copies per k-block)
template <int OFF>
__device__ __forceinline__ void cp_async_16_off(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0 + %3], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes), "n"(OFF) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait_group() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ void cp_async_mbar_arrive_noinc(uint32_t bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}
// TMA bulk copy global -> shared, completion (bytes) on an mbarrier
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
// 2-D tiled tensor-map load (TMA): box lands in shared memory in the map's swizzle mode; completes on `mbar` (tx bytes)
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const void* tensor_map, int c0, int c1, uint32_t mbar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(tensor_map)), "r"(mbar), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// One elected lane of a fully converged warp, for the single-thread roles (TMA bulk copies).  Under a plain `lane == 0`
// predicate the compiler cannot prove uniformity of the operands those instructions take from uniform registers.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.b32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}

// ------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA): 64 x N x 16 per warpgroup, fp16 operands, fp32 accumulators in registers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// The accumulator registers are read and written by the asynchronous MMA: this keeps the compiler from moving
// their uses across wgmma_commit / wgmma_wait.
template <int NR>
__device__ __forceinline__ void wgmma_fence_regs(float* d) {
#pragma unroll
  for (int i = 0; i < NR; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// K-major, 128-byte-swizzled operand tile descriptor (rows of 128 B, 8-row groups 1024 B apart; tile base 1024-aligned).
// Field layout (PTX ISA, "Matrix Descriptor Format" of wgmma): start>>4 [0,14), LBO>>4 [16,30) (unused for swizzled
// K-major: 1), SBO>>4 [32,46) = 1024 B, layout type [62,64) with SWIZZLE_128B = 1.  +2 on the descriptor = next 16 fp16 of K.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
  return static_cast<uint64_t>((smem_addr >> 4) & 0x3FFFu) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}

// D (+)= A[smem] * B[smem]^T, both K-major; scale_d == 0 overwrites D.  Accumulator fragment of thread (warp w of the
// warpgroup, lane = 4 g + t): d[4 j + {0,1}] = row 16 w + g, columns 8 j + 2 t + {0,1}; d[4 j + {2,3}] = row + 8, same columns.
template <int N>
__device__ __forceinline__ void wgmma_ss(float* d, uint64_t da, uint64_t db, uint32_t scale_d);
template <>
__device__ __forceinline__ void wgmma_ss<32>(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma_ss<64>(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma_ss<128>(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <int N>
__device__ __forceinline__ void wgmma_rs(float* d, const uint32_t* a, uint64_t db, uint32_t scale_d);
template <>
__device__ __forceinline__ void wgmma_rs<32>(float* d, const uint32_t* a, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}

}  // namespace aldm
