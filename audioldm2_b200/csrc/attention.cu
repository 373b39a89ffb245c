// K5: fused softmax(scale * Q K^T + mask) V, head_dim 32, flash-style (no N x N score matrix in HBM;
// the reference materialises it: attention.py:354-366).
//
// attention_tc_kernel (wgmma): one CTA = 128 queries of one (batch, head); keys are streamed in
// tiles of 64.  Operands are single fp16 planes (the hi planes written by the projection GEMMs,
// ALDM_OUT_QKV): Q, K row-major, V already transposed (keys contiguous), so every operand tile is
// a plain cp.async copy into the same 128-byte-swizzled K-major layout the GEMM uses.
// attention_short_kernel: CUDA cores, for the <= 32-key cross-attention contexts.
// attention_simt_kernel: CUDA-core checker on the same operands (validation only).
// softmax_rows_kernel: row softmax for the VAE AttnBlock (model.py:216-217).
#include <float.h>
#include <stdlib.h>

#include "common.cuh"

namespace aldm {

static constexpr int ATT_D = 32;

// ------------------------------------------------------------------------------------------------
// wgmma flash attention
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// one query row of one head -> output plane(s) (lo only when the consumer asked for a second plane)
__device__ __forceinline__ void store_out_row(const aldm_attn_desc& d, long long orow, int h, const float* o) {
  aldm_plane_t* hp = reinterpret_cast<aldm_plane_t*>(d.out_hi) + orow * d.ldo + h * ATT_D;
  aldm_plane_t* lp = d.out_lo ? reinterpret_cast<aldm_plane_t*>(d.out_lo) + orow * d.ldo + h * ATT_D : nullptr;
#pragma unroll
  for (int i = 0; i < ATT_D; i += 8) {
    uint4 hh, ll;
    split8(o + i, hh, ll);
    *reinterpret_cast<uint4*>(hp + i) = hh;
    if (lp) *reinterpret_cast<uint4*>(lp + i) = ll;
  }
}

namespace atc {
constexpr int QT = 128, KT = 64, NS = 4;
// Rows are 128 bytes in the SWIZZLE_128B layout; Q and K use the first 64 bytes of each row (32 dims x fp16), V^T all 128
// (64 keys).  P never touches shared memory: the score accumulator is repacked in registers as the A operand of P V.
constexpr int QA = 0;                           // [128][128B]
constexpr int KB = QA + QT * 128;               // NS x [64][128B]
constexpr int VT = KB + NS * KT * 128;          // NS x [32][128B]
constexpr int BAR = VT + NS * ATT_D * 128;
constexpr int SMEM = BAR + 128 + 1024;          // + barriers + round-up slack for the 1024-byte tile alignment
}  // namespace atc

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}

// One CTA = 128 queries of one (batch, head); keys are streamed in tiles of 64 by a loader warp (cp.async + mbarrier, NS
// stages).  Warps 0-7 are two warpgroups of 64 queries each; per key tile a warpgroup computes
//   S = Q K^T        (2 wgmma m64n64k16, operands in shared memory)
//   online softmax   on the accumulator fragment: thread (warp w, lane 4 g + t) holds rows 16 w + g and 16 w + g + 8,
//                    16 keys each; row maxima are combined over the 4 threads of a row with two shuffles
//   O += P V         (4 wgmma m64n32k16, P as fp16 register operand, V^T from shared memory)
// Both operands of the two products are activations; rounding them to 11 bits costs 1.2e-4 of the 1e-3 waveform budget
// at 10 DDIM steps (scripts/precision_study.py --only attn).  The row sum is accumulated from the unrounded values.
__global__ void __launch_bounds__(288, 2) attention_tc_kernel(const __grid_constant__ aldm_attn_desc d) {
  using namespace atc;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const uint32_t bar = base + BAR;
  const uint32_t q_full = bar, kv_full0 = bar + 8, kv_empty0 = kv_full0 + 8 * NS;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * QT;
  const int bkv = d.kv_bmod > 0 ? b % d.kv_bmod : b;
  const int nt = (d.Nk + KT - 1) / KT;

  if (tid == 0) {
    // one arrival per WARP everywhere (per-thread arrivals on one mbarrier word serialise in the smem atomic unit)
    mbar_init(q_full, 32);
    for (int i = 0; i < NS; ++i) { mbar_init(kv_full0 + 8 * i, 32); mbar_init(kv_empty0 + 8 * i, 8); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();

  if (warp < 8) {
    // =============================== S, softmax, P V ===============================
    const int wg = warp >> 2, g = lane >> 2, t = lane & 3;
    const int rloc = wg * 64 + (warp & 3) * 16 + g;      // this thread's first query row in the tile (second: + 8)
    const float sl2 = d.scale * 1.4426950408889634f;
    const float* mrow = d.mask ? d.mask + (long long)bkv * d.Nk : nullptr;
    const uint64_t dQ = wgmma_desc_sw128(base + QA + wg * 64 * 128);
    float o[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) o[i] = 0.f;
    float mrun[2] = {-INFINITY, -INFINITY}, lrun[2] = {0.f, 0.f};
    mbar_wait(q_full, 0);
    for (int it = 0; it < nt; ++it) {
      const int k0 = it * KT, st = it % NS;
      mbar_wait(kv_full0 + 8 * st, (it / NS) & 1);
      fence_proxy_async();          // cp.async-written tiles -> visible to the tensor core (async proxy)
      float s[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) s[i] = 0.f;
      const uint64_t dK = wgmma_desc_sw128(base + KB + st * (KT * 128));
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) wgmma_ss<KT>(s, dQ + 2 * ks, dK + 2 * ks, 1);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs<32>(s);
      // s[4 j + 2 hr + e]: row rloc + 8 hr, key k0 + 8 j + 2 t + e
      float mnew[2], corr[2];
      if (k0 + KT <= d.Nk && !mrow) {
        // interior tile, no mask: max on the raw scores (sl2 > 0), one FFMA + one MUFU per element
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          float tmax = s[2 * hr];
#pragma unroll
          for (int j = 0; j < 8; ++j) tmax = fmaxf(tmax, fmaxf(s[4 * j + 2 * hr], s[4 * j + 2 * hr + 1]));
          tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 1));
          tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 2));
          mnew[hr] = fmaxf(mrun[hr], tmax * sl2);
          corr[hr] = ex2_approx(mrun[hr] - mnew[hr]);      // mrun = -inf on the first tile -> 0
#pragma unroll
          for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) s[4 * j + 2 * hr + e] = ex2_approx(fmaf(s[4 * j + 2 * hr + e], sl2, -mnew[hr]));
        }
      } else {
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          float tmax = -INFINITY;
#pragma unroll
          for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int key = k0 + 8 * j + 2 * t + e;
              float v = s[4 * j + 2 * hr + e] * sl2;
              if (key >= d.Nk) v = -INFINITY;                               // beyond the key range: excluded
              else if (mrow && __ldg(mrow + key) != 1.0f) v = -FLT_MAX;     // masked_fill(-finfo.max), attention.py:356-360
              s[4 * j + 2 * hr + e] = v;
              tmax = fmaxf(tmax, v);
            }
          tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 1));
          tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 2));
          mnew[hr] = fmaxf(mrun[hr], tmax);
          corr[hr] = (mrun[hr] == -INFINITY) ? 0.f : ex2_approx(mrun[hr] - mnew[hr]);
#pragma unroll
          for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float v = s[4 * j + 2 * hr + e];
              s[4 * j + 2 * hr + e] = (v == -INFINITY) ? 0.f : ex2_approx(v - mnew[hr]);
            }
        }
      }
      // row sums (this thread's 16 keys per row; the 4 threads of a row are combined once at the end) and O rescale
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        float ps = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) ps += s[4 * j + 2 * hr] + s[4 * j + 2 * hr + 1];
        lrun[hr] = lrun[hr] * corr[hr] + ps;
        mrun[hr] = mnew[hr];
#pragma unroll
        for (int j = 0; j < 4; ++j) { o[4 * j + 2 * hr] *= corr[hr]; o[4 * j + 2 * hr + 1] *= corr[hr]; }
      }
      // P as the A operand (fp16): k16 chunk kc covers keys 16 kc .. 16 kc + 15 = accumulator column blocks 2 kc, 2 kc + 1
      uint32_t pa[4][4];
#pragma unroll
      for (int kc = 0; kc < 4; ++kc) {
        pa[kc][0] = pack_half2(s[8 * kc + 0], s[8 * kc + 1]);
        pa[kc][1] = pack_half2(s[8 * kc + 2], s[8 * kc + 3]);
        pa[kc][2] = pack_half2(s[8 * kc + 4], s[8 * kc + 5]);
        pa[kc][3] = pack_half2(s[8 * kc + 6], s[8 * kc + 7]);
      }
      const uint64_t dV = wgmma_desc_sw128(base + VT + st * (ATT_D * 128));
      wgmma_fence();
#pragma unroll
      for (int kc = 0; kc < 4; ++kc) wgmma_rs<ATT_D>(o, pa[kc], dV + 2 * kc, 1);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs<16>(o);
      __syncwarp();
      if (lane == 0) mbar_arrive(kv_empty0 + 8 * st);      // this warp's reads of stage st are complete
    }
    if (tid == 0) pdl_launch();
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      float l = lrun[hr];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      const int q = q0 + rloc + 8 * hr;
      if (q < d.Nq) {
        const float inv = 1.0f / l;
        const long long orow = (long long)b * d.Nq + q;
        aldm_plane_t* hp = reinterpret_cast<aldm_plane_t*>(d.out_hi) + orow * d.ldo + h * ATT_D + 2 * t;
        aldm_plane_t* lp = d.out_lo ? reinterpret_cast<aldm_plane_t*>(d.out_lo) + orow * d.ldo + h * ATT_D + 2 * t : nullptr;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          uint32_t hh, ll;
          split2(o[4 * j + 2 * hr] * inv, o[4 * j + 2 * hr + 1] * inv, hh, ll);
          *reinterpret_cast<uint32_t*>(hp + 8 * j) = hh;
          if (lp) *reinterpret_cast<uint32_t*>(lp + 8 * j) = ll;
        }
      }
    }
  } else {
    // =============================== loader ===============================
    const aldm_plane_t* qh = reinterpret_cast<const aldm_plane_t*>(d.q_hi);
    const aldm_plane_t* kh = reinterpret_cast<const aldm_plane_t*>(d.k_hi);
    const aldm_plane_t* vh = reinterpret_cast<const aldm_plane_t*>(d.vt_hi);
    // Q: row r, chunks 0..3 (32 dims)
    for (int idx = lane; idx < QT * 4; idx += 32) {
      const int r = idx >> 2, c = idx & 3;
      const bool ok = q0 + r < d.Nq;
      const long long off = ok ? ((long long)b * d.Nq + q0 + r) * d.ldq + d.q_col + h * ATT_D + c * 8 : 0;
      cp_async_16(base + QA + r * 128 + ((uint32_t)(c ^ (r & 7)) << 4), qh + off, ok ? 16u : 0u);
    }
    cp_async_mbar_arrive_noinc(q_full);
    // K/V tiles: all row bases are hoisted out of the tile loop (the loader is a single warp: per-element 64-bit index
    // arithmetic was the bottleneck).  K: lane -> chunk ck (of 4), rows rk + 8i; V^T: lane -> chunk cv (of 8), rows rv + 4i.
    // Keys beyond Nk are zero-filled (K: finite scores that the softmax excludes; V^T: zero rows of P V).
    const int ck = lane & 3, rk = lane >> 2;
    const int cv = lane & 7, rv = lane >> 3;
    const aldm_plane_t* kcol = kh + (long long)bkv * d.Nk * d.ldk + d.k_col + h * ATT_D + ck * 8;
    const long long vrow0 = ((long long)(bkv * d.heads + h) * ATT_D + rv) * d.ld_t + cv * 8;
    const long long kstep = 8ll * d.ldk, vstep = 4ll * d.ld_t;
    for (int it = 0, s = 0, ph = 1; it < nt; ++it) {
      const int k0 = it * KT;
      mbar_wait(kv_empty0 + 8 * s, ph);
      const uint32_t kb = base + KB + s * (KT * 128);
      const aldm_plane_t* kp = kcol + (long long)(k0 + rk) * d.ldk;
#pragma unroll
      for (int i = 0; i < KT / 8; ++i) {
        const int r = rk + 8 * i;
        const bool ok = k0 + r < d.Nk;
        cp_async_16(kb + r * 128 + ((uint32_t)(ck ^ (r & 7)) << 4), ok ? kp + i * kstep : kcol, ok ? 16u : 0u);
      }
      const uint32_t vb = base + VT + s * (ATT_D * 128);
      const bool vok = k0 + cv * 8 < d.Nk;
#pragma unroll
      for (int i = 0; i < ATT_D / 4; ++i) {
        const int r = rv + 4 * i;
        const aldm_plane_t* vp = vh + vrow0 + i * vstep + k0;
        cp_async_16(vb + r * 128 + ((uint32_t)(cv ^ (r & 7)) << 4), vok ? vp : vh, vok ? 16u : 0u);
      }
      cp_async_mbar_arrive_noinc(kv_full0 + 8 * s);
      if (++s == NS) { s = 0; ph ^= 1; }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Short key sets (cross-attention to the 8-token CLAP/GPT-2 and 32-token T5 contexts): Nk <= 32.
// The tensor-core kernel would pay its whole fixed cost (mbarrier hand-overs, two MMA round trips, a 64-key
// tile that is mostly padding) for ~0.1 GFLOP, 32 times per DDIM step.  Here one thread owns one query, K and V of the (batch, head) sit in shared memory as
// fp32 (converted from their fp16 planes), and the 2 x Nk x 32 FMAs per query run on the CUDA cores.
// ------------------------------------------------------------------------------------------------
template <int NKT>
__global__ void __launch_bounds__(128) attention_short_kernel(const __grid_constant__ aldm_attn_desc d) {
  __shared__ __align__(16) float sk[NKT][ATT_D];
  __shared__ __align__(16) float sv[NKT][ATT_D];
  __shared__ int sstate[NKT];        // 0 = attend, 1 = masked (-FLT_MAX fill), 2 = beyond Nk
  const int tid = threadIdx.x;
  const int b = blockIdx.z, h = blockIdx.y;
  const int bkv = d.kv_bmod > 0 ? b % d.kv_bmod : b;
  pdl_wait();
  {
    const aldm_plane_t* kh = reinterpret_cast<const aldm_plane_t*>(d.k_hi);
    const aldm_plane_t* vh = reinterpret_cast<const aldm_plane_t*>(d.vt_hi);
    for (int idx = tid; idx < NKT * ATT_D; idx += 128) {
      const int key = idx / ATT_D, dim = idx % ATT_D;
      float kv = 0.f, vv = 0.f;
      if (key < d.Nk) {
        const long long ki = ((long long)bkv * d.Nk + key) * d.ldk + d.k_col + h * ATT_D + dim;
        const long long vi = ((long long)(bkv * d.heads + h) * ATT_D + dim) * d.ld_t + key;
        kv = plane_to_f(kh[ki]);
        vv = plane_to_f(vh[vi]);
      }
      sk[key][dim] = kv;
      sv[key][dim] = vv;
    }
    if (tid < NKT) sstate[tid] = tid >= d.Nk ? 2 : ((d.mask && __ldg(d.mask + (long long)bkv * d.Nk + tid) != 1.0f) ? 1 : 0);
  }
  __syncthreads();
  pdl_launch();
  const int q = blockIdx.x * 128 + tid;
  if (q >= d.Nq) return;
  float qv[ATT_D];
  {
    const long long qi = ((long long)b * d.Nq + q) * d.ldq + d.q_col + h * ATT_D;
    const uint4* ph = reinterpret_cast<const uint4*>(reinterpret_cast<const aldm_plane_t*>(d.q_hi) + qi);
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const uint4 a = __ldg(ph + c);
      const uint32_t aw[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = unpack2(aw[e]);
        qv[c * 8 + 2 * e] = f.x;
        qv[c * 8 + 2 * e + 1] = f.y;
      }
    }
  }
  const float sl2 = d.scale * 1.4426950408889634f;
  float sc[NKT];
  float mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < NKT; ++k) {
    float acc = 0.f;
#pragma unroll
    for (int dd = 0; dd < ATT_D; dd += 4) {
      const float4 kk = *reinterpret_cast<const float4*>(&sk[k][dd]);
      acc = fmaf(qv[dd], kk.x, acc); acc = fmaf(qv[dd + 1], kk.y, acc);
      acc = fmaf(qv[dd + 2], kk.z, acc); acc = fmaf(qv[dd + 3], kk.w, acc);
    }
    const int st = sstate[k];
    const float v = st == 0 ? acc * sl2 : (st == 1 ? -FLT_MAX : -INFINITY);   // masked_fill(-finfo.max), attention.py:356-360
    sc[k] = v;
    mx = fmaxf(mx, v);
  }
  float l = 0.f;
#pragma unroll
  for (int k = 0; k < NKT; ++k) {
    const float pk = sc[k] == -INFINITY ? 0.f : ex2_approx(sc[k] - mx);
    sc[k] = pk;
    l += pk;
  }
  float o[ATT_D];
#pragma unroll
  for (int i = 0; i < ATT_D; ++i) o[i] = 0.f;
#pragma unroll
  for (int k = 0; k < NKT; ++k) {
#pragma unroll
    for (int dd = 0; dd < ATT_D; dd += 4) {
      const float4 vv = *reinterpret_cast<const float4*>(&sv[k][dd]);
      o[dd] = fmaf(sc[k], vv.x, o[dd]); o[dd + 1] = fmaf(sc[k], vv.y, o[dd + 1]);
      o[dd + 2] = fmaf(sc[k], vv.z, o[dd + 2]); o[dd + 3] = fmaf(sc[k], vv.w, o[dd + 3]);
    }
  }
  const float inv = 1.0f / l;
#pragma unroll
  for (int i = 0; i < ATT_D; ++i) o[i] *= inv;
  store_out_row(d, (long long)b * d.Nq + q, h, o);
}

// ------------------------------------------------------------------------------------------------
// CUDA-core checker on the same plane operands: one thread per query, fp32
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) attention_simt_kernel(const __grid_constant__ aldm_attn_desc d) {
  const int b = blockIdx.z, h = blockIdx.y;
  const int qi = blockIdx.x * blockDim.x + threadIdx.x;
  if (qi >= d.Nq) return;
  const int bkv = d.kv_bmod > 0 ? b % d.kv_bmod : b;
  auto ld = [](const void* hi, const void* /*lo: the attention operands are single-plane*/, long long i) {
    return plane_to_f(reinterpret_cast<const aldm_plane_t*>(hi)[i]);
  };
  float q[ATT_D], o[ATT_D];
  for (int i = 0; i < ATT_D; ++i) {
    q[i] = ld(d.q_hi, d.q_lo, ((long long)b * d.Nq + qi) * d.ldq + d.q_col + h * ATT_D + i) * d.scale;
    o[i] = 0.f;
  }
  float mrun = -INFINITY, lrun = 0.f;
  for (int k = 0; k < d.Nk; ++k) {
    float s = 0.f;
    const long long kr = ((long long)bkv * d.Nk + k) * d.ldk + d.k_col + h * ATT_D;
    for (int i = 0; i < ATT_D; ++i) s = fmaf(q[i], ld(d.k_hi, d.k_lo, kr + i), s);
    if (d.mask && d.mask[(long long)bkv * d.Nk + k] != 1.0f) s = -FLT_MAX;
    const float mnew = fmaxf(mrun, s);
    const float corr = (mrun == -INFINITY) ? 0.f : expf(mrun - mnew);
    const float p = expf(s - mnew);
    lrun = lrun * corr + p;
    for (int i = 0; i < ATT_D; ++i)
      o[i] = o[i] * corr + p * ld(d.vt_hi, d.vt_lo, ((long long)(bkv * d.heads + h) * ATT_D + i) * d.ld_t + k);
    mrun = mnew;
  }
  for (int i = 0; i < ATT_D; ++i) o[i] /= lrun;
  store_out_row(d, (long long)b * d.Nq + qi, h, o);
}

int attention_launch(const aldm_attn_desc& d, cudaStream_t st) {
  // single-plane operands: the *_lo inputs are ignored; out_lo is written only when non-NULL
  ALDM_REQUIRE(d.q_hi && d.k_hi && d.vt_hi && d.out_hi, ALDM_E_ARG, "attention: null pointer");
  ALDM_REQUIRE(d.B > 0 && d.heads > 0 && d.Nq > 0 && d.Nk > 0, ALDM_E_SHAPE, "attention: B=%d heads=%d Nq=%d Nk=%d", d.B,
               d.heads, d.Nq, d.Nk);
  ALDM_REQUIRE(d.ldq % 8 == 0 && d.ldk % 8 == 0 && d.ld_t % 8 == 0 && d.ldo % 8 == 0 && d.q_col % 8 == 0 && d.k_col % 8 == 0,
               ALDM_E_ALIGN, "attention: leading dims / column offsets must be multiples of 8");
  ALDM_REQUIRE(d.ld_t >= d.Nk, ALDM_E_SHAPE, "attention: ld_t=%d < Nk=%d", d.ld_t, d.Nk);
  ALDM_REQUIRE(aligned16(d.q_hi) && aligned16(d.k_hi) && aligned16(d.vt_hi) && aligned16(d.out_hi) && aligned16(d.out_lo),
               ALDM_E_ALIGN, "attention: pointers must be 16B aligned");
  ALDM_REQUIRE(d.heads <= 65535 && d.B <= 65535, ALDM_E_SHAPE, "attention: grid too large");
  if (d.impl == ALDM_GEMM_SIMT) {
    dim3 grid(cdiv(d.Nq, 128), d.heads, d.B);
    attention_simt_kernel<<<grid, 128, 0, st>>>(d);
  } else if (d.Nk <= 32 && !(getenv("ALDM_ATTN_SHORT") && getenv("ALDM_ATTN_SHORT")[0] == '0')) {
    dim3 grid(cdiv(d.Nq, 128), d.heads, d.B);
    if (d.Nk <= 8) ALDM_CHECK_CUDA(launch_pdl(attention_short_kernel<8>, grid, dim3(128), 0, st, d));
    else if (d.Nk <= 16) ALDM_CHECK_CUDA(launch_pdl(attention_short_kernel<16>, grid, dim3(128), 0, st, d));
    else ALDM_CHECK_CUDA(launch_pdl(attention_short_kernel<32>, grid, dim3(128), 0, st, d));
  } else {
    static bool configured = false;
    if (!configured) {      // ~65 KB: three CTAs per SM
      ALDM_CHECK_CUDA(cudaFuncSetAttribute(attention_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, atc::SMEM));
      configured = true;
    }
    dim3 grid(cdiv(d.Nq, atc::QT), d.heads, d.B);
    ALDM_CHECK_CUDA(launch_pdl(attention_tc_kernel, grid, dim3(288), atc::SMEM, st, d));
  }
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}

// row softmax of x[rows, n] (x already scaled when scale == 1) -> planes [rows, n]; one block per row
__global__ void softmax_rows_kernel(const float* __restrict__ x, int n, float scale, aldm_plane_t* __restrict__ hi,
                                    aldm_plane_t* __restrict__ lo) {
  __shared__ float red[32];
  const long long row = blockIdx.x;
  const float* xp = x + row * n;
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < n; i += blockDim.x) mx = fmaxf(mx, xp[i] * scale);
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
  for (int w = 1; w < (blockDim.x >> 5); ++w) mx = fmaxf(mx, red[w]);
  __syncthreads();
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s += expf(xp[i] * scale - mx);
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  s = 0.f;
  for (int w = 0; w < (blockDim.x >> 5); ++w) s += red[w];
  const float inv = 1.0f / s;
  for (int i = threadIdx.x * 2; i < n; i += blockDim.x * 2) {
    const float a = expf(xp[i] * scale - mx) * inv;
    const float b = (i + 1 < n) ? expf(xp[i + 1] * scale - mx) * inv : 0.f;
    uint32_t h, l;
    split2(a, b, h, l);
    if (i + 1 < n) {
      *reinterpret_cast<uint32_t*>(hi + row * n + i) = h;
      if (lo) *reinterpret_cast<uint32_t*>(lo + row * n + i) = l;
    } else {
      store_split1(hi, lo, row * n + i, a);
    }
  }
}

}  // namespace aldm

extern "C" int aldm_attention(const aldm_attn_desc* d, void* stream) {
  if (!d) { aldm::set_error("aldm_attention: null desc"); return ALDM_E_ARG; }
  return aldm::attention_launch(*d, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int aldm_softmax_rows(const float* x, int32_t rows, int32_t n, float scale, void* out_hi, void* out_lo,
                                 void* stream) {
  using namespace aldm;
  ALDM_REQUIRE(x && out_hi && rows > 0 && n > 0, ALDM_E_ARG, "softmax_rows: bad arguments");
  ALDM_REQUIRE(n % 2 == 0, ALDM_E_UNSUPPORTED, "softmax_rows: n must be even");
  softmax_rows_kernel<<<rows, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, n, scale, reinterpret_cast<aldm_plane_t*>(out_hi), reinterpret_cast<aldm_plane_t*>(out_lo));
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}
