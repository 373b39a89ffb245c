// K3: operand preparation -- GroupNorm / LayerNorm / SiLU / leaky-ReLU applied once per tensor and
// written as the fp16 operand plane(s) the tensor-core GEMM consumes (hi, and lo unless out_lo == NULL).  All kernels are
// HBM/L2-bound streaming kernels: float4 loads, 8/16-byte stores, warp-shuffle reductions.
//
//   GN  : gn_stats_kernel  (per-lane fp32 sums -> fixed-order double tree per block, no atomics, deterministic)
//         gn_apply_kernel  (reduces the partials for its batch row, builds per-channel scale/shift
//                           in shared memory, applies (+SiLU), splits, stores)
//   LN  : ln_kernel        (one warp per token row, two-pass statistics in registers)
//   misc: ew_kernel        (copy / SiLU / leaky-ReLU, optional concat of two sources, NCHW source)
//         pack_b_kernel    (fp32 matrix -> swizzled hi/lo weight tile images, for dynamic B operands)
#include <stdlib.h>

#include "common.cuh"

namespace aldm {

static constexpr int GN_MAX_BLOCKS = 64;   // partial-sum blocks per batch row
static constexpr int GN_MAX_C = 2048;

__device__ __forceinline__ float4 load_cat4(const aldm_prep_desc& d, long long row, int c) {
  // 4 consecutive channels starting at c (c % 4 == 0) of the concatenated tensor; c0 % 4 == 0
  if (c < d.c0) return *reinterpret_cast<const float4*>(d.src0 + row * d.c0 + c);
  return *reinterpret_cast<const float4*>(d.src1 + row * d.c1 + (c - d.c0));
}

// GroupNorm statistics are accumulated relative to a pivot, the first element of the (batch, group) (row 0, channel g * cpg):
// the per-thread fp32 sums of x and x^2 then hold values of the order of the group's spread rather than of its mean, so
// var = E[(x-p)^2] - E[x-p]^2 does not cancel when |mean| >> std (offset activations).
__device__ __forceinline__ float gn_pivot(const aldm_prep_desc& d, int b, int g, int cpg) {
  const int c = g * cpg;
  const long long row = (long long)b * d.HW;
  return c < d.c0 ? __ldg(d.src0 + row * d.c0 + c) : __ldg(d.src1 + row * d.c1 + (c - d.c0));
}
// (sum, sumsq) of x - pivot over n elements -> mean, rstd
__device__ __forceinline__ void gn_finish(double s, double s2, double n, float pivot, float eps, float& mean, float& rstd) {
  const double ms = s / n;
  double var = s2 / n - ms * ms;
  if (var < 0.0) var = 0.0;
  mean = (float)((double)pivot + ms);
  rstd = (float)(1.0 / sqrt(var + (double)eps));
}

// ---------------------------------------------------------------------------------------------
// GroupNorm statistics (generic path, any channels per group): grid (nblk, B); block 256 = 8 warps; warp w owns groups
// w, w + 8, ... of the block's rows.  Each lane accumulates its elements of the group in fp32, the lanes' sums are
// combined as doubles by a fixed shuffle tree, so the result does not depend on scheduling.
// partial[b][blk][g] = (sum, sumsq) of x - pivot as doubles.
// ---------------------------------------------------------------------------------------------
__global__ void gn_stats_kernel(const __grid_constant__ aldm_prep_desc d, int nblk) {
  pdl_wait();
  const int b = blockIdx.y, blk = blockIdx.x;
  const int C = d.c0 + d.c1, cpg = C / d.groups;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int rows_per = (d.HW + nblk - 1) / nblk;
  const int r0 = blk * rows_per;
  const int r1 = min(d.HW, r0 + rows_per);
  const int total = max(0, r1 - r0) * cpg;
  for (int g = warp; g < d.groups; g += nwarps) {
    const float pv = gn_pivot(d, b, g, cpg);
    float acc = 0.f, acc2 = 0.f;
    for (int idx = lane; idx < total; idx += 32) {
      const long long row = (long long)b * d.HW + r0 + idx / cpg;
      const int c = g * cpg + idx % cpg;
      const float x = (c < d.c0 ? __ldg(d.src0 + row * d.c0 + c) : __ldg(d.src1 + row * d.c1 + (c - d.c0))) - pv;
      acc += x;
      acc2 = fmaf(x, x, acc2);
    }
    double s = acc, s2 = acc2;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, o);
      s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    if (lane == 0) {
      double* p = d.scratch + (((long long)b * nblk + blk) * d.groups + g) * 2;
      p[0] = s;
      p[1] = s2;
    }
  }
}

// hp / lp: plane bases (lp may be NULL: single-plane operand), off: element offset
__device__ __forceinline__ void store_planes4(aldm_plane_t* hp, aldm_plane_t* lp, long long off, const float* y) {
  uint2 h, l;
  split2(y[0], y[1], h.x, l.x);
  split2(y[2], y[3], h.y, l.y);
  *reinterpret_cast<uint2*>(hp + off) = h;
  if (lp) *reinterpret_cast<uint2*>(lp + off) = l;
}

// grid (nblk_apply, B); block 256
__global__ void gn_apply_kernel(const __grid_constant__ aldm_prep_desc d, int nblk_stats) {
  pdl_wait();
  __shared__ float s_scale[GN_MAX_C], s_shift[GN_MAX_C];
  __shared__ float s_mean[32], s_rstd[32];
  const int b = blockIdx.y;
  const int C = d.c0 + d.c1, Q = C >> 2, cpg = C / d.groups;
  if (threadIdx.x < d.groups) {
    double s = 0.0, s2 = 0.0;
    for (int k = 0; k < nblk_stats; ++k) {
      const double* p = d.scratch + (((long long)b * nblk_stats + k) * d.groups + threadIdx.x) * 2;
      s += p[0]; s2 += p[1];
    }
    gn_finish(s, s2, (double)d.HW * cpg, gn_pivot(d, b, threadIdx.x, cpg), d.eps, s_mean[threadIdx.x], s_rstd[threadIdx.x]);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int g = c / cpg;
    const float sc = s_rstd[g] * __ldg(d.gamma + c);
    s_scale[c] = sc;
    s_shift[c] = __ldg(d.beta + c) - s_mean[g] * sc;
  }
  __syncthreads();
  const int rows_per = (d.HW + gridDim.x - 1) / gridDim.x;
  const int r0 = blockIdx.x * rows_per;
  const int r1 = min(d.HW, r0 + rows_per);
  const long long total = (long long)max(0, r1 - r0) * Q;
  aldm_plane_t* hi = reinterpret_cast<aldm_plane_t*>(d.out_hi);
  aldm_plane_t* lo = reinterpret_cast<aldm_plane_t*>(d.out_lo);
  const bool act = d.mode == ALDM_PREP_GN_SILU;
  for (long long idx = threadIdx.x; idx < total; idx += blockDim.x) {
    const int pr = (int)(idx / Q), q = (int)(idx % Q);
    const long long row = (long long)b * d.HW + r0 + pr;
    const float4 v = load_cat4(d, row, q * 4);
    float y[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      y[e] = fmaf(y[e], s_scale[q * 4 + e], s_shift[q * 4 + e]);
      if (act) y[e] = silu_f(y[e]);
    }
    store_planes4(hi, lo, row * d.Cp + q * 4, y);
  }
}

// ---------------------------------------------------------------------------------------------
// LayerNorm: one warp per row, C % 4 == 0, C <= 1024
// ---------------------------------------------------------------------------------------------
// NR rows per warp, all their loads issued before the first reduction: with one row per warp the kernel was a chain of
// three dependent latencies (load -> mean -> variance -> store) per warp and 1.7 waves of blocks for 16,384 rows.
template <int NQ, int NR>       // NQ float4 per lane (C <= 128 * NQ)
__global__ void __launch_bounds__(256) ln_kernel(const __grid_constant__ aldm_prep_desc d) {
  const int lane = threadIdx.x & 31;
  const long long row0 = ((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * NR;
  const int C = d.c0, Q = C >> 2;
  pdl_wait();
  if (row0 >= d.rows) return;
  float4 v[NR][NQ];
  float s[NR];
#pragma unroll
  for (int r = 0; r < NR; ++r) {
    s[r] = 0.f;
    const bool rv = row0 + r < d.rows;
#pragma unroll
    for (int i = 0; i < NQ; ++i) {
      const int q = lane + 32 * i;
      v[r][i] = (rv && q < Q) ? *reinterpret_cast<const float4*>(d.src0 + (row0 + r) * C + q * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
#pragma unroll
  for (int r = 0; r < NR; ++r) {
#pragma unroll
    for (int i = 0; i < NQ; ++i) s[r] += (v[r][i].x + v[r][i].y) + (v[r][i].z + v[r][i].w);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int r = 0; r < NR; ++r) s[r] += __shfl_xor_sync(0xffffffffu, s[r], o);
  }
  pdl_launch();      // late trigger: the rows are in registers; see common.cuh on why not at kernel entry
  float mean[NR], s2[NR];
#pragma unroll
  for (int r = 0; r < NR; ++r) {
    mean[r] = s[r] / C;
    s2[r] = 0.f;
#pragma unroll
    for (int i = 0; i < NQ; ++i) {
      if (lane + 32 * i < Q) {
        const float a = v[r][i].x - mean[r], b = v[r][i].y - mean[r], c = v[r][i].z - mean[r], e = v[r][i].w - mean[r];
        s2[r] += (a * a + b * b) + (c * c + e * e);
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int r = 0; r < NR; ++r) s2[r] += __shfl_xor_sync(0xffffffffu, s2[r], o);
  }
  aldm_plane_t* hi = reinterpret_cast<aldm_plane_t*>(d.out_hi);
  aldm_plane_t* lo = reinterpret_cast<aldm_plane_t*>(d.out_lo);
#pragma unroll
  for (int i = 0; i < NQ; ++i) {
    const int q = lane + 32 * i;
    if (q < Q) {
      const float4 g = __ldg(reinterpret_cast<const float4*>(d.gamma + q * 4));
      const float4 be = __ldg(reinterpret_cast<const float4*>(d.beta + q * 4));
#pragma unroll
      for (int r = 0; r < NR; ++r) {
        if (row0 + r < d.rows) {
          const float rstd = rsqrtf(s2[r] / C + d.eps);
          float y[4];
          y[0] = (v[r][i].x - mean[r]) * rstd * g.x + be.x;
          y[1] = (v[r][i].y - mean[r]) * rstd * g.y + be.y;
          y[2] = (v[r][i].z - mean[r]) * rstd * g.z + be.z;
          y[3] = (v[r][i].w - mean[r]) * rstd * g.w + be.w;
          store_planes4(hi, lo, (row0 + r) * d.Cp + q * 4, y);
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// elementwise copy / SiLU / leaky-ReLU -> planes; one thread per (row, 8-channel chunk)
// ---------------------------------------------------------------------------------------------
__global__ void ew_kernel(const __grid_constant__ aldm_prep_desc d) {
  pdl_wait();
  const int C = d.c0 + d.c1;
  const int chunks = d.Cp >> 3;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)d.rows * chunks) return;
  const long long row = idx / chunks;
  const int c = (int)(idx % chunks) * 8;
  float y[8];
  if (d.src_nchw) {
    const long long b = row / d.HW, p = row % d.HW;
#pragma unroll
    for (int e = 0; e < 8; ++e) y[e] = (c + e < C) ? __ldg(d.src0 + (b * C + c + e) * d.HW + p) : 0.f;
  } else if (c + 8 <= C && (d.c0 % 8 == 0) && (d.c1 % 4 == 0)) {
    const float4 a = load_cat4(d, row, c), bb = load_cat4(d, row, c + 4);
    y[0] = a.x; y[1] = a.y; y[2] = a.z; y[3] = a.w; y[4] = bb.x; y[5] = bb.y; y[6] = bb.z; y[7] = bb.w;
  } else {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int cc = c + e;
      y[e] = cc < d.c0 ? d.src0[row * d.c0 + cc] : (cc < C ? d.src1[row * d.c1 + cc - d.c0] : 0.f);
    }
  }
  if (d.mode == ALDM_PREP_SILU) {
#pragma unroll
    for (int e = 0; e < 8; ++e) y[e] = silu_f(y[e]);
  } else if (d.mode == ALDM_PREP_LRELU) {
#pragma unroll
    for (int e = 0; e < 8; ++e) y[e] = y[e] > 0.f ? y[e] : y[e] * d.slope;
  }
  pdl_launch();
  uint4 h, l;
  split8(y, h, l);
  *reinterpret_cast<uint4*>(reinterpret_cast<aldm_plane_t*>(d.out_hi) + row * d.Cp + c) = h;
  if (d.out_lo) *reinterpret_cast<uint4*>(reinterpret_cast<aldm_plane_t*>(d.out_lo) + row * d.Cp + c) = l;
}

// ---------------------------------------------------------------------------------------------
// GroupNorm fast path (channels per group multiple of 4, i.e. C multiple of 128).
//
// Thread layout of both kernels: the block is a (slot, q) grid -- q = 4-channel column (Q = C / 4 of them, QW = min(Q, 256)
// per pass), slot = row phase (RS = 256 / QW of them) -- so a warp reads 512 contiguous bytes of one row, every thread keeps
// its column's group / scale / shift in registers, and the row loop is unrolled four deep (four independent 16-byte loads in
// flight per thread).  The previous version gave a whole column to one thread (32-thread blocks for C = 128): 7 warps per
// SM, one load in flight each -- 1.3 TB/s on an L2-resident tensor.
//
// Statistics are deterministic: per-thread fp32 partials -> fixed-order double sums per block -> scratch; the LAST block of
// a batch row (ticket counter, self-resetting) reduces the per-block partials in fixed order and publishes (mean, rstd), so
// the apply kernel reads 256 bytes per block instead of re-reducing nblk x 32 double pairs (32 KB per block before).
//
// scratch layout (doubles): [B][GN_MAX_BLOCKS][32][2] partials | (float) [B][32][2] mean, rstd | (uint) [B] tickets
// ---------------------------------------------------------------------------------------------
struct GnGeom {
  int Q, QW, RS;
};
__host__ __device__ __forceinline__ GnGeom gn_geom(int C) {
  GnGeom g;
  g.Q = C >> 2;
  g.QW = g.Q < 256 ? g.Q : 256;
  g.RS = 256 / g.QW;
  return g;
}
__device__ __forceinline__ float* gn_stats_ptr(const aldm_prep_desc& d) {
  return reinterpret_cast<float*>(d.scratch + (size_t)d.B * GN_MAX_BLOCKS * 32 * 2);
}
__device__ __forceinline__ unsigned* gn_ticket_ptr(const aldm_prep_desc& d) {
  return reinterpret_cast<unsigned*>(gn_stats_ptr(d) + (size_t)d.B * 32 * 2);
}

__global__ void __launch_bounds__(256) gn_stats_col_kernel(const __grid_constant__ aldm_prep_desc d, int nblk, int finalize) {
  __shared__ float s_a[GN_MAX_C / 4], s_a2[GN_MAX_C / 4];      // [slot][q], RS * Q <= max(256, Q)
  __shared__ double s_red[8][32][2];
  __shared__ int s_last;
  const int b = blockIdx.y, blk = blockIdx.x;
  const int C = d.c0 + d.c1, cpg = C / d.groups;
  const GnGeom gg = gn_geom(C);
  const int slot = threadIdx.x / gg.QW, q0 = threadIdx.x - slot * gg.QW;
  const int rows_per = (d.HW + nblk - 1) / nblk;
  const int r0 = blk * rows_per, r1 = min(d.HW, r0 + rows_per);
  pdl_wait();
  for (int q = q0; q < gg.Q; q += gg.QW) {
    float a = 0.f, a2 = 0.f;
    const float pv = gn_pivot(d, b, (q * 4) / cpg, cpg);      // cpg % 4 == 0 on this path: one group per float4
    int r = r0 + slot;
    const long long rb = (long long)b * d.HW;
    for (; r + 3 * gg.RS < r1; r += 4 * gg.RS) {
      float4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = load_cat4(d, rb + r + u * gg.RS, q * 4);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        v[u].x -= pv; v[u].y -= pv; v[u].z -= pv; v[u].w -= pv;
        a += (v[u].x + v[u].y) + (v[u].z + v[u].w);
        a2 = fmaf(v[u].x, v[u].x, fmaf(v[u].y, v[u].y, fmaf(v[u].z, v[u].z, fmaf(v[u].w, v[u].w, a2))));
      }
    }
    for (; r < r1; r += gg.RS) {
      float4 v = load_cat4(d, rb + r, q * 4);
      v.x -= pv; v.y -= pv; v.z -= pv; v.w -= pv;
      a += (v.x + v.y) + (v.z + v.w);
      a2 = fmaf(v.x, v.x, fmaf(v.y, v.y, fmaf(v.z, v.z, fmaf(v.w, v.w, a2))));
    }
    s_a[slot * gg.Q + q] = a;
    s_a2[slot * gg.Q + q] = a2;
  }
  pdl_launch();
  __syncthreads();
  if (threadIdx.x < d.groups) {
    const int g = threadIdx.x, qpg = cpg >> 2;
    double s = 0.0, s2 = 0.0;
    for (int sl = 0; sl < gg.RS; ++sl)
      for (int k = 0; k < qpg; ++k) {
        s += (double)s_a[sl * gg.Q + g * qpg + k];
        s2 += (double)s_a2[sl * gg.Q + g * qpg + k];
      }
    double* p = d.scratch + (((long long)b * nblk + blk) * d.groups + g) * 2;
    p[0] = s;
    p[1] = s2;
    if (finalize) __threadfence();
  }
  if (!finalize) return;      // few blocks per batch row: the apply kernel reduces the partials itself (no ticket round trip)
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned t = atomicAdd(gn_ticket_ptr(d) + b, 1u);
    s_last = (t == (unsigned)nblk - 1u);
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // last block of this batch row: fixed-order reduction of the nblk partials (8 slices of blocks, then the slices)
  {
    const int g = threadIdx.x & 31, ks = threadIdx.x >> 5, nsl = blockDim.x >> 5;
    double s = 0.0, s2 = 0.0;
    for (int k = ks; k < nblk; k += nsl) {
      const double* p = d.scratch + (((long long)b * nblk + k) * d.groups + g) * 2;
      s += __ldcg(p);
      s2 += __ldcg(p + 1);
    }
    s_red[ks][g][0] = s;
    s_red[ks][g][1] = s2;
    __syncthreads();
    if (threadIdx.x < 32) {
      s = 0.0; s2 = 0.0;
      for (int k = 0; k < nsl; ++k) { s += s_red[k][g][0]; s2 += s_red[k][g][1]; }
      float* st = gn_stats_ptr(d) + ((long long)b * 32 + g) * 2;
      gn_finish(s, s2, (double)d.HW * cpg, gn_pivot(d, b, g, cpg), d.eps, st[0], st[1]);
    }
    if (threadIdx.x == 0) gn_ticket_ptr(d)[b] = 0u;      // self-resetting: the next GroupNorm starts from zero
  }
}

__global__ void __launch_bounds__(256) gn_apply_col_kernel(const __grid_constant__ aldm_prep_desc d, int nblk_partials) {
  __shared__ double s_red[8][32][2];
  __shared__ float s_st[64];
  const int b = blockIdx.y;
  const int C = d.c0 + d.c1, cpg = C / d.groups;
  const GnGeom gg = gn_geom(C);
  const int slot = threadIdx.x / gg.QW, q0 = threadIdx.x - slot * gg.QW;
  const int rows_per = (d.HW + gridDim.x - 1) / gridDim.x;
  const int r0 = blockIdx.x * rows_per, r1 = min(d.HW, r0 + rows_per);
  aldm_plane_t* hi = reinterpret_cast<aldm_plane_t*>(d.out_hi);
  aldm_plane_t* lo = reinterpret_cast<aldm_plane_t*>(d.out_lo);
  const bool act = d.mode == ALDM_PREP_GN_SILU;
  pdl_wait();
  if (nblk_partials > 0) {
    // small tensors: fixed-order reduction of the (<= 8) per-block partials, all threads in parallel
    const int g = threadIdx.x & 31, ks = threadIdx.x >> 5, nsl = blockDim.x >> 5;
    double s = 0.0, s2 = 0.0;
    for (int k = ks; k < nblk_partials; k += nsl) {
      const double* p = d.scratch + (((long long)b * nblk_partials + k) * d.groups + g) * 2;
      s += p[0];
      s2 += p[1];
    }
    s_red[ks][g][0] = s;
    s_red[ks][g][1] = s2;
    __syncthreads();
    if (threadIdx.x < 32) {
      s = 0.0; s2 = 0.0;
      for (int k = 0; k < nsl; ++k) { s += s_red[k][g][0]; s2 += s_red[k][g][1]; }
      gn_finish(s, s2, (double)d.HW * cpg, gn_pivot(d, b, g, cpg), d.eps, s_st[2 * g], s_st[2 * g + 1]);
    }
  } else if (threadIdx.x < 64) {
    s_st[threadIdx.x] = __ldcg(gn_stats_ptr(d) + (long long)b * 64 + threadIdx.x);
  }
  __syncthreads();
  const float* st = s_st;
  const long long rb = (long long)b * d.HW;
  for (int q = q0; q < gg.Q; q += gg.QW) {
    const int g = (q * 4) / cpg;
    const float4 ga = __ldg(reinterpret_cast<const float4*>(d.gamma + q * 4));
    const float4 be = __ldg(reinterpret_cast<const float4*>(d.beta + q * 4));
    const float mu = st[g * 2], rs = st[g * 2 + 1];
    const float sc[4] = {rs * ga.x, rs * ga.y, rs * ga.z, rs * ga.w};
    const float sh[4] = {be.x - mu * sc[0], be.y - mu * sc[1], be.z - mu * sc[2], be.w - mu * sc[3]};
    auto emit = [&](long long row, const float4& v) {
      float y[4] = {fmaf(v.x, sc[0], sh[0]), fmaf(v.y, sc[1], sh[1]), fmaf(v.z, sc[2], sh[2]), fmaf(v.w, sc[3], sh[3])};
      if (act) {
#pragma unroll
        for (int e = 0; e < 4; ++e) y[e] = silu_f(y[e]);
      }
      store_planes4(hi, lo, row * d.Cp + q * 4, y);
    };
    int r = r0 + slot;
    for (; r + 3 * gg.RS < r1; r += 4 * gg.RS) {
      float4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = load_cat4(d, rb + r + u * gg.RS, q * 4);
#pragma unroll
      for (int u = 0; u < 4; ++u) emit(rb + r + u * gg.RS, v[u]);
    }
    for (; r < r1; r += gg.RS) emit(rb + r, load_cat4(d, rb + r, q * 4));
  }
  pdl_launch();
}

// ---------------------------------------------------------------------------------------------
// Single-pass GroupNorm: one CTA owns ALL rows of a batch element for a chunk of G whole groups (G * cpg >= 32 channels, i.e. row
// pieces of >= 128 bytes), parks them in shared memory while it reduces the statistics, then normalises out of shared memory.  The
// tensor is read once instead of twice, one launch instead of two, no scratch, no tickets; deterministic (fixed-order sums).  Used
// whenever HW x G x cpg x 4 bytes fits (every UNet level except the 4096-pixel one, the VAE mid blocks); the two-kernel path above
// takes the rest.
// ---------------------------------------------------------------------------------------------
static constexpr int GN_FUSED_MAX_SMEM = 200 * 1024;

struct GnFusedPlan {
  int G, CW, QW, RS;
  size_t smem;
  bool ok;
};
static GnFusedPlan gn_fused_plan(const aldm_prep_desc& d) {
  GnFusedPlan p{};
  const int C = d.c0 + d.c1;
  if (d.groups != 32 || C % 128 != 0) return p;
  static const bool on = [] { const char* e = getenv("ALDM_GN_FUSED"); return !(e && e[0] == '0'); }();      // A/B switch
  if (!on) return p;
  const int cpg = C / 32;
  int G = 1;
  while (G * cpg < 32) G *= 2;
  p.G = G; p.CW = G * cpg; p.QW = p.CW / 4; p.RS = 256 / p.QW;
  p.smem = (size_t)d.HW * p.CW * 4;
  p.ok = G <= 32 && p.QW <= 256 && p.RS >= 1 && p.smem <= (size_t)GN_FUSED_MAX_SMEM && d.HW >= 1;
  return p;
}

__global__ void __launch_bounds__(256) gn_fused_kernel(const __grid_constant__ aldm_prep_desc d, int G) {
  extern __shared__ float4 gn_sx[];                   // [HW][QW]
  __shared__ float s_a[256], s_a2[256];               // per-thread partials: [slot][q]
  __shared__ float s_mean[32], s_rstd[32];
  const int b = blockIdx.y;
  const int C = d.c0 + d.c1, cpg = C / d.groups;
  const int CW = G * cpg, QW = CW >> 2, RS = 256 / QW;
  const int c_base = blockIdx.x * CW;
  const int slot = threadIdx.x / QW, q = threadIdx.x - slot * QW;
  const bool active = slot < RS;
  const long long rb = (long long)b * d.HW;
  pdl_wait();
  float a = 0.f, a2 = 0.f;
  if (active) {
    const float pv = gn_pivot(d, b, (c_base + q * 4) / cpg, cpg);      // cpg % 4 == 0 here: one group per float4
    int r = slot;
    constexpr int U = 8;        // independent 16-byte loads in flight per thread
    for (; r + (U - 1) * RS < d.HW; r += U * RS) {
      float4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) v[u] = load_cat4(d, rb + r + u * RS, c_base + q * 4);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        gn_sx[(r + u * RS) * QW + q] = v[u];
        const float4 x = make_float4(v[u].x - pv, v[u].y - pv, v[u].z - pv, v[u].w - pv);
        a += (x.x + x.y) + (x.z + x.w);
        a2 = fmaf(x.x, x.x, fmaf(x.y, x.y, fmaf(x.z, x.z, fmaf(x.w, x.w, a2))));
      }
    }
    for (; r < d.HW; r += RS) {
      const float4 v = load_cat4(d, rb + r, c_base + q * 4);
      gn_sx[r * QW + q] = v;
      const float4 x = make_float4(v.x - pv, v.y - pv, v.z - pv, v.w - pv);
      a += (x.x + x.y) + (x.z + x.w);
      a2 = fmaf(x.x, x.x, fmaf(x.y, x.y, fmaf(x.z, x.z, fmaf(x.w, x.w, a2))));
    }
    s_a[slot * QW + q] = a;
    s_a2[slot * QW + q] = a2;
  }
  pdl_launch();
  __syncthreads();
  if (threadIdx.x < G) {
    const int g = threadIdx.x, qpg = cpg >> 2;
    double s = 0.0, s2 = 0.0;
    for (int sl = 0; sl < RS; ++sl)
      for (int k = 0; k < qpg; ++k) {
        s += (double)s_a[sl * QW + g * qpg + k];
        s2 += (double)s_a2[sl * QW + g * qpg + k];
      }
    gn_finish(s, s2, (double)d.HW * cpg, gn_pivot(d, b, blockIdx.x * G + g, cpg), d.eps, s_mean[g], s_rstd[g]);
  }
  __syncthreads();
  if (!active) return;
  aldm_plane_t* hi = reinterpret_cast<aldm_plane_t*>(d.out_hi);
  aldm_plane_t* lo = reinterpret_cast<aldm_plane_t*>(d.out_lo);
  const bool act = d.mode == ALDM_PREP_GN_SILU;
  const int g = (q * 4) / cpg;
  const float4 ga = __ldg(reinterpret_cast<const float4*>(d.gamma + c_base + q * 4));
  const float4 be = __ldg(reinterpret_cast<const float4*>(d.beta + c_base + q * 4));
  const float mu = s_mean[g], rs = s_rstd[g];
  const float sc[4] = {rs * ga.x, rs * ga.y, rs * ga.z, rs * ga.w};
  const float sh[4] = {be.x - mu * sc[0], be.y - mu * sc[1], be.z - mu * sc[2], be.w - mu * sc[3]};
  for (int r = slot; r < d.HW; r += RS) {
    const float4 v = gn_sx[r * QW + q];
    float y[4] = {fmaf(v.x, sc[0], sh[0]), fmaf(v.y, sc[1], sh[1]), fmaf(v.z, sc[2], sh[2]), fmaf(v.w, sc[3], sh[3])};
    if (act) {
#pragma unroll
      for (int e = 0; e < 4; ++e) y[e] = silu_f(y[e]);
    }
    store_planes4(hi, lo, (rb + r) * d.Cp + c_base + q * 4, y);
  }
}

int prep_num_launches(const aldm_prep_desc& d) {
  if (d.mode != ALDM_PREP_GN && d.mode != ALDM_PREP_GN_SILU) return 1;
  return gn_fused_plan(d).ok ? 1 : 2;      // single-pass kernel, or statistics + apply
}

int prep_launch(const aldm_prep_desc& d, cudaStream_t st) {
  ALDM_REQUIRE(d.src0 && d.out_hi, ALDM_E_ARG, "prep: null pointer");        // out_lo == NULL: single-plane output
  ALDM_REQUIRE(d.rows > 0 && d.c0 > 0 && d.c1 >= 0, ALDM_E_SHAPE, "prep: rows=%d c0=%d c1=%d", d.rows, d.c0, d.c1);
  const int C = d.c0 + d.c1;
  ALDM_REQUIRE(d.Cp % 8 == 0 && d.Cp >= C && d.Cp < C + 8, ALDM_E_SHAPE, "prep: Cp=%d for C=%d", d.Cp, C);
  ALDM_REQUIRE(aligned16(d.src0) && aligned16(d.out_hi) && aligned16(d.out_lo), ALDM_E_ALIGN, "prep: alignment");
  if (d.mode == ALDM_PREP_GN || d.mode == ALDM_PREP_GN_SILU) {
    ALDM_REQUIRE(d.gamma && d.beta && d.scratch, ALDM_E_ARG, "prep GN: null gamma/beta/scratch");
    ALDM_REQUIRE(d.groups == 32 && C % d.groups == 0 && C <= GN_MAX_C, ALDM_E_UNSUPPORTED, "prep GN: C=%d groups=%d", C, d.groups);
    ALDM_REQUIRE(C % 4 == 0 && d.c0 % 4 == 0 && d.Cp == C, ALDM_E_SHAPE, "prep GN: channels must be multiples of 4/8");
    ALDM_REQUIRE(d.rows == d.B * d.HW, ALDM_E_SHAPE, "prep GN: rows != B*HW");
    ALDM_REQUIRE(!d.src_nchw, ALDM_E_UNSUPPORTED, "prep GN: NCHW source");
    const int cpg = C / d.groups;
    const GnFusedPlan fp = gn_fused_plan(d);
    if (fp.ok) {
      static bool configured = false;
      if (!configured) {
        ALDM_CHECK_CUDA(cudaFuncSetAttribute(gn_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GN_FUSED_MAX_SMEM));
        configured = true;
      }
      ALDM_CHECK_CUDA(launch_pdl(gn_fused_kernel, dim3(32 / fp.G, d.B), dim3(256), fp.smem, st, d, fp.G));
      ALDM_CHECK_CUDA(cudaGetLastError());
    } else if (cpg % 4 == 0) {
      // (slot, q) kernels: every thread streams ~8-16 float4 rows; ~4 blocks per SM over the whole batch
      const GnGeom gg = gn_geom(C);
      const int thr = gg.QW * gg.RS;                 // multiple of 32 (Q is a multiple of 32 here), <= 256
      const int unit = 4 * gg.RS * cdiv(gg.Q, gg.QW);   // rows that give one thread four loads per column pass
      int nblk = cdiv(4 * num_sms(), d.B);
      if (nblk > cdiv(d.HW, 2 * unit)) nblk = cdiv(d.HW, 2 * unit);
      if (nblk > GN_MAX_BLOCKS) nblk = GN_MAX_BLOCKS;
      if (nblk < 1) nblk = 1;
      const int finalize = nblk > 8 ? 1 : 0;       // last-block finalisation only pays when the apply blocks would re-reduce many partials
      ALDM_CHECK_CUDA(launch_pdl(gn_stats_col_kernel, dim3(nblk, d.B), dim3(thr), 0, st, d, nblk, finalize));
      ALDM_CHECK_CUDA(cudaGetLastError());
      int nap = cdiv(8 * num_sms(), d.B);
      if (nap > cdiv(d.HW, unit)) nap = cdiv(d.HW, unit);
      if (nap < 1) nap = 1;
      ALDM_CHECK_CUDA(launch_pdl(gn_apply_col_kernel, dim3(nap, d.B), dim3(thr), 0, st, d, finalize ? 0 : nblk));
      ALDM_CHECK_CUDA(cudaGetLastError());
    } else {
      int nblk = cdiv(d.HW, 32);
      if (nblk > GN_MAX_BLOCKS) nblk = GN_MAX_BLOCKS;
      ALDM_CHECK_CUDA(launch_pdl(gn_stats_kernel, dim3(nblk, d.B), dim3(256), 0, st, d, nblk));
      ALDM_CHECK_CUDA(cudaGetLastError());
      int nap = cdiv(d.HW, 16);
      if (nap > 128) nap = 128;
      ALDM_CHECK_CUDA(launch_pdl(gn_apply_kernel, dim3(nap, d.B), dim3(256), 0, st, d, nblk));
      ALDM_CHECK_CUDA(cudaGetLastError());
    }
  } else if (d.mode == ALDM_PREP_LN) {
    ALDM_REQUIRE(d.gamma && d.beta, ALDM_E_ARG, "prep LN: null gamma/beta");
    ALDM_REQUIRE(d.c1 == 0 && C % 4 == 0 && C <= 1024 && d.Cp == C, ALDM_E_UNSUPPORTED, "prep LN: C=%d", C);
    // one row per warp; float4 per lane sized to C
    const dim3 grid(cdiv(d.rows, 8));
    ALDM_CHECK_CUDA(C <= 256 ? launch_pdl(ln_kernel<2, 1>, grid, dim3(256), 0, st, d)
                             : (C <= 512 ? launch_pdl(ln_kernel<4, 1>, grid, dim3(256), 0, st, d) : launch_pdl(ln_kernel<8, 1>, grid, dim3(256), 0, st, d)));
    ALDM_CHECK_CUDA(cudaGetLastError());
  } else {
    ALDM_REQUIRE(d.mode == ALDM_PREP_COPY || d.mode == ALDM_PREP_SILU || d.mode == ALDM_PREP_LRELU, ALDM_E_ARG,
                 "prep: mode=%d", d.mode);
    if (d.src_nchw) ALDM_REQUIRE(d.c1 == 0 && d.HW > 0 && d.rows % d.HW == 0, ALDM_E_SHAPE, "prep: NCHW source shape");
    const long long total = (long long)d.rows * (d.Cp >> 3);
    ALDM_CHECK_CUDA(launch_pdl(ew_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, st, d));
    ALDM_CHECK_CUDA(cudaGetLastError());
  }
  return ALDM_OK;
}


// ---------------------------------------------------------------------------------------------
// pack_b: fp32 [N,K] (or its transpose) -> tile images  [n_tile][k_blk][hi|lo][bn rows][128 B swizzled]
//         and (optionally) a plain fp32 [Npad, Kpad] copy for the SIMT checker.
// ---------------------------------------------------------------------------------------------
__global__ void pack_b_kernel(const float* __restrict__ src, int lds, int transpose, int N, int K, int bn,
                              int Kpad, int Npad, uint8_t* __restrict__ dst, float* __restrict__ plain) {
  const int chunks = Kpad >> 3;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)Npad * chunks) return;
  const int n = (int)(idx / chunks);
  const int k0 = (int)(idx % chunks) * 8;
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int k = k0 + e;
    v[e] = (n < N && k < K) ? (transpose ? src[(long long)k * lds + n] : src[(long long)n * lds + k]) : 0.f;
  }
  if (plain) {
#pragma unroll
    for (int e = 0; e < 8; ++e) plain[(long long)n * Kpad + k0 + e] = v[e];
  }
  uint4 h, l;
  split8(v, h, l);
  const int tile = n / bn, r = n % bn, kb = k0 >> 6, j = (k0 & 63) >> 3;
  const long long tile_bytes = (long long)bn * 128;
  uint8_t* base = dst + ((long long)tile * (Kpad >> 6) + kb) * (2 * tile_bytes);
  const int off = r * 128 + ((j ^ (r & 7)) << 4);
  *reinterpret_cast<uint4*>(base + off) = h;
  *reinterpret_cast<uint4*>(base + tile_bytes + off) = l;
}

}  // namespace aldm

extern "C" int aldm_prep(const aldm_prep_desc* d, void* stream) {
  if (!d) { aldm::set_error("aldm_prep: null desc"); return ALDM_E_ARG; }
  return aldm::prep_launch(*d, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int aldm_pack_b(const float* src, int32_t lds, int32_t transpose, int32_t N, int32_t K, int32_t bn,
                           void* dst_packed, float* dst_plain, void* stream) {
  using namespace aldm;
  ALDM_REQUIRE(src && dst_packed, ALDM_E_ARG, "pack_b: null pointer");
  ALDM_REQUIRE(bn == 32 || bn == 64 || bn == 128, ALDM_E_UNSUPPORTED, "pack_b: bn=%d", bn);
  ALDM_REQUIRE(N > 0 && K > 0, ALDM_E_SHAPE, "pack_b: N=%d K=%d", N, K);
  const int Kpad = cdiv(K, 64) * 64, Npad = cdiv(N, bn) * bn;
  const long long total = (long long)Npad * (Kpad >> 3);
  pack_b_kernel<<<(unsigned)((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      src, lds, transpose, N, K, bn, Kpad, Npad, reinterpret_cast<uint8_t*>(dst_packed), dst_plain);
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}
