// Text encoder: the CLAP text branch (CLAP.get_text_embedding, clap/open_clip/model.py:656-663, 730-750) from token ids:
// RoBERTa-base (12 post-LN blocks, width 768, 12 heads of 64, erf-GELU FFN of 3072), the pooler, text_projection and
// F.normalize.  The four projections of every block (fused q | k | v, attention output, intermediate, output) run on the
// tensor-core GEMM (csrc/gemm.cu) with two-plane operands; this file holds what is specific to CLAP:
//   clap_embed_kernel      word[id] + token_type[0] + position[pid], with HF's position ids computed from the ids
//   clap_layernorm_kernel  LayerNorm (two-pass statistics) -> the fp32 residual stream AND operand planes, one pass
//   clap_attention_kernel  bidirectional attention, scale 1/8, masked keys at probability exactly 0, fp32 softmax and P V
//   clap_gelu_kernel       erf-GELU of the intermediate GEMM's fp32 output -> operand planes for the output GEMM
//   clap_head_kernel       tanh pooler on token 0, Linear-ReLU-Linear projection, L2 normalisation, all fp32
// Everything is deterministic: every sum runs in a fixed order, no atomics.
#include "../common.cuh"

namespace aldm {

constexpr int CL_HD = 64;              // head dim
constexpr int CL_LMAX = 512;           // the tokenizer's max_length

__device__ __forceinline__ float cl_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float cl_warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// grid (C / 4 / 128 blocks, B * L rows), one thread per 4 channels.  The position id is HF's
// create_position_ids_from_input_ids: pid = (number of non-pad ids among ids[b, 0..t]) * (id != pad) + pad, counted by every
// warp for itself (at most 512 ids: 16 loads per lane, an exact integer sum).  An id outside [0, vocab) (the host rejects
// those before upload) yields a NaN row rather than an out-of-bounds read.
__global__ void clap_embed_kernel(const __grid_constant__ aldm_clap_embed_desc d) {
  const int r = blockIdx.y;
  const int b = r / d.L, t = r - b * d.L;
  const int lane = threadIdx.x & 31;
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  pdl_wait();
  const int64_t* row = d.ids + (long long)b * d.L;
  int n = 0;
  for (int k = lane; k <= t; k += 32) n += row[k] != d.pad;
  n = __reduce_add_sync(0xffffffffu, n);
  if (c >= d.C) return;
  const int64_t id = row[t];
  const int pid = id != d.pad ? n + d.pad : d.pad;
  float4 v;
  if (id >= 0 && id < d.vocab && pid < d.n_pos) {
    const float4 w = __ldg(reinterpret_cast<const float4*>(d.word + id * d.C + c));
    const float4 y = __ldg(reinterpret_cast<const float4*>(d.type + c));
    const float4 p = __ldg(reinterpret_cast<const float4*>(d.pos + (long long)pid * d.C + c));
    v = make_float4((w.x + y.x) + p.x, (w.y + y.y) + p.y, (w.z + y.z) + p.z, (w.w + y.w) + p.w);
  } else {
    v = make_float4(NAN, NAN, NAN, NAN);
  }
  *reinterpret_cast<float4*>(d.out + (long long)r * d.C + c) = v;
}

// One warp per row, CL_LN_WARPS rows per block.  Lane l holds the float4 chunks l, l + 32, ... of the row.  Two-pass
// statistics: the sum of x, then the sum of (x - mean)^2, each summed per lane in chunk order, then a fixed xor-shuffle
// tree (every lane ends with the same bits).  y = (x - mean) * rstd * gamma + beta goes to out_f32 (the post-LN residual
// stream) and to the operand planes of the next GEMM.
constexpr int CL_LN_WARPS = 4;
constexpr int CL_LN_MAXC = 1024;       // 8 float4 per lane
__global__ void __launch_bounds__(CL_LN_WARPS * 32) clap_layernorm_kernel(const __grid_constant__ aldm_clap_ln_desc d) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * CL_LN_WARPS + (threadIdx.x >> 5);
  pdl_wait();
  if (r >= d.rows) return;
  const float* xr = d.x + (long long)r * d.C;
  const int n4 = d.C / 128;
  float4 v[CL_LN_MAXC / 128];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < CL_LN_MAXC / 128; ++i) {
    if (i < n4) {
      v[i] = *reinterpret_cast<const float4*>(xr + (i * 32 + lane) * 4);
      s += v[i].x; s += v[i].y; s += v[i].z; s += v[i].w;
    }
  }
  const float mean = cl_warp_sum(s) / (float)d.C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < CL_LN_MAXC / 128; ++i) {
    if (i < n4) {
      v[i].x -= mean; v[i].y -= mean; v[i].z -= mean; v[i].w -= mean;
      q = fmaf(v[i].x, v[i].x, q); q = fmaf(v[i].y, v[i].y, q);
      q = fmaf(v[i].z, v[i].z, q); q = fmaf(v[i].w, v[i].w, q);
    }
  }
  const float rs = 1.0f / sqrtf(cl_warp_sum(q) / (float)d.C + d.eps);
#pragma unroll
  for (int i = 0; i < CL_LN_MAXC / 128; ++i) {
    if (i < n4) {
      const int c = (i * 32 + lane) * 4;
      const float4 g = __ldg(reinterpret_cast<const float4*>(d.gamma + c));
      const float4 be = __ldg(reinterpret_cast<const float4*>(d.beta + c));
      const float y0 = fmaf(v[i].x * rs, g.x, be.x), y1 = fmaf(v[i].y * rs, g.y, be.y);
      const float y2 = fmaf(v[i].z * rs, g.z, be.z), y3 = fmaf(v[i].w * rs, g.w, be.w);
      *reinterpret_cast<float4*>(d.out_f32 + (long long)r * d.C + c) = make_float4(y0, y1, y2, y3);
      uint2 hi, lo;
      split2(y0, y1, hi.x, lo.x);
      split2(y2, y3, hi.y, lo.y);
      *reinterpret_cast<uint2*>(reinterpret_cast<aldm_plane_t*>(d.out_hi) + (long long)r * d.ldo + c) = hi;
      if (d.out_lo) *reinterpret_cast<uint2*>(reinterpret_cast<aldm_plane_t*>(d.out_lo) + (long long)r * d.ldo + c) = lo;
    }
  }
}

// Block = (chunk of CL_ATT_Q queries, head, batch row), CL_ATT_WARPS warps; warp w owns the chunk's queries
// 4w .. 4w + 3.  The scores of the block's queries against all L keys stay in shared memory ([32][L] fp32, 64 KB at
// L = 512); K and then V pass through a staging tile of CL_ATT_KC keys (rows padded to 65 floats: lane j reads key j's
// row without bank conflicts).
//   scores: lane owns keys lane and lane + 32 of a tile and sums q[d] k[d] over d = 0..63 in order with fmaf, times 1/8
//           (exact); a key with mask != 1 gets -inf, i.e. probability exactly 0 (the reference's finfo.min fill, as long
//           as one key is valid, which the host checks);
//   softmax: warp max and sum of exp(s - max) over the lane's keys in order, then a fixed xor tree;
//   P V:    lane owns dimensions lane and lane + 32 and sums over the keys in order; the result is divided by the sum
//           and split into two fp16 planes.
constexpr int CL_ATT_WARPS = 8;
constexpr int CL_ATT_QW = 4;
constexpr int CL_ATT_Q = CL_ATT_WARPS * CL_ATT_QW;
constexpr int CL_ATT_KC = 64;
constexpr int CL_ATT_KLD = CL_HD + 1;
__host__ __device__ constexpr size_t clap_att_smem(int L) {
  return (size_t)(CL_ATT_Q * L + CL_ATT_KC * CL_ATT_KLD + CL_ATT_Q * CL_HD) * 4;
}
__global__ void __launch_bounds__(CL_ATT_WARPS * 32) clap_attention_kernel(const __grid_constant__ aldm_clap_attn_desc d) {
  extern __shared__ float smem[];
  const int L = d.L, C = d.heads * CL_HD;
  float* s_s = smem;                                  // [32][L]
  float* kv_s = s_s + CL_ATT_Q * L;                   // [64][65]
  float* q_s = kv_s + CL_ATT_KC * CL_ATT_KLD;         // [32][64]
  const int h = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int q0 = blockIdx.x * CL_ATT_Q;
  const float* base = d.qkv + (long long)b * L * d.ld_qkv + h * CL_HD;
  const float* mrow = d.mask + (long long)b * L;
  pdl_wait();
  for (int e = tid; e < CL_ATT_Q * CL_HD; e += CL_ATT_WARPS * 32) {
    const int i = e >> 6, c = e & 63;
    q_s[e] = q0 + i < L ? base[(long long)(q0 + i) * d.ld_qkv + c] : 0.f;
  }
  const float* qw = q_s + warp * CL_ATT_QW * CL_HD;
  float* sw = s_s + warp * CL_ATT_QW * L;
  // scores
  for (int j0 = 0; j0 < L; j0 += CL_ATT_KC) {
    const int kc = min(CL_ATT_KC, L - j0);
    __syncthreads();                                  // the previous tile is consumed (and q_s is written)
    for (int e = tid; e < kc * CL_HD; e += CL_ATT_WARPS * 32) {
      const int j = e >> 6, c = e & 63;
      kv_s[j * CL_ATT_KLD + c] = base[(long long)(j0 + j) * d.ld_qkv + C + c];
    }
    __syncthreads();
    float acc[CL_ATT_QW][2];
#pragma unroll
    for (int qi = 0; qi < CL_ATT_QW; ++qi) acc[qi][0] = acc[qi][1] = 0.f;
    const float* k0 = kv_s + lane * CL_ATT_KLD;
    const float* k1 = kv_s + (lane + 32) * CL_ATT_KLD;
#pragma unroll 8
    for (int c = 0; c < CL_HD; ++c) {
      const float a0 = k0[c], a1 = k1[c];       // rows >= kc hold stale values: their scores are never stored
#pragma unroll
      for (int qi = 0; qi < CL_ATT_QW; ++qi) {
        const float qv = qw[qi * CL_HD + c];
        acc[qi][0] = fmaf(qv, a0, acc[qi][0]);
        acc[qi][1] = fmaf(qv, a1, acc[qi][1]);
      }
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int j = lane + 32 * u;
      if (j < kc) {
        const bool keep = mrow[j0 + j] == 1.0f;
#pragma unroll
        for (int qi = 0; qi < CL_ATT_QW; ++qi) sw[qi * L + j0 + j] = keep ? acc[qi][u] * 0.125f : -INFINITY;
      }
    }
  }
  // softmax numerators (each warp its own rows of s_s)
  __syncwarp();
  float sum[CL_ATT_QW];
#pragma unroll
  for (int qi = 0; qi < CL_ATT_QW; ++qi) {
    float* sr = sw + qi * L;
    float mx = -INFINITY;
    for (int j = lane; j < L; j += 32) mx = fmaxf(mx, sr[j]);
    mx = cl_warp_max(mx);
    float sm = 0.f;
    for (int j = lane; j < L; j += 32) {
      const float e = expf(sr[j] - mx);
      sr[j] = e;
      sm += e;
    }
    sum[qi] = cl_warp_sum(sm);
  }
  // P V
  float o[CL_ATT_QW][2];
#pragma unroll
  for (int qi = 0; qi < CL_ATT_QW; ++qi) o[qi][0] = o[qi][1] = 0.f;
  for (int j0 = 0; j0 < L; j0 += CL_ATT_KC) {
    const int kc = min(CL_ATT_KC, L - j0);
    __syncthreads();
    for (int e = tid; e < kc * CL_HD; e += CL_ATT_WARPS * 32) {
      const int j = e >> 6, c = e & 63;
      kv_s[j * CL_ATT_KLD + c] = base[(long long)(j0 + j) * d.ld_qkv + 2 * C + c];
    }
    __syncthreads();
    for (int j = 0; j < kc; ++j) {
      const float v0 = kv_s[j * CL_ATT_KLD + lane], v1 = kv_s[j * CL_ATT_KLD + lane + 32];
#pragma unroll
      for (int qi = 0; qi < CL_ATT_QW; ++qi) {
        const float p = sw[qi * L + j0 + j];
        o[qi][0] = fmaf(p, v0, o[qi][0]);
        o[qi][1] = fmaf(p, v1, o[qi][1]);
      }
    }
  }
#pragma unroll
  for (int qi = 0; qi < CL_ATT_QW; ++qi) {
    const int i = q0 + warp * CL_ATT_QW + qi;
    if (i < L) {
      const long long orow = ((long long)b * L + i) * d.ldo + h * CL_HD;
      aldm_plane_t* hp = reinterpret_cast<aldm_plane_t*>(d.out_hi) + orow;
      aldm_plane_t* lp = d.out_lo ? reinterpret_cast<aldm_plane_t*>(d.out_lo) + orow : nullptr;
      store_split1(hp, lp, lane, o[qi][0] / sum[qi]);
      store_split1(hp, lp, lane + 32, o[qi][1] / sum[qi]);
    }
  }
}

// One thread per 4 outputs: gelu(x) = 0.5 x (1 + erf(x / sqrt(2))) with the accurate erff (transformers GELUActivation,
// hidden_act = "gelu"), split into operand planes.
__global__ void clap_gelu_kernel(const __grid_constant__ aldm_clap_gelu_desc d) {
  const int r = blockIdx.y;
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  pdl_wait();
  if (c >= d.F) return;
  const float4 a = *reinterpret_cast<const float4*>(d.x + (long long)r * d.ld_x + c);
  float y[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
  for (int k = 0; k < 4; ++k) y[k] = 0.5f * y[k] * (1.0f + erff(y[k] * 0.70710678118654752440f));
  uint2 hi, lo;
  split2(y[0], y[1], hi.x, lo.x);
  split2(y[2], y[3], hi.y, lo.y);
  *reinterpret_cast<uint2*>(reinterpret_cast<aldm_plane_t*>(d.out_hi) + (long long)r * d.ldo + c) = hi;
  if (d.out_lo) *reinterpret_cast<uint2*>(reinterpret_cast<aldm_plane_t*>(d.out_lo) + (long long)r * d.ldo + c) = lo;
}

// One block per batch row, fp32 throughout.  Thread n computes outputs n, n + CL_HEAD_T, ... of each layer as a dot
// product over the inputs in order (the weights are stored transposed, [in, out], so a warp's loads are coalesced), then
// adds the bias.  The squared norm is summed per thread in output order, then a fixed warp tree, then warp 0 sums the
// warps' partials in order.
constexpr int CL_HEAD_T = 512;
constexpr int CL_HEAD_MAXC = 1024;
constexpr int CL_HEAD_MAXP = 1024;
__global__ void __launch_bounds__(CL_HEAD_T) clap_head_kernel(const __grid_constant__ aldm_clap_head_desc d) {
  __shared__ float h_s[CL_HEAD_MAXC], p_s[CL_HEAD_MAXC], t_s[CL_HEAD_MAXP], y_s[CL_HEAD_MAXP];
  __shared__ float red[CL_HEAD_T / 32];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int C = d.C, P = d.P;
  pdl_wait();
  const float* x0 = d.x + (long long)b * d.L * C;     // token 0 of row b
  for (int c = tid; c < C; c += CL_HEAD_T) h_s[c] = x0[c];
  __syncthreads();
  for (int n = tid; n < C; n += CL_HEAD_T) {          // pooler: tanh(Wp h + bp)
    float a = 0.f;
    for (int k = 0; k < C; ++k) a = fmaf(h_s[k], __ldg(d.wp_t + (long long)k * C + n), a);
    p_s[n] = tanhf(a + __ldg(d.bp + n));
  }
  __syncthreads();
  for (int n = tid; n < P; n += CL_HEAD_T) {          // text_projection[0], ReLU
    float a = 0.f;
    for (int k = 0; k < C; ++k) a = fmaf(p_s[k], __ldg(d.w1_t + (long long)k * P + n), a);
    t_s[n] = fmaxf(a + __ldg(d.b1 + n), 0.f);
  }
  __syncthreads();
  float ss = 0.f;
  for (int n = tid; n < P; n += CL_HEAD_T) {          // text_projection[2]
    float a = 0.f;
    for (int k = 0; k < P; ++k) a = fmaf(t_s[k], __ldg(d.w2_t + (long long)k * P + n), a);
    a += __ldg(d.b2 + n);
    y_s[n] = a;
    ss = fmaf(a, a, ss);
  }
  ss = cl_warp_sum(ss);
  if ((tid & 31) == 0) red[tid >> 5] = ss;
  __syncthreads();
  if (tid == 0) {
    float t = 0.f;
    for (int w = 0; w < CL_HEAD_T / 32; ++w) t += red[w];
    red[0] = t;
  }
  __syncthreads();
  const float den = fmaxf(sqrtf(red[0]), 1e-12f);     // F.normalize: x / max(||x||_2, eps)
  for (int n = tid; n < P; n += CL_HEAD_T) d.out[(long long)b * P + n] = y_s[n] / den;
}

int clap_embed_launch(const aldm_clap_embed_desc& d, cudaStream_t st) {
  ALDM_REQUIRE(d.ids && d.word && d.pos && d.type && d.out, ALDM_E_ARG, "clap_embed: null pointer");
  ALDM_REQUIRE(d.B > 0 && d.L > 0 && d.L <= CL_LMAX && (long long)d.B * d.L <= 65535 && d.vocab > 0 && d.n_pos > 0 &&
                   d.C > 0 && d.C % 4 == 0,
               ALDM_E_SHAPE, "clap_embed: B=%d L=%d vocab=%d n_pos=%d C=%d (L <= %d)", d.B, d.L, d.vocab, d.n_pos, d.C, CL_LMAX);
  ALDM_REQUIRE(aligned16(d.word) && aligned16(d.pos) && aligned16(d.type) && aligned16(d.out), ALDM_E_ALIGN,
               "clap_embed: alignment");
  ALDM_CHECK_CUDA(launch_pdl(clap_embed_kernel, dim3(cdiv(d.C / 4, 128), d.B * d.L), dim3(128), 0, st, d));
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}

int clap_layernorm_launch(const aldm_clap_ln_desc& d, cudaStream_t st) {
  ALDM_REQUIRE(d.x && d.gamma && d.beta && d.out_f32 && d.out_hi, ALDM_E_ARG, "clap_layernorm: null pointer");
  ALDM_REQUIRE(d.rows > 0 && d.C > 0 && d.C % 128 == 0 && d.C <= CL_LN_MAXC && d.ldo >= d.C && d.ldo % 4 == 0, ALDM_E_SHAPE,
               "clap_layernorm: rows=%d C=%d ldo=%d (C a multiple of 128, <= %d)", d.rows, d.C, d.ldo, CL_LN_MAXC);
  ALDM_REQUIRE(aligned16(d.x) && aligned16(d.gamma) && aligned16(d.beta) && aligned16(d.out_f32), ALDM_E_ALIGN,
               "clap_layernorm: alignment");
  ALDM_CHECK_CUDA(launch_pdl(clap_layernorm_kernel, dim3(cdiv(d.rows, CL_LN_WARPS)), dim3(CL_LN_WARPS * 32), 0, st, d));
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}

int clap_attention_launch(const aldm_clap_attn_desc& d, cudaStream_t st) {
  ALDM_REQUIRE(d.qkv && d.mask && d.out_hi, ALDM_E_ARG, "clap_attention: null pointer");
  ALDM_REQUIRE(d.B > 0 && d.B <= 65535 && d.heads > 0 && d.heads <= 65535 && d.heads * CL_HD == d.C, ALDM_E_SHAPE,
               "clap_attention: B=%d heads=%d C=%d (heads x %d must equal C)", d.B, d.heads, d.C, CL_HD);
  ALDM_REQUIRE(d.L > 0 && d.L <= CL_LMAX, ALDM_E_SHAPE, "clap_attention: L=%d (1..%d)", d.L, CL_LMAX);
  ALDM_REQUIRE(d.ld_qkv >= 3 * d.C && d.ldo >= d.C, ALDM_E_SHAPE, "clap_attention: ld_qkv=%d ldo=%d", d.ld_qkv, d.ldo);
  static bool attr = false;
  if (!attr) {
    ALDM_CHECK_CUDA(cudaFuncSetAttribute(clap_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)clap_att_smem(CL_LMAX)));
    attr = true;
  }
  ALDM_CHECK_CUDA(launch_pdl(clap_attention_kernel, dim3(cdiv(d.L, CL_ATT_Q), d.heads, d.B), dim3(CL_ATT_WARPS * 32),
                             clap_att_smem(d.L), st, d));
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}

int clap_gelu_launch(const aldm_clap_gelu_desc& d, cudaStream_t st) {
  ALDM_REQUIRE(d.x && d.out_hi, ALDM_E_ARG, "clap_gelu: null pointer");
  ALDM_REQUIRE(d.rows > 0 && d.rows <= 65535 && d.F > 0 && d.F % 4 == 0 && d.ld_x >= d.F && d.ld_x % 4 == 0 &&
                   d.ldo >= d.F && d.ldo % 4 == 0,
               ALDM_E_SHAPE, "clap_gelu: rows=%d F=%d ld_x=%d ldo=%d", d.rows, d.F, d.ld_x, d.ldo);
  ALDM_REQUIRE(aligned16(d.x), ALDM_E_ALIGN, "clap_gelu: alignment");
  ALDM_CHECK_CUDA(launch_pdl(clap_gelu_kernel, dim3(cdiv(d.F / 4, 128), d.rows), dim3(128), 0, st, d));
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}

int clap_head_launch(const aldm_clap_head_desc& d, cudaStream_t st) {
  ALDM_REQUIRE(d.x && d.wp_t && d.bp && d.w1_t && d.b1 && d.w2_t && d.b2 && d.out, ALDM_E_ARG, "clap_head: null pointer");
  ALDM_REQUIRE(d.B > 0 && d.B <= 65535 && d.L > 0 && d.C > 0 && d.C <= CL_HEAD_MAXC && d.P > 0 && d.P <= CL_HEAD_MAXP,
               ALDM_E_SHAPE, "clap_head: B=%d L=%d C=%d P=%d (C, P <= %d)", d.B, d.L, d.C, d.P, CL_HEAD_MAXC);
  ALDM_CHECK_CUDA(launch_pdl(clap_head_kernel, dim3(d.B), dim3(CL_HEAD_T), 0, st, d));
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}

}  // namespace aldm

extern "C" int aldm_clap_embed(const aldm_clap_embed_desc* d, void* stream) {
  if (!d) { aldm::set_error("aldm_clap_embed: null desc"); return ALDM_E_ARG; }
  return aldm::clap_embed_launch(*d, reinterpret_cast<cudaStream_t>(stream));
}
extern "C" int aldm_clap_layernorm(const aldm_clap_ln_desc* d, void* stream) {
  if (!d) { aldm::set_error("aldm_clap_layernorm: null desc"); return ALDM_E_ARG; }
  return aldm::clap_layernorm_launch(*d, reinterpret_cast<cudaStream_t>(stream));
}
extern "C" int aldm_clap_attention(const aldm_clap_attn_desc* d, void* stream) {
  if (!d) { aldm::set_error("aldm_clap_attention: null desc"); return ALDM_E_ARG; }
  return aldm::clap_attention_launch(*d, reinterpret_cast<cudaStream_t>(stream));
}
extern "C" int aldm_clap_gelu(const aldm_clap_gelu_desc* d, void* stream) {
  if (!d) { aldm::set_error("aldm_clap_gelu: null desc"); return ALDM_E_ARG; }
  return aldm::clap_gelu_launch(*d, reinterpret_cast<cudaStream_t>(stream));
}
extern "C" int aldm_clap_head(const aldm_clap_head_desc* d, void* stream) {
  if (!d) { aldm::set_error("aldm_clap_head: null desc"); return ALDM_E_ARG; }
  return aldm::clap_head_launch(*d, reinterpret_cast<cudaStream_t>(stream));
}
