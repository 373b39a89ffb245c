// Text encoder: Flan-T5-large's encoder stack (T5EncoderModel, encoders/modules.py:113-198) from token ids.  The four
// projections of every block (fused q | k | v, o, fused wi_0 | wi_1, wo) run on the tensor-core GEMM (csrc/gemm.cu) with
// two-plane operands; this file holds what is specific to T5:
//   t5_embed_kernel      token ids -> fp32 residual rows gathered from shared.weight (the embedding is not scaled)
//   t5_rmsnorm_kernel    T5LayerNorm: x * rsqrt(mean(x^2) + eps) * w, no mean, no bias -> operand planes, or fp32 for
//                        final_layer_norm
//   t5_attention_kernel  unscaled q.k^T + the relative-position bias of layer 0 + the key mask, fp32 softmax and P V
//   t5_gate_kernel       gelu_new(wi_0 x) * wi_1 x -> operand planes for wo, counting values beyond the fp16 range
// Everything is deterministic: every sum runs in a fixed order.
#include "../common.cuh"

namespace aldm {

constexpr int T5_HD = 64;              // d_kv
constexpr int T5_LMAX = 128;           // the tokenizer's max_length: every key of a (row, head) fits in shared memory
constexpr int T5_NOFF = 2 * T5_LMAX - 1;   // bias table columns: offsets j - i in [-127, 127]

__device__ __forceinline__ float t5_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float t5_warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// One thread per 4 channels of one row.  An id outside [0, vocab) (the host rejects those before upload) yields a NaN row
// rather than an out-of-bounds read.
__global__ void t5_embed_kernel(const __grid_constant__ aldm_t5_embed_desc d) {
  const int r = blockIdx.y;
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  pdl_wait();
  if (c >= d.C) return;
  const long long id = d.ids[r];
  float4 v;
  if (id >= 0 && id < d.vocab) v = __ldg(reinterpret_cast<const float4*>(d.table + id * d.C + c));
  else v = make_float4(NAN, NAN, NAN, NAN);
  *reinterpret_cast<float4*>(d.out + (long long)r * d.C + c) = v;
}

// One warp per row, T5_RMS_WARPS rows per block.  Lane l holds the float4 chunks l, l + 32, ... of the row; its squares
// are summed in that order, then a fixed xor-shuffle tree (every lane ends with the same bits).
constexpr int T5_RMS_WARPS = 4;
constexpr int T5_RMS_MAXC = 2048;      // 16 float4 per lane
__global__ void __launch_bounds__(T5_RMS_WARPS * 32) t5_rmsnorm_kernel(const __grid_constant__ aldm_t5_rmsnorm_desc d) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * T5_RMS_WARPS + (threadIdx.x >> 5);
  pdl_wait();
  if (r >= d.rows) return;
  const float* xr = d.x + (long long)r * d.C;
  const int n4 = d.C / 128;            // float4 chunks per lane
  float4 v[T5_RMS_MAXC / 128];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < T5_RMS_MAXC / 128; ++i) {
    if (i < n4) {
      v[i] = *reinterpret_cast<const float4*>(xr + (i * 32 + lane) * 4);
      s = fmaf(v[i].x, v[i].x, s);
      s = fmaf(v[i].y, v[i].y, s);
      s = fmaf(v[i].z, v[i].z, s);
      s = fmaf(v[i].w, v[i].w, s);
    }
  }
  s = t5_warp_sum(s);
  const float rs = 1.0f / sqrtf(s / (float)d.C + d.eps);
#pragma unroll
  for (int i = 0; i < T5_RMS_MAXC / 128; ++i) {
    if (i < n4) {
      const int c = (i * 32 + lane) * 4;
      const float4 g = __ldg(reinterpret_cast<const float4*>(d.gamma + c));
      const float y0 = g.x * (v[i].x * rs), y1 = g.y * (v[i].y * rs), y2 = g.z * (v[i].z * rs), y3 = g.w * (v[i].w * rs);
      if (d.out_f32) {
        *reinterpret_cast<float4*>(d.out_f32 + (long long)r * d.ldo + c) = make_float4(y0, y1, y2, y3);
      } else {
        uint2 hi, lo;
        split2(y0, y1, hi.x, lo.x);
        split2(y2, y3, hi.y, lo.y);
        *reinterpret_cast<uint2*>(reinterpret_cast<aldm_plane_t*>(d.out_hi) + (long long)r * d.ldo + c) = hi;
        if (d.out_lo) *reinterpret_cast<uint2*>(reinterpret_cast<aldm_plane_t*>(d.out_lo) + (long long)r * d.ldo + c) = lo;
      }
    }
  }
}

// Block = (chunk of T5_ATT_Q queries, head, batch row), T5_ATT_WARPS warps; warp w takes the chunk's queries w, w + 8, ....
// K (rows padded to 65 floats: lane j reads key j's row without bank conflicts) and V of the (row, head) are staged in
// shared memory once per block.  Scores: lane j owns keys j, j + 32, ... and sums q[d] k[d] over d = 0..63 in order with
// fmaf; + bias[h, j - i + 127]; a key with mask != 1 gets probability exactly 0 (the reference's finfo.min fill, as long
// as one key is valid, which the host checks).  P V: lane owns dimensions lane and lane + 32 and sums over the keys in
// order; the output is divided by the fixed-order warp sum of the probabilities and split into two fp16 planes.
constexpr int T5_ATT_WARPS = 8;
constexpr int T5_ATT_Q = 32;
constexpr int T5_ATT_KLD = T5_HD + 1;
constexpr size_t T5_ATT_SMEM = (size_t)(T5_LMAX * T5_ATT_KLD + T5_LMAX * T5_HD + T5_ATT_WARPS * (T5_HD + T5_LMAX)) * 4;
__global__ void __launch_bounds__(T5_ATT_WARPS * 32) t5_attention_kernel(const __grid_constant__ aldm_t5_attn_desc d) {
  extern __shared__ float smem[];
  float* k_s = smem;                                  // [L][65]
  float* v_s = k_s + T5_LMAX * T5_ATT_KLD;            // [L][64]
  float* q_s = v_s + T5_LMAX * T5_HD;                 // [warp][64]
  float* p_s = q_s + T5_ATT_WARPS * T5_HD;            // [warp][128]
  const int h = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int L = d.L, C = d.heads * T5_HD;
  const float* base = d.qkv + (long long)b * L * d.ld_qkv;
  pdl_wait();
  for (int e = tid; e < L * T5_HD; e += T5_ATT_WARPS * 32) {
    const int j = e >> 6, c = e & 63;
    const float* row = base + (long long)j * d.ld_qkv + h * T5_HD + c;
    k_s[j * T5_ATT_KLD + c] = row[C];
    v_s[j * T5_HD + c] = row[2 * C];
  }
  __syncthreads();
  const float* mrow = d.mask + (long long)b * L;
  const float* brow = d.bias + (long long)h * T5_NOFF + (T5_LMAX - 1);
  float* qw = q_s + warp * T5_HD;
  float* pw = p_s + warp * T5_LMAX;
  const int i_end = min(L, (int)(blockIdx.x + 1) * T5_ATT_Q);
  for (int i = blockIdx.x * T5_ATT_Q + warp; i < i_end; i += T5_ATT_WARPS) {
    const float* qr = base + (long long)i * d.ld_qkv + h * T5_HD;
    qw[lane] = qr[lane];
    qw[lane + 32] = qr[lane + 32];
    __syncwarp();
    float mx = -INFINITY;
    for (int j = lane; j < L; j += 32) {
      const float* kr = k_s + j * T5_ATT_KLD;
      float s = 0.f;
#pragma unroll 16
      for (int c = 0; c < T5_HD; ++c) s = fmaf(qw[c], kr[c], s);
      s += __ldg(brow + (j - i));
      s = mrow[j] == 1.0f ? s : -INFINITY;
      pw[j] = s;
      mx = fmaxf(mx, s);
    }
    mx = t5_warp_max(mx);
    float sum = 0.f;
    for (int j = lane; j < L; j += 32) {
      const float e = expf(pw[j] - mx);
      pw[j] = e;
      sum += e;
    }
    sum = t5_warp_sum(sum);
    __syncwarp();
    float a0 = 0.f, a1 = 0.f;
    for (int j = 0; j < L; ++j) {
      const float p = pw[j];
      a0 = fmaf(p, v_s[j * T5_HD + lane], a0);
      a1 = fmaf(p, v_s[j * T5_HD + lane + 32], a1);
    }
    const long long orow = ((long long)b * L + i) * d.ldo + h * T5_HD;
    aldm_plane_t* hp = reinterpret_cast<aldm_plane_t*>(d.out_hi) + orow;
    aldm_plane_t* lp = d.out_lo ? reinterpret_cast<aldm_plane_t*>(d.out_lo) + orow : nullptr;
    store_split1(hp, lp, lane, a0 / sum);
    store_split1(hp, lp, lane + 32, a1 / sum);
    __syncwarp();                       // q / p of this warp are rewritten by its next query
  }
}

// One thread per 4 outputs.  |y| > 65504 (or a non-finite y) would be clamped by the operand split: such elements are
// counted (warp-aggregated atomics) into *sat, which the host reads after the run.
__global__ void t5_gate_kernel(const __grid_constant__ aldm_t5_gate_desc d) {
  const int r = blockIdx.y;
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  pdl_wait();
  unsigned n_sat = 0;
  if (c < d.F) {
    const float* xr = d.x + (long long)r * d.ld_x;
    const float4 a = *reinterpret_cast<const float4*>(xr + c);
    const float4 g = *reinterpret_cast<const float4*>(xr + d.F + c);
    float y[4] = {gelu_tanh_f(a.x) * g.x, gelu_tanh_f(a.y) * g.y, gelu_tanh_f(a.z) * g.z, gelu_tanh_f(a.w) * g.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) n_sat += !(fabsf(y[k]) <= 65504.0f);
    uint2 hi, lo;
    split2(y[0], y[1], hi.x, lo.x);
    split2(y[2], y[3], hi.y, lo.y);
    *reinterpret_cast<uint2*>(reinterpret_cast<aldm_plane_t*>(d.out_hi) + (long long)r * d.ldo + c) = hi;
    if (d.out_lo) *reinterpret_cast<uint2*>(reinterpret_cast<aldm_plane_t*>(d.out_lo) + (long long)r * d.ldo + c) = lo;
  }
  n_sat = __reduce_add_sync(0xffffffffu, n_sat);
  if (n_sat && (threadIdx.x & 31) == 0) atomicAdd(d.sat, n_sat);
}

int t5_embed_launch(const aldm_t5_embed_desc& d, cudaStream_t st) {
  ALDM_REQUIRE(d.ids && d.table && d.out, ALDM_E_ARG, "t5_embed: null pointer");
  ALDM_REQUIRE(d.rows > 0 && d.rows <= 65535 && d.vocab > 0 && d.C > 0 && d.C % 4 == 0, ALDM_E_SHAPE,
               "t5_embed: rows=%d vocab=%d C=%d", d.rows, d.vocab, d.C);
  ALDM_REQUIRE(aligned16(d.table) && aligned16(d.out), ALDM_E_ALIGN, "t5_embed: alignment");
  ALDM_CHECK_CUDA(launch_pdl(t5_embed_kernel, dim3(cdiv(d.C / 4, 128), d.rows), dim3(128), 0, st, d));
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}

int t5_rmsnorm_launch(const aldm_t5_rmsnorm_desc& d, cudaStream_t st) {
  ALDM_REQUIRE(d.x && d.gamma && (d.out_f32 || d.out_hi), ALDM_E_ARG, "t5_rmsnorm: null pointer");
  ALDM_REQUIRE(d.rows > 0 && d.C > 0 && d.C % 128 == 0 && d.C <= T5_RMS_MAXC && d.ldo >= d.C && d.ldo % 4 == 0, ALDM_E_SHAPE,
               "t5_rmsnorm: rows=%d C=%d ldo=%d (C a multiple of 128, <= %d)", d.rows, d.C, d.ldo, T5_RMS_MAXC);
  ALDM_REQUIRE(aligned16(d.x) && aligned16(d.gamma) && (!d.out_f32 || aligned16(d.out_f32)), ALDM_E_ALIGN,
               "t5_rmsnorm: alignment");
  ALDM_CHECK_CUDA(launch_pdl(t5_rmsnorm_kernel, dim3(cdiv(d.rows, T5_RMS_WARPS)), dim3(T5_RMS_WARPS * 32), 0, st, d));
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}

int t5_attention_launch(const aldm_t5_attn_desc& d, cudaStream_t st) {
  ALDM_REQUIRE(d.qkv && d.bias && d.mask && d.out_hi, ALDM_E_ARG, "t5_attention: null pointer");
  ALDM_REQUIRE(d.d_kv == T5_HD, ALDM_E_UNSUPPORTED, "t5_attention: d_kv=%d (only %d)", d.d_kv, T5_HD);
  ALDM_REQUIRE(d.B > 0 && d.B <= 65535 && d.heads > 0 && d.heads <= 65535 && d.heads * T5_HD == d.C, ALDM_E_SHAPE,
               "t5_attention: B=%d heads=%d C=%d (heads x %d must equal C)", d.B, d.heads, d.C, T5_HD);
  ALDM_REQUIRE(d.L > 0 && d.L <= T5_LMAX, ALDM_E_SHAPE, "t5_attention: L=%d (1..%d)", d.L, T5_LMAX);
  ALDM_REQUIRE(d.ld_qkv >= 3 * d.C && d.ldo >= d.C, ALDM_E_SHAPE, "t5_attention: ld_qkv=%d ldo=%d", d.ld_qkv, d.ldo);
  static bool attr = false;
  if (!attr) {
    ALDM_CHECK_CUDA(cudaFuncSetAttribute(t5_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)T5_ATT_SMEM));
    attr = true;
  }
  ALDM_CHECK_CUDA(launch_pdl(t5_attention_kernel, dim3(cdiv(d.L, T5_ATT_Q), d.heads, d.B), dim3(T5_ATT_WARPS * 32),
                             T5_ATT_SMEM, st, d));
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}

int t5_gate_launch(const aldm_t5_gate_desc& d, cudaStream_t st) {
  ALDM_REQUIRE(d.x && d.out_hi && d.sat, ALDM_E_ARG, "t5_gate: null pointer");
  ALDM_REQUIRE(d.rows > 0 && d.rows <= 65535 && d.F > 0 && d.F % 4 == 0 && d.ld_x >= 2 * d.F && d.ld_x % 4 == 0 &&
                   d.ldo >= d.F && d.ldo % 4 == 0,
               ALDM_E_SHAPE, "t5_gate: rows=%d F=%d ld_x=%d ldo=%d", d.rows, d.F, d.ld_x, d.ldo);
  ALDM_REQUIRE(aligned16(d.x), ALDM_E_ALIGN, "t5_gate: alignment");
  ALDM_CHECK_CUDA(launch_pdl(t5_gate_kernel, dim3(cdiv(d.F / 4, 128), d.rows), dim3(128), 0, st, d));
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}

}  // namespace aldm

extern "C" int aldm_t5_embed(const aldm_t5_embed_desc* d, void* stream) {
  if (!d) { aldm::set_error("aldm_t5_embed: null desc"); return ALDM_E_ARG; }
  return aldm::t5_embed_launch(*d, reinterpret_cast<cudaStream_t>(stream));
}
extern "C" int aldm_t5_rmsnorm(const aldm_t5_rmsnorm_desc* d, void* stream) {
  if (!d) { aldm::set_error("aldm_t5_rmsnorm: null desc"); return ALDM_E_ARG; }
  return aldm::t5_rmsnorm_launch(*d, reinterpret_cast<cudaStream_t>(stream));
}
extern "C" int aldm_t5_attention(const aldm_t5_attn_desc* d, void* stream) {
  if (!d) { aldm::set_error("aldm_t5_attention: null desc"); return ALDM_E_ARG; }
  return aldm::t5_attention_launch(*d, reinterpret_cast<cudaStream_t>(stream));
}
extern "C" int aldm_t5_gate(const aldm_t5_gate_desc* d, void* stream) {
  if (!d) { aldm::set_error("aldm_t5_gate: null desc"); return ALDM_E_ARG; }
  return aldm::t5_gate_launch(*d, reinterpret_cast<cudaStream_t>(stream));
}
