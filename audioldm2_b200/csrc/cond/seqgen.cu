// Conditioning stage: the AudioMAE token generator of the sequence-generation models (GPT-2 small over the CLAP and
// Flan-T5 encodings, audiomae_gen/sequence_input.py:110-201,294-325) with a KV cache.  The four linear layers of every
// GPT-2 block and both input projections run on the tensor-core GEMM (csrc/gemm.cu), ln_1 / ln_2 on the LayerNorm prep
// kernel; this file holds what is specific to autoregressive generation:
//   seq_assemble_kernel  the prefill residual stream [sos0, clap, eos0, sos1, t5, eos1] + wpe and the key mask
//   kv_attention_kernel  causal attention of the new positions against every cached position (prefill and decode)
//   seq_feedback_kernel  ln_f of the last position -> generated token, and token + wpe as the next pass's input
// Everything is fp32: the sequence buffer the c_attn GEMM writes (q | k | v per position), the softmax, the accumulation
// and the fed-back hidden state (the reference feeds the fp32 ln_f output back as an input embedding).
#include "../common.cuh"

namespace aldm {

constexpr int KV_HD = 64;            // GPT-2 head dimension
constexpr int KV_MAX = 1024;         // n_positions
constexpr int KV_THREADS = 256;      // 8 warps

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// One block per (query, head, batch row).  Scores: warp w takes keys w, w + 8, ...; lanes hold q[lane], q[lane + 32]
// and read the key's 64 values as two coalesced 128-byte lines, a fixed shuffle tree sums them.  Masked keys (causal
// limit or mask != 1) get probability 0 exactly, which equals the reference's finfo.min fill once a key is unmasked
// (key 0 always is).  P V: thread t owns dimension t & 63 of key group t >> 6 (keys g, g + 4, ...); the four partial
// sums are added in a fixed order.  Everything is deterministic.
__global__ void __launch_bounds__(KV_THREADS) kv_attention_kernel(const __grid_constant__ aldm_kv_attn_desc d) {
  __shared__ float q_s[KV_HD];
  __shared__ float p_s[KV_MAX];
  __shared__ float part[4][KV_HD];
  __shared__ float red[KV_THREADS / 32];
  const int qi = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int C = d.heads * KV_HD;
  const int pos = d.p0 + qi;
  const int nk = pos + 1;
  const float* seq = d.seq + (long long)b * d.lmax * d.ld_seq;
  const float* mrow = d.mask + (long long)b * d.lmax;
  pdl_wait();
  if (tid < KV_HD) q_s[tid] = seq[(long long)pos * d.ld_seq + h * KV_HD + tid];
  __syncthreads();
  const float qa = q_s[lane], qb = q_s[lane + 32];
  float mx = -INFINITY;
  for (int j = warp; j < nk; j += KV_THREADS / 32) {
    const float* kr = seq + (long long)j * d.ld_seq + C + h * KV_HD;
    float s = warp_sum(fmaf(qa, kr[lane], qb * kr[lane + 32])) * d.scale;
    s = mrow[j] == 1.0f ? s : -INFINITY;
    if (lane == 0) p_s[j] = s;
    mx = fmaxf(mx, s);
  }
  mx = warp_max(mx);
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int w = 1; w < KV_THREADS / 32; ++w) mx = fmaxf(mx, red[w]);
  __syncthreads();                      // everyone has read red[] before it is reused for the sums
  float sum = 0.f;
  for (int j = tid; j < nk; j += KV_THREADS) {
    const float e = expf(p_s[j] - mx);
    p_s[j] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  if (lane == 0) red[warp] = sum;
  __syncthreads();                      // p_s complete, red[] holds the warp sums
  sum = 0.f;
#pragma unroll
  for (int w = 0; w < KV_THREADS / 32; ++w) sum += red[w];
  const int dim = tid & (KV_HD - 1), g = tid >> 6;
  const float* vcol = seq + 2 * C + h * KV_HD + dim;
  float acc = 0.f;
  for (int j = g; j < nk; j += 4) acc = fmaf(p_s[j], vcol[(long long)j * d.ld_seq], acc);
  part[g][dim] = acc;
  __syncthreads();
  if (tid < KV_HD) {
    const float o = (((part[0][tid] + part[1][tid]) + part[2][tid]) + part[3][tid]) / sum;
    const long long row = (long long)b * d.nq + qi;
    aldm_plane_t* hp = reinterpret_cast<aldm_plane_t*>(d.out_hi) + row * d.ldo + h * KV_HD;
    aldm_plane_t* lp = d.out_lo ? reinterpret_cast<aldm_plane_t*>(d.out_lo) + row * d.ldo + h * KV_HD : nullptr;
    store_split1(hp, lp, tid, o);
  }
}

// One block per (position, batch row), one thread per 4 channels.
__global__ void seq_assemble_kernel(const __grid_constant__ aldm_seq_assemble_desc d) {
  const int p = blockIdx.x, b = blockIdx.y;
  const int P = d.L + 5;
  pdl_wait();
  float* xr = d.x + ((long long)b * P + p) * d.C;
  const float* tok = nullptr;          // SOS / EOS row, or NULL for a projected row (already in x)
  if (p == 0) tok = d.sos;
  else if (p == 2) tok = d.eos;
  else if (p == 3) tok = d.sos + d.C;
  else if (p == P - 1) tok = d.eos + d.C;
  for (int c = threadIdx.x * 4; c < d.C; c += blockDim.x * 4) {
    const float4 w = __ldg(reinterpret_cast<const float4*>(d.wpe + (long long)p * d.C + c));
    float4 v = tok ? __ldg(reinterpret_cast<const float4*>(tok + c)) : *reinterpret_cast<const float4*>(xr + c);
    v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w;
    *reinterpret_cast<float4*>(xr + c) = v;
  }
  // key mask: block p of row b writes positions p, p + P, p + 2P, ... (the generated positions P.. are all 1)
  if (threadIdx.x == 0) {
    const bool t5 = p >= 4 && p < 4 + d.L;
    d.mask[(long long)b * d.lmax + p] = t5 ? d.t5_mask[(long long)b * d.L + (p - 4)] : 1.0f;
    for (int q = p + P; q < d.lmax; q += P) d.mask[(long long)b * d.lmax + q] = 1.0f;
  }
}

// One block per batch row; thread t holds channels t, t + 256, ... (C <= 1024).  Two-pass fp32 statistics, combined by a
// fixed shuffle tree and a fixed-order sum of the warp results.
constexpr int FB_THREADS = 256;
__global__ void __launch_bounds__(FB_THREADS) seq_feedback_kernel(const __grid_constant__ aldm_seq_feedback_desc d) {
  __shared__ float red[FB_THREADS / 32];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  pdl_wait();
  const float* xr = d.x + ((long long)b * d.nq + d.nq - 1) * d.C;
  float v[4];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = tid + FB_THREADS * i;
    v[i] = c < d.C ? xr[c] : 0.f;
    s += v[i];
  }
  s = warp_sum(s);
  if (lane == 0) red[warp] = s;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < FB_THREADS / 32; ++w) tot += red[w];
  const float mean = tot / d.C;
  __syncthreads();
  float s2 = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = tid + FB_THREADS * i;
    if (c < d.C) { const float e = v[i] - mean; s2 = fmaf(e, e, s2); }
  }
  s2 = warp_sum(s2);
  if (lane == 0) red[warp] = s2;
  __syncthreads();
  float var = 0.f;
#pragma unroll
  for (int w = 0; w < FB_THREADS / 32; ++w) var += red[w];
  const float rstd = 1.0f / sqrtf(var / d.C + d.eps);
  float* orow = d.out + ((long long)b * d.gen_len + d.k) * d.C;
  float* nrow = d.next ? d.next + (long long)b * d.C : nullptr;
  const float* wrow = d.wpe + (long long)(d.pos + 1) * d.C;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = tid + FB_THREADS * i;
    if (c < d.C) {
      const float y = (v[i] - mean) * rstd * __ldg(d.gamma + c) + __ldg(d.beta + c);
      orow[c] = y;
      if (nrow) nrow[c] = y + __ldg(wrow + c);
    }
  }
}

int kv_attention_launch(const aldm_kv_attn_desc& d, cudaStream_t st) {
  ALDM_REQUIRE(d.seq && d.mask && d.out_hi, ALDM_E_ARG, "kv_attention: null pointer");
  ALDM_REQUIRE(d.B > 0 && d.heads > 0 && d.nq > 0 && d.p0 >= 0, ALDM_E_SHAPE, "kv_attention: B=%d heads=%d nq=%d p0=%d", d.B,
               d.heads, d.nq, d.p0);
  ALDM_REQUIRE(d.lmax <= KV_MAX && d.p0 + d.nq <= d.lmax, ALDM_E_SHAPE, "kv_attention: positions [%d, %d) beyond lmax=%d (<= %d)",
               d.p0, d.p0 + d.nq, d.lmax, KV_MAX);
  ALDM_REQUIRE(d.ld_seq >= 3 * d.heads * KV_HD && d.ldo >= d.heads * KV_HD, ALDM_E_SHAPE, "kv_attention: ld_seq=%d ldo=%d",
               d.ld_seq, d.ldo);
  ALDM_REQUIRE(d.nq <= 65535 && d.heads <= 65535 && d.B <= 65535, ALDM_E_SHAPE, "kv_attention: grid");
  ALDM_CHECK_CUDA(launch_pdl(kv_attention_kernel, dim3(d.nq, d.heads, d.B), dim3(KV_THREADS), 0, st, d));
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}

int seq_assemble_launch(const aldm_seq_assemble_desc& d, cudaStream_t st) {
  ALDM_REQUIRE(d.x && d.sos && d.eos && d.wpe && d.t5_mask && d.mask, ALDM_E_ARG, "seq_assemble: null pointer");
  ALDM_REQUIRE(d.B > 0 && d.L > 0 && d.C > 0 && d.C % 4 == 0 && d.lmax >= d.L + 5 && d.lmax <= KV_MAX, ALDM_E_SHAPE,
               "seq_assemble: B=%d L=%d C=%d lmax=%d", d.B, d.L, d.C, d.lmax);
  ALDM_REQUIRE(aligned16(d.x) && aligned16(d.sos) && aligned16(d.eos) && aligned16(d.wpe), ALDM_E_ALIGN, "seq_assemble: alignment");
  ALDM_CHECK_CUDA(launch_pdl(seq_assemble_kernel, dim3(d.L + 5, d.B), dim3(192), 0, st, d));
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}

int seq_feedback_launch(const aldm_seq_feedback_desc& d, cudaStream_t st) {
  ALDM_REQUIRE(d.x && d.gamma && d.beta && d.out && (d.wpe || !d.next), ALDM_E_ARG, "seq_feedback: null pointer");
  ALDM_REQUIRE(d.B > 0 && d.nq > 0 && d.C > 0 && d.C <= 4 * FB_THREADS && d.k >= 0 && d.k < d.gen_len && d.pos >= 0 &&
                   (!d.next || d.pos + 1 < KV_MAX),
               ALDM_E_SHAPE, "seq_feedback: B=%d nq=%d C=%d k=%d gen_len=%d pos=%d", d.B, d.nq, d.C, d.k, d.gen_len, d.pos);
  ALDM_CHECK_CUDA(launch_pdl(seq_feedback_kernel, dim3(d.B), dim3(FB_THREADS), 0, st, d));
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}

}  // namespace aldm

extern "C" int aldm_kv_attention(const aldm_kv_attn_desc* d, void* stream) {
  if (!d) { aldm::set_error("aldm_kv_attention: null desc"); return ALDM_E_ARG; }
  return aldm::kv_attention_launch(*d, reinterpret_cast<cudaStream_t>(stream));
}
extern "C" int aldm_seq_assemble(const aldm_seq_assemble_desc* d, void* stream) {
  if (!d) { aldm::set_error("aldm_seq_assemble: null desc"); return ALDM_E_ARG; }
  return aldm::seq_assemble_launch(*d, reinterpret_cast<cudaStream_t>(stream));
}
extern "C" int aldm_seq_feedback(const aldm_seq_feedback_desc* d, void* stream) {
  if (!d) { aldm::set_error("aldm_seq_feedback: null desc"); return ALDM_E_ARG; }
  return aldm::seq_feedback_launch(*d, reinterpret_cast<cudaStream_t>(stream));
}
