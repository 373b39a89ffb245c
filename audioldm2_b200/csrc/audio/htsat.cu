// Audio encoder: the CLAP HTSAT-base audio branch (HTSAT_Swin_Transformer, clap/open_clip/htsat.py, non-fusion path) and
// audio_projection (clap/open_clip/model.py:564-568, 752-777), from the waveform to the L2-normalised audio embedding.
// The projections of every Swin block (qkv, proj, fc1, fc2) and of every PatchMerging (reduction) run on the tensor-core
// GEMM (csrc/gemm.cu) with two-plane operands; LN1 / LN2 are ALDM_PREP_LN and the erf-GELU is clap_gelu_kernel.  This file
// holds what is specific to HTSAT:
//   htsat_logmel_kernel            torchaudio resample 16 -> 48 kHz on the fly, torchlibrosa Spectrogram (periodic Hann,
//                                  reflect-centred, n_fft 1024, hop 480) as an FFT, power, melW, 10 log10, bn0
//   htsat_patch_kernel             reshape_wav2img (bicubic time interpolation to 1024 frames, the 4-chunk fold to
//                                  256 x 256), the 4 x 4 stride-4 patch conv with bias, LayerNorm(128)
//   htsat_window_attention_kernel  (shifted) window attention over 8 x 8 windows with the relative-position bias and the
//                                  shift mask, read from and written back to natural token order
//   htsat_merge_kernel             PatchMerging's 2 x 2 gather and LayerNorm(4C) -> operand planes of the reduction GEMM
//   htsat_head_kernel              final LayerNorm, the mean over tokens, audio_projection, F.normalize
// All arithmetic is fp32; every sum runs in a fixed order, no atomics.
#include "../common.cuh"

namespace aldm {

constexpr int HT_NFFT = 1024, HT_LOG2N = 10, HT_HOP = 480, HT_NBIN = HT_NFFT / 2 + 1, HT_MEL = 64;
constexpr int HT_RS_TAPS = 15, HT_RS_WIDTH = 7;       // torchaudio resample 16 -> 48 kHz: 3 phases x (2 * 7 + 1) taps
constexpr int HT_MAX_SAMPLES = 480000;                 // get_audio_features' max_len (clap/training/data.py:421-450)
constexpr int HT_FRAMES = 1024;                        // spec_size * freq_ratio: the time axis after interpolation
constexpr int HT_EMBED = 128, HT_GRID = 64, HT_WIN = 8, HT_WTOK = HT_WIN * HT_WIN, HT_HD = 32;

__device__ __forceinline__ float ht_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float ht_warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// One CTA per (frame, clip).  Sample i of the 48 kHz signal (i < L48 = min(up * L, 480000)): x[i] at 48 kHz; at 16 kHz
// torchaudio's resample (functional.py _apply_sinc_resample_kernel: zero padding of 7 left / 8 right, conv1d stride 1,
// output phase j = i mod 3) y[3q + j] = sum_m taps[j][m] x[q + m - 7], m = 0..14 in order.  The frame's 1024 samples are
// centred with reflect padding (torchlibrosa STFT center=True, pad_mode "reflect"), windowed by the periodic Hann window and
// transformed by a radix-2 FFT (as stft_mel_kernel); then power re^2 + im^2, mel[m] = sum_k power[k] melW[k, m] (one warp
// per mel bin, lane-strided partial sums and a fixed xor tree), 10 log10(max(mel, 1e-10)) (ref 1, no top_db) and bn0 with
// running statistics: (v - mean) * (1 / sqrt(var + eps)) * w + b.
__global__ void __launch_bounds__(256) htsat_logmel_kernel(const __grid_constant__ aldm_htsat_logmel_desc d) {
  __shared__ float2 s[HT_NFFT];
  __shared__ float2 tw[HT_NFFT / 2];
  __shared__ float pw[HT_NBIN];
  __shared__ float taps[3 * HT_RS_TAPS];
  const int f = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  for (int k = tid; k < HT_NFFT / 2; k += blockDim.x) {
    float sn, cs;
    sincospif(-2.0f * (float)k / (float)HT_NFFT, &sn, &cs);
    tw[k] = make_float2(cs, sn);
  }
  pdl_wait();
  if (d.up == 3)
    for (int k = tid; k < 3 * HT_RS_TAPS; k += blockDim.x) taps[k] = d.taps[k];
  __syncthreads();
  const float* w = d.wav + (long long)b * d.L;
  for (int n = tid; n < HT_NFFT; n += blockDim.x) {
    int i = f * HT_HOP + n - HT_NFFT / 2;
    if (i < 0) i = -i;
    if (i >= d.L48) i = 2 * (d.L48 - 1) - i;
    float x;
    if (d.up == 1) {
      x = w[i];
    } else {
      const int q = i / 3, j = i - 3 * q;
      const float* tj = taps + j * HT_RS_TAPS;
      x = 0.f;
#pragma unroll
      for (int m = 0; m < HT_RS_TAPS; ++m) {
        const int p = q + m - HT_RS_WIDTH;
        x = fmaf(tj[m], (p >= 0 && p < d.L) ? w[p] : 0.f, x);
      }
    }
    const float win = 0.5f - 0.5f * cospif(2.0f * (float)n / (float)HT_NFFT);
    const int r = (int)(__brev((unsigned)n) >> (32 - HT_LOG2N));
    s[r] = make_float2(x * win, 0.f);
  }
  __syncthreads();
#pragma unroll 1
  for (int st = 1; st <= HT_LOG2N; ++st) {
    const int half = 1 << (st - 1);
    for (int k = tid; k < HT_NFFT / 2; k += blockDim.x) {
      const int grp = k / half, j = k % half;
      const int i0 = grp * (half << 1) + j, i1 = i0 + half;
      const float2 t = tw[j << (HT_LOG2N - st)];
      const float2 a = s[i0], c = s[i1];
      const float2 m = make_float2(c.x * t.x - c.y * t.y, c.x * t.y + c.y * t.x);
      s[i0] = make_float2(a.x + m.x, a.y + m.y);
      s[i1] = make_float2(a.x - m.x, a.y - m.y);
    }
    __syncthreads();
  }
  for (int k = tid; k < HT_NBIN; k += blockDim.x) pw[k] = s[k].x * s[k].x + s[k].y * s[k].y;
  __syncthreads();
  const int lane = tid & 31, warp = tid >> 5;
  for (int m = warp; m < HT_MEL; m += (blockDim.x >> 5)) {
    float acc = 0.f;
    for (int k = lane; k < HT_NBIN; k += 32) acc = fmaf(pw[k], __ldg(d.melW + (long long)k * HT_MEL + m), acc);
    acc = ht_warp_sum(acc);
    if (lane == 0) {
      const float v = 10.0f * log10f(fmaxf(acc, 1e-10f));
      const float y = (v - d.bn_mean[m]) * (1.0f / sqrtf(d.bn_var[m] + d.eps)) * d.bn_w[m] + d.bn_b[m];
      d.out[((long long)b * d.T + f) * HT_MEL + m] = y;
    }
  }
}

// One warp per patch token (gh, gw) of the 64 x 64 grid, 4 tokens per block.  Lane k < 16 computes pixel (dy, dx) =
// (k / 4, k % 4) of the patch: image row r = 4 gh + dy holds mel bin r % 64 of chunk r / 64, column c = 4 gw + dx is frame
// t' = 256 (r / 64) + c of the time axis interpolated to 1024 frames (reshape_wav2img, htsat.py:1074-1101).  The
// interpolation is upsample_bicubic2d with align_corners: source x = ((T - 1) / 1023) t' in fp32, i0 = floor(x), the four
// cubic-convolution weights of t = x - i0 (A = -0.75) on rows i0 - 1 .. i0 + 2 clamped to [0, T), summed in that order (the
// mel axis maps 64 -> 64 onto itself: weights 0, 1, 0, 0, exact).  Then every lane holds channels 4 lane .. 4 lane + 3:
// bias + the 16 taps in (dy, dx) order, and LayerNorm(128) with two-pass statistics.  Output: the fp32 residual stream,
// row b * 4096 + gh * 64 + gw.
constexpr int HT_PATCH_WARPS = 4;
__device__ __forceinline__ float ht_cubic1(float x, float A) { return ((A + 2.0f) * x - (A + 3.0f)) * x * x + 1.0f; }
__device__ __forceinline__ float ht_cubic2(float x, float A) { return ((A * x - 5.0f * A) * x + 8.0f * A) * x - 4.0f * A; }
__global__ void __launch_bounds__(HT_PATCH_WARPS * 32) htsat_patch_kernel(const __grid_constant__ aldm_htsat_patch_desc d) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * HT_PATCH_WARPS + (threadIdx.x >> 5);
  const int b = r / (HT_GRID * HT_GRID), tok = r - b * HT_GRID * HT_GRID;
  const int gh = tok / HT_GRID, gw = tok - gh * HT_GRID;
  pdl_wait();
  if (b >= d.n) return;
  float pix = 0.f;
  if (lane < 16) {
    const int row = 4 * gh + (lane >> 2), col = 4 * gw + (lane & 3);
    const int chunk = row / HT_MEL, mel = row - chunk * HT_MEL;
    const int tp = chunk * (HT_FRAMES / 4) + col;
    const float scale = (float)(d.T - 1) / (float)(HT_FRAMES - 1);
    const float x = scale * (float)tp;
    const int i0 = min((int)floorf(x), d.T - 1);
    const float t = fminf(fmaxf(x - (float)i0, 0.f), 1.f);
    const float A = -0.75f;
    const float t2 = 1.0f - t;                        // get_cubic_upsample_coefficients' x2
    const float c0 = ht_cubic2(t + 1.0f, A), c1 = ht_cubic1(t, A), c2 = ht_cubic1(t2, A), c3 = ht_cubic2(t2 + 1.0f, A);
    const float* src = d.mel + (long long)b * d.T * HT_MEL + mel;
    const float x0 = src[(long long)min(max(i0 - 1, 0), d.T - 1) * HT_MEL];
    const float x1 = src[(long long)min(max(i0, 0), d.T - 1) * HT_MEL];
    const float x2 = src[(long long)min(max(i0 + 1, 0), d.T - 1) * HT_MEL];
    const float x3 = src[(long long)min(max(i0 + 2, 0), d.T - 1) * HT_MEL];
    pix = x0 * c0;
    pix += x1 * c1;
    pix += x2 * c2;
    pix += x3 * c3;
  }
  float v[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) v[e] = __ldg(d.bias + lane * 4 + e);
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    const float p = __shfl_sync(0xffffffffu, pix, k);
#pragma unroll
    for (int e = 0; e < 4; ++e) v[e] = fmaf(__ldg(d.w + (lane * 4 + e) * 16 + k), p, v[e]);
  }
  const float mean = ht_warp_sum((v[0] + v[1]) + (v[2] + v[3])) / (float)HT_EMBED;
  float q = 0.f;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    v[e] -= mean;
    q = fmaf(v[e], v[e], q);
  }
  const float rs = 1.0f / sqrtf(ht_warp_sum(q) / (float)HT_EMBED + d.eps);
  const float4 g = __ldg(reinterpret_cast<const float4*>(d.gamma) + lane);
  const float4 be = __ldg(reinterpret_cast<const float4*>(d.beta) + lane);
  *reinterpret_cast<float4*>(d.out + (long long)r * HT_EMBED + lane * 4) =
      make_float4(fmaf(v[0] * rs, g.x, be.x), fmaf(v[1] * rs, g.y, be.y), fmaf(v[2] * rs, g.z, be.z),
                  fmaf(v[3] * rs, g.w, be.w));
}

// Block = (window, head, clip), 4 warps; warp w owns the window's queries 16 w .. 16 w + 15.  Window (wh, ww) of an R x R
// grid rolled by -shift (torch.roll, htsat.py:584-590) holds at position p = 8 i + j the token
// ((8 wh + i + shift) mod R) * R + (8 ww + j + shift) mod R; the output of p goes back to that same token, which is what
// window_reverse and the +shift roll do.  q, k, v (head h: columns h * 32 + [0, 32) of each third of the QKV GEMM's fp32
// output) are staged in shared memory (rows padded to 33 floats).  Per query: lane owns keys lane and lane + 32,
// s = (scale * q) . k summed over d in order (q is scaled first, as the reference does), + bias[h, p, key] + mask[w, p, key]
// (0 / -100 where the shifted window joins regions that are not adjacent), then the warp max, exp(s - max) and a fixed xor
// sum; P V with lane = output dimension, keys in order, divided by the sum and split into two fp16 planes.
constexpr int HT_ATT_WARPS = 4;
constexpr int HT_ATT_LD = HT_HD + 1;
__global__ void __launch_bounds__(HT_ATT_WARPS * 32) htsat_window_attention_kernel(const __grid_constant__ aldm_htsat_attn_desc d) {
  __shared__ float q_s[HT_WTOK * HT_ATT_LD], k_s[HT_WTOK * HT_ATT_LD], v_s[HT_WTOK * HT_ATT_LD];
  __shared__ float p_s[HT_ATT_WARPS][HT_WTOK];
  __shared__ int tok_s[HT_WTOK];
  const int win = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nww = d.R / HT_WIN, wh = win / nww, ww = win - wh * nww;
  if (tid < HT_WTOK) {
    const int i = tid >> 3, j = tid & 7;
    const int y = (wh * HT_WIN + i + d.shift) % d.R, x = (ww * HT_WIN + j + d.shift) % d.R;
    tok_s[tid] = y * d.R + x;
  }
  __syncthreads();
  pdl_wait();
  const float* base = d.qkv + (long long)b * d.R * d.R * d.ld_qkv + h * HT_HD;
  for (int e = tid; e < HT_WTOK * HT_HD; e += HT_ATT_WARPS * 32) {
    const int p = e >> 5, c = e & 31;
    const float* row = base + (long long)tok_s[p] * d.ld_qkv + c;
    q_s[p * HT_ATT_LD + c] = row[0] * d.scale;
    k_s[p * HT_ATT_LD + c] = row[d.C];
    v_s[p * HT_ATT_LD + c] = row[2 * d.C];
  }
  __syncthreads();
  const float* bias = d.bias + (long long)h * HT_WTOK * HT_WTOK;
  const float* mask = d.mask ? d.mask + (long long)win * HT_WTOK * HT_WTOK : nullptr;
  float* pw = p_s[warp];
  for (int qi = 0; qi < HT_WTOK / HT_ATT_WARPS; ++qi) {
    const int p = warp * (HT_WTOK / HT_ATT_WARPS) + qi;
    const float* qr = q_s + p * HT_ATT_LD;
    float s0 = 0.f, s1 = 0.f;
#pragma unroll 8
    for (int c = 0; c < HT_HD; ++c) {
      const float qv = qr[c];
      s0 = fmaf(qv, k_s[lane * HT_ATT_LD + c], s0);
      s1 = fmaf(qv, k_s[(lane + 32) * HT_ATT_LD + c], s1);
    }
    s0 += __ldg(bias + p * HT_WTOK + lane);
    s1 += __ldg(bias + p * HT_WTOK + lane + 32);
    if (mask) {
      s0 += __ldg(mask + p * HT_WTOK + lane);
      s1 += __ldg(mask + p * HT_WTOK + lane + 32);
    }
    const float mx = ht_warp_max(fmaxf(s0, s1));
    const float e0 = expf(s0 - mx), e1 = expf(s1 - mx);
    const float sum = ht_warp_sum(e0 + e1);
    pw[lane] = e0;
    pw[lane + 32] = e1;
    __syncwarp();
    float o = 0.f;
    for (int j = 0; j < HT_WTOK; ++j) o = fmaf(pw[j], v_s[j * HT_ATT_LD + lane], o);
    __syncwarp();
    const long long orow = ((long long)b * d.R * d.R + tok_s[p]) * d.ldo + h * HT_HD;
    store_split1(reinterpret_cast<aldm_plane_t*>(d.out_hi) + orow,
                 d.out_lo ? reinterpret_cast<aldm_plane_t*>(d.out_lo) + orow : nullptr, lane, o / sum);
  }
}

// One warp per output token (a, b) of the R/2 x R/2 grid, 4 per block.  Lane l holds the float4 chunks l, l + 32, ... of
// the 4C-wide row torch.cat([x(2a, 2b), x(2a+1, 2b), x(2a, 2b+1), x(2a+1, 2b+1)]) (htsat.py:664-668); LayerNorm(4C) with
// two-pass statistics (per lane in chunk order, then a fixed xor tree) and the planes of the reduction GEMM.
constexpr int HT_MERGE_WARPS = 4;
template <int NV>
__global__ void __launch_bounds__(HT_MERGE_WARPS * 32) htsat_merge_kernel(const __grid_constant__ aldm_htsat_merge_desc d) {
  const int lane = threadIdx.x & 31;
  const int Ro = d.R / 2;
  const long long r = (long long)blockIdx.x * HT_MERGE_WARPS + (threadIdx.x >> 5);
  pdl_wait();
  if (r >= (long long)d.n * Ro * Ro) return;
  const int b = (int)(r / (Ro * Ro)), t = (int)(r - (long long)b * Ro * Ro);
  const int a = t / Ro, c2 = t - a * Ro;
  constexpr int C = NV * 32, C4 = 4 * C;           // C is 128, 256 or 512
  float4 v[NV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = (i * 32 + lane) * 4;
    const int qd = c / C, cc = c - qd * C;
    const int y = 2 * a + (qd & 1), x = 2 * c2 + (qd >> 1);
    v[i] = *reinterpret_cast<const float4*>(d.x + ((long long)b * d.R * d.R + (long long)y * d.R + x) * C + cc);
    s += v[i].x; s += v[i].y; s += v[i].z; s += v[i].w;
  }
  const float mean = ht_warp_sum(s) / (float)C4;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    v[i].x -= mean; v[i].y -= mean; v[i].z -= mean; v[i].w -= mean;
    q = fmaf(v[i].x, v[i].x, q); q = fmaf(v[i].y, v[i].y, q);
    q = fmaf(v[i].z, v[i].z, q); q = fmaf(v[i].w, v[i].w, q);
  }
  const float rs = 1.0f / sqrtf(ht_warp_sum(q) / (float)C4 + d.eps);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = (i * 32 + lane) * 4;
    const float4 g = __ldg(reinterpret_cast<const float4*>(d.gamma + c));
    const float4 be = __ldg(reinterpret_cast<const float4*>(d.beta + c));
    uint2 hi, lo;
    split2(fmaf(v[i].x * rs, g.x, be.x), fmaf(v[i].y * rs, g.y, be.y), hi.x, lo.x);
    split2(fmaf(v[i].z * rs, g.z, be.z), fmaf(v[i].w * rs, g.w, be.w), hi.y, lo.y);
    *reinterpret_cast<uint2*>(reinterpret_cast<aldm_plane_t*>(d.out_hi) + r * d.ldo + c) = hi;
    if (d.out_lo) *reinterpret_cast<uint2*>(reinterpret_cast<aldm_plane_t*>(d.out_lo) + r * d.ldo + c) = lo;
  }
}

// One block per clip, fp32.  For each token t = 0 .. ntok-1 in order: LayerNorm over C with two-pass block statistics
// (thread partials over its channels tid, tid + 512, then a fixed warp tree and warp partials summed in order), and each
// thread adds the normalised values of its channels to a running sum -- the mean over tokens is then sum / ntok (the
// "embedding" output: avgpool over all tokens; the reshapes before it only permute them, htsat.py:1021-1039).  Then
// audio_projection: Linear(C -> P), ReLU, Linear(P -> P) (weights transposed, [in, out]), and F.normalize.
constexpr int HT_HEAD_T = 512;
constexpr int HT_HEAD_MAXC = 1024;
constexpr int HT_HEAD_MAXP = 1024;
__device__ __forceinline__ float ht_block_sum(float v, float* red) {
  v = ht_warp_sum(v);
  __syncthreads();                                    // red is free again
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
  for (int w = 0; w < HT_HEAD_T / 32; ++w) t += red[w];
  return t;
}
__global__ void __launch_bounds__(HT_HEAD_T) htsat_head_kernel(const __grid_constant__ aldm_htsat_head_desc d) {
  __shared__ float m_s[HT_HEAD_MAXC], t_s[HT_HEAD_MAXP], y_s[HT_HEAD_MAXP];
  __shared__ float red[HT_HEAD_T / 32];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int C = d.C, P = d.P;
  const bool has0 = tid < C, has1 = tid + HT_HEAD_T < C;
  pdl_wait();
  const float g0 = has0 ? d.gamma[tid] : 0.f, be0 = has0 ? d.beta[tid] : 0.f;
  const float g1 = has1 ? d.gamma[tid + HT_HEAD_T] : 0.f, be1 = has1 ? d.beta[tid + HT_HEAD_T] : 0.f;
  float acc0 = 0.f, acc1 = 0.f;
  for (int t = 0; t < d.ntok; ++t) {
    const float* xr = d.x + ((long long)b * d.ntok + t) * C;
    const float x0 = has0 ? xr[tid] : 0.f, x1 = has1 ? xr[tid + HT_HEAD_T] : 0.f;
    const float mean = ht_block_sum(x0 + x1, red) / (float)C;
    const float y0 = has0 ? x0 - mean : 0.f, y1 = has1 ? x1 - mean : 0.f;
    const float rs = 1.0f / sqrtf(ht_block_sum(fmaf(y0, y0, y1 * y1), red) / (float)C + d.eps);
    acc0 += fmaf(y0 * rs, g0, be0);
    acc1 += fmaf(y1 * rs, g1, be1);
  }
  if (has0) m_s[tid] = acc0 / (float)d.ntok;
  if (has1) m_s[tid + HT_HEAD_T] = acc1 / (float)d.ntok;
  __syncthreads();
  for (int n = tid; n < P; n += HT_HEAD_T) {          // audio_projection[0], ReLU
    float a = 0.f;
    for (int k = 0; k < C; ++k) a = fmaf(m_s[k], __ldg(d.w1_t + (long long)k * P + n), a);
    t_s[n] = fmaxf(a + __ldg(d.b1 + n), 0.f);
  }
  __syncthreads();
  float ss = 0.f;
  for (int n = tid; n < P; n += HT_HEAD_T) {          // audio_projection[2]
    float a = 0.f;
    for (int k = 0; k < P; ++k) a = fmaf(t_s[k], __ldg(d.w2_t + (long long)k * P + n), a);
    a += __ldg(d.b2 + n);
    y_s[n] = a;
    ss = fmaf(a, a, ss);
  }
  const float den = fmaxf(sqrtf(ht_block_sum(ss, red)), 1e-12f);     // F.normalize: x / max(||x||_2, eps)
  for (int n = tid; n < P; n += HT_HEAD_T) d.out[(long long)b * P + n] = y_s[n] / den;
}

int htsat_logmel_launch(const aldm_htsat_logmel_desc& d, cudaStream_t st) {
  ALDM_REQUIRE(d.wav && d.melW && d.bn_mean && d.bn_var && d.bn_w && d.bn_b && d.out && (d.up == 1 || d.taps), ALDM_E_ARG,
               "htsat_logmel: null pointer");
  ALDM_REQUIRE(d.up == 1 || d.up == 3, ALDM_E_UNSUPPORTED, "htsat_logmel: up=%d (1: 48 kHz input, 3: 16 kHz input)", d.up);
  ALDM_REQUIRE(d.n > 0 && d.n <= 65535 && d.L > 0 && d.L48 == min((long long)d.up * d.L, (long long)HT_MAX_SAMPLES) &&
                   d.L48 > HT_NFFT / 2 && d.T == d.L48 / HT_HOP + 1,
               ALDM_E_SHAPE, "htsat_logmel: n=%d L=%d up=%d L48=%d T=%d (L48 = min(up L, %d) > %d, T = L48 / %d + 1)", d.n,
               d.L, d.up, d.L48, d.T, HT_MAX_SAMPLES, HT_NFFT / 2, HT_HOP);
  ALDM_CHECK_CUDA(launch_pdl(htsat_logmel_kernel, dim3(d.T, d.n), dim3(256), 0, st, d));
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}

int htsat_patch_launch(const aldm_htsat_patch_desc& d, cudaStream_t st) {
  ALDM_REQUIRE(d.mel && d.w && d.bias && d.gamma && d.beta && d.out, ALDM_E_ARG, "htsat_patch: null pointer");
  ALDM_REQUIRE(d.n > 0 && d.n <= 65535 && d.T >= 2 && d.T <= HT_FRAMES, ALDM_E_SHAPE, "htsat_patch: n=%d T=%d (2 .. %d)", d.n,
               d.T, HT_FRAMES);
  ALDM_REQUIRE(aligned16(d.gamma) && aligned16(d.beta) && aligned16(d.out), ALDM_E_ALIGN, "htsat_patch: alignment");
  const int rows = d.n * HT_GRID * HT_GRID;
  ALDM_CHECK_CUDA(launch_pdl(htsat_patch_kernel, dim3(cdiv(rows, HT_PATCH_WARPS)), dim3(HT_PATCH_WARPS * 32), 0, st, d));
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}

int htsat_window_attention_launch(const aldm_htsat_attn_desc& d, cudaStream_t st) {
  ALDM_REQUIRE(d.qkv && d.bias && d.out_hi, ALDM_E_ARG, "htsat_window_attention: null pointer");
  ALDM_REQUIRE(d.head_dim == HT_HD, ALDM_E_UNSUPPORTED, "htsat_window_attention: head_dim=%d (only %d)", d.head_dim, HT_HD);
  ALDM_REQUIRE(d.n > 0 && d.n <= 65535 && d.heads > 0 && d.heads <= 65535 && d.heads * HT_HD == d.C && d.R >= HT_WIN &&
                   d.R % HT_WIN == 0 && d.shift >= 0 && d.shift < HT_WIN && (d.shift == 0 || d.mask) &&
                   d.ld_qkv >= 3 * d.C && d.ldo >= d.C,
               ALDM_E_SHAPE, "htsat_window_attention: n=%d R=%d shift=%d heads=%d C=%d ld_qkv=%d ldo=%d", d.n, d.R, d.shift,
               d.heads, d.C, d.ld_qkv, d.ldo);
  const int nW = (d.R / HT_WIN) * (d.R / HT_WIN);
  ALDM_CHECK_CUDA(launch_pdl(htsat_window_attention_kernel, dim3(nW, d.heads, d.n), dim3(HT_ATT_WARPS * 32), 0, st, d));
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}

int htsat_merge_launch(const aldm_htsat_merge_desc& d, cudaStream_t st) {
  ALDM_REQUIRE(d.x && d.gamma && d.beta && d.out_hi, ALDM_E_ARG, "htsat_merge: null pointer");
  ALDM_REQUIRE(d.n > 0 && d.R >= 2 && d.R % 2 == 0 && (d.C == 128 || d.C == 256 || d.C == 512) && d.ldo >= 4 * d.C &&
                   d.ldo % 4 == 0,
               ALDM_E_SHAPE, "htsat_merge: n=%d R=%d C=%d ldo=%d (C 128, 256 or 512)", d.n, d.R, d.C, d.ldo);
  ALDM_REQUIRE(aligned16(d.x) && aligned16(d.gamma) && aligned16(d.beta), ALDM_E_ALIGN, "htsat_merge: alignment");
  const long long rows = (long long)d.n * (d.R / 2) * (d.R / 2);
  const dim3 grid((unsigned)cdiv(rows, (long long)HT_MERGE_WARPS)), block(HT_MERGE_WARPS * 32);
  if (d.C == 128) ALDM_CHECK_CUDA(launch_pdl(htsat_merge_kernel<4>, grid, block, 0, st, d));
  else if (d.C == 256) ALDM_CHECK_CUDA(launch_pdl(htsat_merge_kernel<8>, grid, block, 0, st, d));
  else ALDM_CHECK_CUDA(launch_pdl(htsat_merge_kernel<16>, grid, block, 0, st, d));
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}

int htsat_head_launch(const aldm_htsat_head_desc& d, cudaStream_t st) {
  ALDM_REQUIRE(d.x && d.gamma && d.beta && d.w1_t && d.b1 && d.w2_t && d.b2 && d.out, ALDM_E_ARG, "htsat_head: null pointer");
  ALDM_REQUIRE(d.n > 0 && d.n <= 65535 && d.ntok > 0 && d.C > 0 && d.C <= HT_HEAD_MAXC && d.P > 0 && d.P <= HT_HEAD_MAXP,
               ALDM_E_SHAPE, "htsat_head: n=%d ntok=%d C=%d P=%d (C, P <= %d)", d.n, d.ntok, d.C, d.P, HT_HEAD_MAXC);
  ALDM_CHECK_CUDA(launch_pdl(htsat_head_kernel, dim3(d.n), dim3(HT_HEAD_T), 0, st, d));
  ALDM_CHECK_CUDA(cudaGetLastError());
  return ALDM_OK;
}

}  // namespace aldm

extern "C" int aldm_htsat_logmel(const aldm_htsat_logmel_desc* d, void* stream) {
  if (!d) { aldm::set_error("aldm_htsat_logmel: null desc"); return ALDM_E_ARG; }
  return aldm::htsat_logmel_launch(*d, reinterpret_cast<cudaStream_t>(stream));
}
extern "C" int aldm_htsat_patch(const aldm_htsat_patch_desc* d, void* stream) {
  if (!d) { aldm::set_error("aldm_htsat_patch: null desc"); return ALDM_E_ARG; }
  return aldm::htsat_patch_launch(*d, reinterpret_cast<cudaStream_t>(stream));
}
extern "C" int aldm_htsat_window_attention(const aldm_htsat_attn_desc* d, void* stream) {
  if (!d) { aldm::set_error("aldm_htsat_window_attention: null desc"); return ALDM_E_ARG; }
  return aldm::htsat_window_attention_launch(*d, reinterpret_cast<cudaStream_t>(stream));
}
extern "C" int aldm_htsat_merge(const aldm_htsat_merge_desc* d, void* stream) {
  if (!d) { aldm::set_error("aldm_htsat_merge: null desc"); return ALDM_E_ARG; }
  return aldm::htsat_merge_launch(*d, reinterpret_cast<cudaStream_t>(stream));
}
extern "C" int aldm_htsat_head(const aldm_htsat_head_desc* d, void* stream) {
  if (!d) { aldm::set_error("aldm_htsat_head: null desc"); return ALDM_E_ARG; }
  return aldm::htsat_head_launch(*d, reinterpret_cast<cudaStream_t>(stream));
}
