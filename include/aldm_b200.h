/*
 * aldm_b200.h -- C-ABI of the native AudioLDM2 sampling hot path (H100, sm_90a).
 *
 * Drop-in boundary (SURVEY.md 8b).  The reference (haoheliu/AudioLDM2) is pure Python/PyTorch;
 * its "FFI" for this path is the set of torch module calls listed below.  A Python host
 * (audioldm2_b200/engine.py, bound with ctypes -- see INTEGRATION.md) builds a flat table of
 * `aldm_op` records from the reference config dicts + state_dict and hands it to this library;
 * everything that touches the mel-latent tensor then runs as hand-written sm_90a kernels.
 *
 *   reference call (file:line)                                   replaced by
 *   -----------------------------------------------------------  ---------------------------------
 *   DiffusionWrapper.forward -> UNetModel.forward                aldm_program_run(unet program)
 *       latent_diffusion/models/ddpm.py:1821-1879,
 *       modules/diffusionmodules/openaimodel.py:837-885
 *   DDIMSampler.p_sample_ddim CFG combine + x_{t-1} update       aldm_ddim_step
 *       latent_diffusion/models/ddim.py:298-300,339-354
 *   masked blend + q_sample                                      aldm_ddim_step (mask != NULL)
 *   DDIMSampler.stochastic_encode (+ AudioLDM 1's latent guard)   aldm_stochastic_encode (style transfer)
 *       latent_diffusion/models/ddim.py:434-449
 *       models/ddim.py:226-231, models/ddpm.py:430-436
 *   PLMSSampler.p_sample_plms CFG combine + e' + x_{t-1} update  aldm_plms_step (one call per UNet evaluation;
 *       latent_diffusion/models/plms.py:288-292,319-360            the first step takes two)
 *   LatentDiffusion.decode_first_stage -> AutoencoderKL.decode   aldm_program_run(vae-decoder program)
 *       models/ddpm.py:922-926, latent_encoder/autoencoder.py:111-117,
 *       modules/diffusionmodules/model.py:653-686
 *   encode_first_stage -> Encoder.forward + quant_conv           aldm_program_run(vae-encoder program)
 *       models/ddpm.py:941-943, model.py:519-543, autoencoder.py:103-109
 *   first_stage_model.vocoder(mel)  (HiFi-GAN Generator.forward) aldm_program_run(vocoder program)
 *       models/ddpm.py:928-939, hifigan/models.py:149-165
 *   TacotronSTFT.mel_spectrogram                                 aldm_stft_mel
 *       utilities/audio/stft.py:159-178
 *   SequenceGenAudioMAECond.forward -> Sequence2AudioMAE.generate aldm_program_run(seqgen program: GPT-2 prefill +
 *       audiomae_gen/sequence_input.py:110-201,294-325,           7 KV-cached decode passes; ALDM_OP_SEQ_ASSEMBLE,
 *       encoders/modules.py:271-300                                ALDM_OP_KV_ATTN, ALDM_OP_SEQ_FEEDBACK)
 *   FlanT5HiddenState.encode_text -> T5EncoderModel (from the      aldm_program_run(t5 program: embedding + 24
 *       token ids)  encoders/modules.py:113-198                    blocks; ALDM_OP_T5_EMBED .. ALDM_OP_T5_GATE)
 *   CLAP.get_text_embedding (RoBERTa text branch, pooler,         aldm_program_run(clap program: embedding + LN +
 *       text_projection, F.normalize) clap/open_clip/model.py:     12 blocks + head; ALDM_OP_CLAP_EMBED ..
 *       656-663,730-750; encoders/modules.py:660-735               ALDM_OP_CLAP_HEAD)
 *   CLAP.get_audio_embedding (HTSAT-base audio branch,             aldm_program_run(clap audio program: log-mel, patch
 *       audio_projection, F.normalize) clap/open_clip/htsat.py,    embedding, 18 Swin blocks, 3 merges, head;
 *       model.py:752-777; encoders/modules.py:689-716              ALDM_OP_HTSAT_LOGMEL .. ALDM_OP_HTSAT_HEAD)
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless named host_*; buffers are caller-owned (torch
 *     tensors), 16-byte aligned, and must stay alive while a program that references them exists;
 *   - every entry point returns 0 on success or a negative ALDM_E_* code; no exceptions, no
 *     abort; `aldm_last_error()` returns a thread-local message;
 *   - kernels are enqueued on the caller's stream and never synchronise; there is no CPU
 *     fallback: an unsupported shape is ALDM_E_UNSUPPORTED.
 *   - activations are channels-last: [B, H, W, C] fp32 ("f32 tensors") or, when they feed a
 *     tensor-core GEMM, "operand planes": two bf16 arrays hi,lo of shape [rows, Cp] with
 *     x ~= hi + lo (Cp = C rounded up to 8).  Weights are packed by the host into 128-byte
 *     swizzled tile images (audioldm2_b200/packing.py).
 */
#ifndef ALDM_B200_H_
#define ALDM_B200_H_

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ALDM_ABI_VERSION 14
#define ALDM_MAX_TAPS 16

enum {
  ALDM_OK = 0,
  ALDM_E_ARG = -1,
  ALDM_E_SHAPE = -2,
  ALDM_E_ALIGN = -3,
  ALDM_E_CUDA = -4,
  ALDM_E_NOMEM = -5,
  ALDM_E_UNSUPPORTED = -6
};

/* ---- GEMM / implicit-GEMM convolution ---------------------------------------------------- */

enum { ALDM_GEMM_TC = 0, ALDM_GEMM_SIMT = 1, ALDM_GEMM_TC_V1 = 2 };   /* aldm_gemm_desc.impl: persistent wgmma | CUDA-core checker | retired, selects the persistent kernel */
/* OR-ed into aldm_gemm_desc.impl: w_packed is never written while the program runs (model weights), so the
 * kernel may start streaming it before its programmatic-dependency wait (overlapping the previous kernel's tail). */
#define ALDM_GEMM_STATIC_B (1 << 16)
/* ALDM_ACT_GELU_TANH: 0.5 v (1 + tanh(sqrt(2/pi) (v + 0.044715 v^3))), GPT-2's gelu_new (accurate tanhf) */
enum { ALDM_ACT_NONE = 0, ALDM_ACT_GEGLU = 1, ALDM_ACT_TANH = 2, ALDM_ACT_SILU = 3, ALDM_ACT_GELU_TANH = 4 };
enum { ALDM_OUT_F32 = 0, ALDM_OUT_PLANES = 1, ALDM_OUT_NCHW = 2, ALDM_OUT_QKV = 3 };

/* out[row(m), n] = epilogue( sum_k A[m, k] * W[n, k] ),  k = tap * Cp + c
 * A is gathered from operand planes laid out [B, Hs, Ws, Cp]:
 *    m -> (b, oh, ow);  ih = oh*sy + dy[tap], iw = ow*sx + dx[tap]  (zero outside [0,H)x[0,W));
 *    source pixel = (ih >> up, iw >> up), Hs = H >> up, Ws = W >> up; source batch = b % bmod.
 * epilogue: v = acc + bias[n] + rowvec[b*ld_rowvec + n]; v = act(v); v += res[row(m)*ld_res + n];
 *           v *= alpha; if (accumulate) v += out_old;  store.
 * GEGLU: weights are packed so that tile columns [0,BN/2) are values and [BN/2,BN) their gates;
 *        the stored width is N/2.
 * Output row mapping: orow = (b*OHF + oh*osy + ooy)*OWF + ow ; element = out[orow*ldo + n]
 *        (ALDM_OUT_NCHW: out[((b*N + n)*OH + oh)*OW + ow]).
 * ALDM_OUT_F32 with out_hi/out_lo != NULL: dual output, the values are additionally stored as operand
 *        planes [orow, ldo] (saves the copy-prep kernel in front of the next GEMM).
 * ALDM_OUT_QKV (attention projections): columns n < n_split go to the planes out_hi/out_lo
 *        [row m, ldo]; columns n >= n_split (the V projection) are stored TRANSPOSED into
 *        out2_hi/out2_lo[((m / tok_per_batch) * (N - n_split) + (n - n_split)) * ld_t + m % tok_per_batch]
 *        so that the attention kernel finds V^T K-major (keys contiguous).  n_split % bn == 0. */
typedef struct aldm_gemm_desc {
  const void* a_hi;          /* bf16 [B_src, Hs, Ws, Cp] */
  const void* a_lo;
  const void* w_packed;      /* tile images, see packing.py */
  const float* w_plain;      /* optional fp32 [N, Kpad] (SIMT reference path) */
  const float* bias;         /* [N] or NULL */
  const float* rowvec;       /* [B, ld_rowvec] or NULL (timestep-embedding add) */
  const float* res;          /* residual, same row mapping as out, or NULL */
  float* out;                /* fp32 output (ALDM_OUT_F32 / NCHW) */
  void* out_hi;              /* operand-plane output (ALDM_OUT_PLANES), [rows, ldo] bf16 */
  void* out_lo;
  void* out2_hi;             /* ALDM_OUT_QKV: transposed planes of the columns >= n_split */
  void* out2_lo;
  float* ws;                 /* split-K workspace [splitk, Mpad, Npad] fp32 or NULL */
  int32_t B, H, W, Cp;       /* logical conv input (after nearest-upsample if up=1) */
  int32_t up, bmod;
  int32_t OH, OW, sy, sx;
  int32_t ntaps;
  int16_t dy[ALDM_MAX_TAPS];
  int16_t dx[ALDM_MAX_TAPS];
  int32_t N, K, Kpad, bn;    /* bn: N tile (32/64/128); Kpad multiple of 64 */
  int32_t ldo, ld_res, ld_rowvec;
  int32_t OHF, OWF, osy, ooy;
  int32_t act, out_mode, accumulate, splitk, impl;
  int32_t n_split, tok_per_batch, ld_t;
  float alpha;
} aldm_gemm_desc;

int aldm_gemm(const aldm_gemm_desc* d, void* stream);

/* Which tensor-core kernel variant aldm_gemm runs for `d` (host only, no GPU needed; the launch makes the same choice):
 *   out[0] N tile (32 / 64 / 128)          out[1] epilogue body ALDM_EPI_*      out[2] A planes (1 / 2)
 *   out[3] split-K reduction ALDM_RED_*    out[4] store mode ALDM_STORE_*
 * Epilogue bodies: FAST (bias / row vector / residual, fp32 / planes / dual / QKV outputs), GEGLU, GENERIC (everything
 * else, and every split-K GEMM), F32N / PLN (compact bodies: fp32 / plane output with bias and residual only).
 * Reductions: REDUCE4 (coalesced, no activation / alpha / accumulate; fp32, planes or dual out), GENERIC (any epilogue).
 * Store modes: ROW (per-warp rows), COMPACT (swizzled staging tile of the compact bodies), PAIR_* (a warp assembles the
 * two 32-column chunks of a 64-column group into full 128-byte fp16 lines: single-plane PLN output, GEGLU planes output,
 * Q|K columns of a QKV output).
 * Returns ALDM_E_UNSUPPORTED for the SIMT checker (impl = ALDM_GEMM_SIMT) and the aldm_gemm error for a bad descriptor. */
enum { ALDM_EPI_FAST = 0, ALDM_EPI_GEGLU = 1, ALDM_EPI_GENERIC = 2, ALDM_EPI_F32N = 3, ALDM_EPI_PLN = 4 };
enum { ALDM_RED_NONE = 0, ALDM_RED_REDUCE4 = 1, ALDM_RED_GENERIC = 2 };
enum { ALDM_STORE_ROW = 0, ALDM_STORE_COMPACT = 1, ALDM_STORE_PAIR_PLN = 2, ALDM_STORE_PAIR_GEGLU = 3, ALDM_STORE_PAIR_QK = 4 };
int aldm_gemm_variant(const aldm_gemm_desc* d, int32_t out[5]);
/* How the tensor-core kernel loads A for `d` (no CUDA calls): GATHER fetches every (tap, pixel) row of the implicit GEMM
 * separately; HALO loads each 64-channel block of a 3x3, stride-1 convolution's input tile once, with its one-pixel
 * border, and issues all nine taps from that one copy.  HALO is chosen for bn = 64 or 128 (the kernel then runs 64-wide N
 * tiles, which aldm_gemm_variant reports), no GEGLU, no split-K, nine taps within one pixel, sy = sx = 1 (up = 0 or 1),
 * Cp % 64 == 0, and W % 16 == 0 with H % 8 == 0 (8 x 16-pixel tiles) or W == 8 with H % 16 == 0 (16 x 8).
 * ALDM_CONV_HALO=0 in the environment turns it off. */
enum { ALDM_AMODE_GATHER = 0, ALDM_AMODE_HALO = 1 };
int aldm_gemm_a_mode(const aldm_gemm_desc* d, int32_t* mode);

/* ---- operand preparation (normalise / activate / split into bf16 hi+lo planes) ----------- */

enum { ALDM_PREP_COPY = 0, ALDM_PREP_SILU = 1, ALDM_PREP_LRELU = 2,
       ALDM_PREP_GN = 3, ALDM_PREP_GN_SILU = 4, ALDM_PREP_LN = 5 };

/* x = cat(src0[rows,c0], src1[rows,c1]) (fp32) -> f(x) -> planes hi/lo [rows, Cp].
 * GN: rows = B*HW, 32 groups over C = c0+c1, statistics per (b, group), eps as given
 *     (1e-5 UNet ResBlock/out, 1e-6 SpatialTransformer + VAE; SURVEY.md 8a').
 * LN: per-row statistics over C, eps 1e-5.  gamma/beta are [C]. */
typedef struct aldm_prep_desc {
  const float* src0; const float* src1;
  const float* gamma; const float* beta;
  void* out_hi; void* out_lo;
  double* scratch;           /* GN: B*(64*32*2*8 + 32*2*4 + 4) bytes: per-block double partials, (mean, rstd) floats, ticket
                                counters; must be ZERO before the first GroupNorm that uses it (the tickets reset themselves) */
  int32_t rows, c0, c1, Cp;
  int32_t B, HW, groups;
  int32_t mode;
  float eps, slope;
  int32_t src_nchw;          /* src0 is [B, C, HW] (NCHW) instead of [B*HW, C] */
} aldm_prep_desc;

int aldm_prep(const aldm_prep_desc* d, void* stream);

/* fp32 matrix -> weight tile images on the device (dynamic B operands: VAE attention K, V^T).
 * src is [N, K] with row stride lds (transpose=0) or [K, N] (transpose=1). */
int aldm_pack_b(const float* src, int32_t lds, int32_t transpose, int32_t N, int32_t K,
                int32_t bn, void* dst_packed, float* dst_plain, void* stream);

/* ---- attention --------------------------------------------------------------------------- */

/* softmax(scale * Q K^T + mask) V per (batch, head), head_dim = 32 (SURVEY.md 8a row A8).
 * All operands are bf16 hi/lo planes written by the projection GEMMs (ALDM_OUT_QKV / ALDM_OUT_PLANES):
 *   Q : [B*Nq, ldq], head h at columns [q_col + h*32, +32)
 *   K : [Bkv*Nk, ldk], head h at columns [k_col + h*32, +32)
 *   Vt: [(bkv*heads*32 + h*32 + d), ld_t] keys contiguous (V transposed), ld_t >= Nk, ld_t % 8 == 0
 * kv batch index bkv = b % kv_bmod (0: bkv = b).  mask: [Bkv, Nk] floats (1 = keep) or NULL; entries != 1
 * are filled with -FLT_MAX before the softmax exactly like attention.py:356-360.
 * Output: operand planes [B*Nq, ldo], head h at columns [h*32, +32).
 * impl: ALDM_GEMM_TC = wgmma flash kernel, ALDM_GEMM_SIMT = CUDA-core checker. */
typedef struct aldm_attn_desc {
  const void* q_hi; const void* q_lo; const void* k_hi; const void* k_lo; const void* vt_hi; const void* vt_lo;
  const float* mask;
  void* out_hi; void* out_lo;
  int32_t B, heads, Nq, Nk, ldq, ldk, ld_t, ldo, q_col, k_col, kv_bmod, impl;
  float scale;
} aldm_attn_desc;

int aldm_attention(const aldm_attn_desc* d, void* stream);

/* row softmax in place: x[rows, n] (VAE AttnBlock, model.py:216-217), then split to planes */
int aldm_softmax_rows(const float* x, int32_t rows, int32_t n, float scale, void* out_hi, void* out_lo,
                      void* stream);

/* ---- small fused elementwise kernels ------------------------------------------------------ */

/* timestep_embedding (util.py:172-196): t[B] int64 -> planes [B, dim] (cos | sin);
 * freqs[dim/2] = exp(-ln(max_period)*i/(dim/2)) is tabulated by the host (util.py:183-187) */
int aldm_timestep_embedding(const int64_t* t, int32_t B, int32_t dim, const float* freqs,
                            void* out_hi, void* out_lo, void* stream);

/* K6: CFG combine + DDIM update (+ optional masked blend of the NEXT step's input is done by the
 * caller through `aldm_masked_blend`).  eps holds [2B, ...]: rows [0,B) uncond, [B,2B) cond.
 * x_prev = sqrt(a_prev)*pred_x0 + sqrt(1-a_prev-sigma^2)*e + sigma*noise, all fp32, n elements
 * per batch row; pred_x0 may be NULL. */
int aldm_ddim_step(const float* x, const float* eps_uncond, const float* eps_cond, const float* noise,
                   float* x_prev, float* pred_x0, int64_t n_total,
                   float a_t, float a_prev, float sigma_t, float sqrt_one_minus_at, float guidance,
                   void* stream);

/* PLMS step (plms.py:341-358), sigma = 0 (make_schedule forces eta = 0, plms.py:30): e_t = e_u + guidance*(e_c - e_u);
 * e' from `order`:
 *   1                  e' = e_t                                   (first evaluation of the first step)
 *   2, 3, 4            Adams-Bashforth over e_t and order-1 held values, held1 the most recent:
 *                      (3 e_t - h1) / 2, (23 e_t - 16 h1 + 5 h2) / 12, (55 e_t - 59 h1 + 37 h2 - 9 h3) / 24
 *   ALDM_PLMS_AVERAGE  e' = (held1 + e_t) / 2, held1 = the first evaluation's e_t (second evaluation of the first step)
 * then pred_x0 = (x - sqrt_one_minus_at*e') / sqrt(a_t), x_prev = sqrt(a_prev)*pred_x0 + sqrt(1-a_prev)*e', every
 * operation rounded in the reference's order.  e_t_out (NULL: not stored; must be NULL with ALDM_PLMS_AVERAGE) receives
 * e_t, the value the reference keeps in old_eps.  Unused held pointers may be NULL; pred_x0 may be NULL. */
enum { ALDM_PLMS_AVERAGE = 0 };
int aldm_plms_step(const float* x, const float* eps_uncond, const float* eps_cond, const float* held1,
                   const float* held2, const float* held3, int32_t order, float* e_t_out, float* x_prev,
                   float* pred_x0, int64_t n_total, float a_t, float a_prev, float sqrt_one_minus_at, float guidance,
                   void* stream);

/* DDIMSampler.stochastic_encode (ddim.py:434-449) of style transfer: out = c0*x0' + c1*noise, c0 = sqrt(ddim_alphas)[t],
 * c1 = ddim_sqrt_one_minus_alphas[t] (fp32), the two products and the sum rounded one by one.  x0' = x0, or
 * clip(x0, -10, 10) when clip_flag (a device int32; NULL: no guard) is non-zero: AudioLDM 1's latent guard, decided on
 * the device so that no host synchronisation separates the VAE encoder from the first UNet step.  NaN passes through
 * the clip.  out must not overlap x0, noise or clip_flag. */
int aldm_stochastic_encode(const float* x0, const float* noise, float* out, int64_t n_total, float c0, float c1,
                           const int32_t* clip_flag, void* stream);

/* img = (sqrt_acp*x0 + sqrt_1m_acp*q_noise)*mask + (1-mask)*img; mask is [B,1,T,F] broadcast over C */
int aldm_masked_blend(float* img, const float* x0, const float* mask, const float* q_noise,
                      int32_t B, int32_t C, int32_t TF, float sqrt_acp, float sqrt_1m_acp, void* stream);

/* [B, C, HW] <-> [B, HW, C] fp32 */
int aldm_transpose_chw(const float* src, float* dst, int32_t B, int32_t C, int32_t HW, int32_t to_nhwc,
                       void* stream);

/* out = scale * (mean + exp(0.5*clamp(logvar,-30,20)) * noise)  from NHWC moments [rows, 2*zc]
 * -> NCHW latent [B, zc, HW]   (distributions.py:24-41, ddpm.py:802) */
int aldm_posterior_sample(const float* moments, const float* noise_nchw, float* z_nchw,
                          int32_t B, int32_t zc, int32_t HW, float scale, void* stream);

/* ---- STFT + mel front end (K9) ------------------------------------------------------------ */

/* wav [B, T] fp32 in [-1,1] -> log-mel [B, frames, n_mels] (frames = T/hop + 1), reflect pad n_fft/2,
 * periodic Hann, radix-2 FFT (n_fft power of two <= 2048), magnitude, mel_basis [n_mels, n_fft/2+1]
 * GEMV, log(max(., 1e-5)).  (stft.py:52-81,159-178; audio_processing.py:85-91) */
int aldm_stft_mel(const float* wav, int32_t B, int32_t T, int32_t n_fft, int32_t hop,
                  const float* mel_basis, int32_t n_mels, float* out, int32_t out_frames, void* stream);

/* ---- AudioMAE token generation: GPT-2 with a KV cache (csrc/cond/seqgen.cu) ------------------
 * The sequence of one generator call is [sos0, clap, eos0, sos1, t5[0..L), eos1] (P = L + 5 positions) followed by the
 * generated tokens.  Each GPT-2 layer keeps an fp32 sequence buffer seq[B, lmax, 3C] with one row of q | k | v per
 * position, written in place by the c_attn GEMM through its output row mapping (OHF = lmax, ooy = first position).
 * mask[B, lmax] holds 1 for the positions a query may attend to (the T5 padding holds 0); key 0 must be 1. */

/* Causal attention, head_dim 64, queries at positions [p0, p0 + nq) of every batch row, keys [0, p0 + q] with
 * mask[b, key] == 1; scale applied to q.k; fp32 softmax and accumulation.  Output: planes [B * nq, ldo], head h at
 * columns [h*64, +64) (row b * nq + q).  lmax <= 1024, p0 + nq <= lmax. */
typedef struct aldm_kv_attn_desc {
  const float* seq;          /* [B, lmax, ld_seq]: q at columns [0, C), k at [C, 2C), v at [2C, 3C), C = heads * 64 */
  const float* mask;         /* [B, lmax] */
  void* out_hi; void* out_lo;
  int32_t B, heads, lmax, ld_seq, p0, nq, ldo;
  float scale;
} aldm_kv_attn_desc;
int aldm_kv_attention(const aldm_kv_attn_desc* d, void* stream);

/* Prefill residual stream x[B * P, C], P = L + 5: rows 1 and [4, 4 + L) of every batch row already hold the CLAP and T5
 * projections (written there by their GEMMs); rows 0, 2, 3, L + 4 become sos[0], eos[0], sos[1], eos[1]; then
 * x[b, p] += wpe[p] for every p < P.  mask[B, lmax] = t5_mask at the T5 positions, 1 everywhere else (lmax >= P). */
typedef struct aldm_seq_assemble_desc {
  float* x;
  const float* sos; const float* eos;     /* [>= 2, C] */
  const float* wpe;                       /* [>= P, C] */
  const float* t5_mask;                   /* [B, L] */
  float* mask;                            /* [B, lmax] */
  int32_t B, L, lmax, C;
} aldm_seq_assemble_desc;
int aldm_seq_assemble(const aldm_seq_assemble_desc* d, void* stream);

/* Last position of every batch row (x row b * nq + nq - 1, at sequence position pos): y = ln_f(x) in fp32 (two-pass
 * statistics); out[b, k, :] = y (out is [B, gen_len, C]); next[b, :] = y + wpe[pos + 1] unless next is NULL. */
typedef struct aldm_seq_feedback_desc {
  const float* x;
  const float* gamma; const float* beta;
  const float* wpe;
  float* out;
  float* next;
  int32_t B, nq, C, pos, k, gen_len;
  float eps;
} aldm_seq_feedback_desc;
int aldm_seq_feedback(const aldm_seq_feedback_desc* d, void* stream);

/* ---- Flan-T5 encoder from token ids (csrc/text/t5.cu) ----------------------------------------
 * The residual stream is fp32 [B * L, C]; every projection is a two-plane GEMM.  Sequences hold at most 128 tokens (the
 * tokenizer's max_length), heads of d_kv = 64. */

/* out[r, :] = table[ids[r], :] (shared.weight, fp32, not scaled).  The host checks 0 <= id < vocab; an id outside that
 * range writes a NaN row. */
typedef struct aldm_t5_embed_desc {
  const int64_t* ids;        /* [rows] */
  const float* table;        /* [vocab, C] */
  float* out;                /* [rows, C] */
  int32_t rows, vocab, C;
} aldm_t5_embed_desc;
int aldm_t5_embed(const aldm_t5_embed_desc* d, void* stream);

/* T5LayerNorm: y = gamma * (x * 1 / sqrt(mean(x^2) + eps)) per row of C (C % 128 == 0, <= 2048), fixed-order fp32 sum.
 * Writes operand planes out_hi / out_lo [rows, ldo], or fp32 out_f32 [rows, ldo] when out_f32 is not NULL. */
typedef struct aldm_t5_rmsnorm_desc {
  const float* x;            /* [rows, C] */
  const float* gamma;        /* [C] */
  void* out_hi; void* out_lo;
  float* out_f32;
  int32_t rows, C, ldo;
  float eps;
} aldm_t5_rmsnorm_desc;
int aldm_t5_rmsnorm(const aldm_t5_rmsnorm_desc* d, void* stream);

/* Bidirectional self-attention of B sequences of L <= 128 tokens: s[i, j] = q_i . k_j (no 1/sqrt(d) scaling) +
 * bias[h, j - i + 127]; keys with mask[b, j] != 1 get probability 0 (at least one key per row must be valid); fp32
 * softmax and P V.  qkv [B * L, ld_qkv] holds q | k | v at columns [0, C), [C, 2C), [2C, 3C), head h at [h*64, +64).
 * Output: planes [B * L, ldo].  d_kv != 64 is ALDM_E_UNSUPPORTED; L > 128 or heads * 64 != C is ALDM_E_SHAPE. */
typedef struct aldm_t5_attn_desc {
  const float* qkv;
  const float* bias;         /* [heads, 255]: the relative-position bias for offsets j - i = -127 .. 127 */
  const float* mask;         /* [B, L] */
  void* out_hi; void* out_lo;
  int32_t B, L, heads, d_kv, C, ld_qkv, ldo;
} aldm_t5_attn_desc;
int aldm_t5_attention(const aldm_t5_attn_desc* d, void* stream);

/* Gated-GELU: y[r, c] = gelu_new(x[r, c]) * x[r, F + c] for c < F (x = the fp32 output of the fused [wi_0 | wi_1] GEMM),
 * written as operand planes [rows, ldo].  Elements with |y| > 65504 or non-finite y, which the planes would clamp, are
 * counted into *sat (atomically; the caller zeroes it and reads it back). */
typedef struct aldm_t5_gate_desc {
  const float* x;            /* [rows, ld_x] */
  void* out_hi; void* out_lo;
  uint32_t* sat;
  int32_t rows, F, ld_x, ldo;
} aldm_t5_gate_desc;
int aldm_t5_gate(const aldm_t5_gate_desc* d, void* stream);

/* ---- CLAP text branch from token ids (csrc/clap/clap_text.cu) --------------------------------
 * RoBERTa-base, post-LN: the residual stream is the fp32 output of each LayerNorm, [B * L, C]; every projection is a
 * two-plane GEMM.  Sequences hold at most 512 tokens (the tokenizer's max_length), heads of 64. */

/* out[b * L + t, :] = (word[id] + type[0]) + pos[pid] with HF's position ids, computed from the ids:
 * pid = (number of ids != pad among ids[b, 0..t]) * (id != pad) + pad.  The host checks 0 <= id < vocab; an id outside
 * that range (or a pid >= n_pos) writes a NaN row.  L > 512 is ALDM_E_SHAPE. */
typedef struct aldm_clap_embed_desc {
  const int64_t* ids;        /* [B, L] */
  const float* word;         /* [vocab, C] */
  const float* pos;          /* [n_pos, C] */
  const float* type;         /* [C]: token_type_embeddings row 0 */
  float* out;                /* [B * L, C] */
  int32_t B, L, vocab, n_pos, C, pad;
} aldm_clap_embed_desc;
int aldm_clap_embed(const aldm_clap_embed_desc* d, void* stream);

/* LayerNorm per row of C (C % 128 == 0, <= 1024): two-pass fp32 statistics in a fixed order, y = (x - mean) * rstd *
 * gamma + beta.  Writes BOTH fp32 out_f32 [rows, C] (the post-LN residual stream) and operand planes out_hi / out_lo
 * [rows, ldo] for the next GEMM. */
typedef struct aldm_clap_ln_desc {
  const float* x;            /* [rows, C] */
  const float* gamma;        /* [C] */
  const float* beta;         /* [C] */
  float* out_f32;
  void* out_hi; void* out_lo;
  int32_t rows, C, ldo;
  float eps;
} aldm_clap_ln_desc;
int aldm_clap_layernorm(const aldm_clap_ln_desc* d, void* stream);

/* Bidirectional self-attention of B sequences of L <= 512 tokens: s[i, j] = (q_i . k_j) / 8; keys with mask[b, j] != 1
 * get probability exactly 0 (at least one key per row must be valid); fp32 softmax and P V.  qkv [B * L, ld_qkv] holds
 * q | k | v at columns [0, C), [C, 2C), [2C, 3C), head h at [h*64, +64).  Output: planes [B * L, ldo].  L > 512 or
 * heads * 64 != C is ALDM_E_SHAPE. */
typedef struct aldm_clap_attn_desc {
  const float* qkv;
  const float* mask;         /* [B, L] */
  void* out_hi; void* out_lo;
  int32_t B, L, heads, C, ld_qkv, ldo;
} aldm_clap_attn_desc;
int aldm_clap_attention(const aldm_clap_attn_desc* d, void* stream);

/* erf-GELU: y[r, c] = 0.5 x (1 + erf(x / sqrt(2))) of x = the fp32 output of the intermediate GEMM (bias added), c < F,
 * written as operand planes [rows, ldo]. */
typedef struct aldm_clap_gelu_desc {
  const float* x;            /* [rows, ld_x] */
  void* out_hi; void* out_lo;
  int32_t rows, F, ld_x, ldo;
} aldm_clap_gelu_desc;
int aldm_clap_gelu(const aldm_clap_gelu_desc* d, void* stream);

/* Per batch row b, fp32: p = tanh(Wp x[b * L] + bp) (the pooler, token 0), t = relu(W1 p + b1), y = W2 t + b2,
 * out[b] = y / max(||y||_2, 1e-12).  Weights are stored transposed ([in, out], row-major).  C, P <= 1024. */
typedef struct aldm_clap_head_desc {
  const float* x;            /* [B * L, C]: the last LayerNorm's fp32 output */
  const float* wp_t; const float* bp;     /* [C, C], [C] */
  const float* w1_t; const float* b1;     /* [C, P], [P] */
  const float* w2_t; const float* b2;     /* [P, P], [P] */
  float* out;                /* [B, P] */
  int32_t B, L, C, P;
} aldm_clap_head_desc;
int aldm_clap_head(const aldm_clap_head_desc* d, void* stream);

/* ---- CLAP HTSAT-base audio branch (csrc/audio/htsat.cu) -----------------------------------------
 * Pre-LN Swin transformer over a 64 x 64 patch grid (stages of 64, 32, 16 and 8): the residual stream is fp32 [n * R * R, C]
 * in natural token order (row-major over the grid); every projection is a two-plane GEMM. */

/* Log-mel front end, one frame per CTA: the 48 kHz signal (up = 1: wav itself; up = 3: torchaudio's 16 -> 48 kHz resample
 * with taps [3][15], sample 3q + j = sum_m taps[j][m] wav[q + m - 7], zeros outside), truncated to L48 = min(up L, 480000)
 * samples, reflect-centred frames of 1024 every 480 (T = L48 / 480 + 1), periodic Hann, power spectrum, power @ melW
 * [513, 64], 10 log10(max(., 1e-10)), then BatchNorm with running statistics.  L48 <= 512 (no reflect padding) is
 * ALDM_E_SHAPE; up other than 1 or 3 is ALDM_E_UNSUPPORTED. */
typedef struct aldm_htsat_logmel_desc {
  const float* wav;          /* [n, L] */
  const float* taps;         /* [3, 15] (up = 3), else unused */
  const float* melW;         /* [513, 64] */
  const float* bn_mean; const float* bn_var; const float* bn_w; const float* bn_b;   /* [64] */
  float* out;                /* [n, T, 64] */
  int32_t n, L, up, L48, T;
  float eps;
} aldm_htsat_logmel_desc;
int aldm_htsat_logmel(const aldm_htsat_logmel_desc* d, void* stream);

/* reshape_wav2img + patch embedding: bicubic (align_corners, A = -0.75) interpolation of the T frames to 1024, the fold
 * image[chunk * 64 + mel, t - 256 chunk], Conv2d(1, 128, 4, stride 4) with bias (w [128, 16] in (dy, dx) order) and
 * LayerNorm(128).  out: the fp32 residual stream [n * 4096, 128].  2 <= T <= 1024. */
typedef struct aldm_htsat_patch_desc {
  const float* mel;          /* [n, T, 64] */
  const float* w; const float* bias;      /* [128, 16], [128] */
  const float* gamma; const float* beta;  /* [128] */
  float* out;
  int32_t n, T;
  float eps;
} aldm_htsat_patch_desc;
int aldm_htsat_patch(const aldm_htsat_patch_desc* d, void* stream);

/* (Shifted) window attention over 8 x 8 windows of an R x R grid rolled by -shift: s = (scale q) . k + bias[h, i, j]
 * (+ mask[w, i, j] when shift > 0), fp32 softmax and P V.  qkv [n * R * R, ld_qkv] holds q | k | v at columns [0, C),
 * [C, 2C), [2C, 3C) in natural token order; the output planes [n * R * R, ldo] are written at the same (un-rolled) tokens.
 * head_dim other than 32 is ALDM_E_UNSUPPORTED; R not a multiple of 8, or shift > 0 without a mask, is ALDM_E_SHAPE. */
typedef struct aldm_htsat_attn_desc {
  const float* qkv;
  const float* bias;         /* [heads, 64, 64] */
  const float* mask;         /* [(R / 8)^2, 64, 64] (0 / -100), or null when shift = 0 */
  void* out_hi; void* out_lo;
  int32_t n, R, shift, heads, head_dim, C, ld_qkv, ldo;
  float scale;
} aldm_htsat_attn_desc;
int aldm_htsat_window_attention(const aldm_htsat_attn_desc* d, void* stream);

/* PatchMerging's gather and norm: row (a, b) of the R/2 x R/2 grid is cat(x(2a, 2b), x(2a+1, 2b), x(2a, 2b+1),
 * x(2a+1, 2b+1)) [4C], LayerNorm(4C) -> operand planes [n * (R/2)^2, ldo].  C is 128, 256 or 512. */
typedef struct aldm_htsat_merge_desc {
  const float* x;            /* [n * R * R, C] */
  const float* gamma; const float* beta;  /* [4C] */
  void* out_hi; void* out_lo;
  int32_t n, R, C, ldo;
  float eps;
} aldm_htsat_merge_desc;
int aldm_htsat_merge(const aldm_htsat_merge_desc* d, void* stream);

/* Per clip, fp32: m = mean over the ntok tokens of LayerNorm(x), t = relu(W1 m + b1), y = W2 t + b2,
 * out = y / max(||y||_2, 1e-12).  Weights transposed ([in, out]).  C, P <= 1024. */
typedef struct aldm_htsat_head_desc {
  const float* x;            /* [n * ntok, C] */
  const float* gamma; const float* beta;  /* [C] */
  const float* w1_t; const float* b1;     /* [C, P], [P] */
  const float* w2_t; const float* b2;     /* [P, P], [P] */
  float* out;                /* [n, P] */
  int32_t n, ntok, C, P;
  float eps;
} aldm_htsat_head_desc;
int aldm_htsat_head(const aldm_htsat_head_desc* d, void* stream);

/* ---- programs: flat op tables replayed on a stream / as a CUDA graph ---------------------- */

enum { ALDM_OP_GEMM = 1, ALDM_OP_PREP = 2, ALDM_OP_ATTN = 3, ALDM_OP_SOFTMAX = 4, ALDM_OP_TEMB = 5,
       ALDM_OP_TRANSPOSE = 6, ALDM_OP_PACKB = 7, ALDM_OP_COPY = 8, ALDM_OP_SEQ_ASSEMBLE = 9, ALDM_OP_KV_ATTN = 10,
       ALDM_OP_SEQ_FEEDBACK = 11, ALDM_OP_T5_EMBED = 12, ALDM_OP_T5_RMSNORM = 13, ALDM_OP_T5_ATTN = 14,
       ALDM_OP_T5_GATE = 15, ALDM_OP_CLAP_EMBED = 16, ALDM_OP_CLAP_LN = 17, ALDM_OP_CLAP_ATTN = 18,
       ALDM_OP_CLAP_GELU = 19, ALDM_OP_CLAP_HEAD = 20, ALDM_OP_HTSAT_LOGMEL = 21, ALDM_OP_HTSAT_PATCH = 22,
       ALDM_OP_HTSAT_ATTN = 23, ALDM_OP_HTSAT_MERGE = 24, ALDM_OP_HTSAT_HEAD = 25 };

typedef struct aldm_op {
  int32_t kind;
  int32_t tag;               /* free for the host (layer index, for profiling) */
  union {
    aldm_gemm_desc gemm;
    aldm_prep_desc prep;
    aldm_attn_desc attn;
    struct { const float* x; void* out_hi; void* out_lo; int32_t rows, n; float scale; } softmax;
    struct { const int64_t* t; const float* freqs; void* out_hi; void* out_lo; int32_t B, dim; } temb;
    struct { const float* src; float* dst; int32_t B, C, HW, to_nhwc; } transpose;
    struct { const float* src; void* dst_packed; float* dst_plain; int32_t lds, transpose, N, K, bn; } packb;
    struct { const void* src; void* dst; int64_t bytes; } copy;
    aldm_seq_assemble_desc seq_assemble;
    aldm_kv_attn_desc kv_attn;
    aldm_seq_feedback_desc seq_feedback;
    aldm_t5_embed_desc t5_embed;
    aldm_t5_rmsnorm_desc t5_rmsnorm;
    aldm_t5_attn_desc t5_attn;
    aldm_t5_gate_desc t5_gate;
    aldm_clap_embed_desc clap_embed;
    aldm_clap_ln_desc clap_ln;
    aldm_clap_attn_desc clap_attn;
    aldm_clap_gelu_desc clap_gelu;
    aldm_clap_head_desc clap_head;
    aldm_htsat_logmel_desc htsat_logmel;
    aldm_htsat_patch_desc htsat_patch;
    aldm_htsat_attn_desc htsat_attn;
    aldm_htsat_merge_desc htsat_merge;
    aldm_htsat_head_desc htsat_head;
  } u;
} aldm_op;

typedef struct aldm_program aldm_program;

int aldm_program_create(const aldm_op* ops, int32_t n_ops, aldm_program** out);
int aldm_program_run(aldm_program* p, void* stream);            /* plain launches */
int aldm_program_run_range(aldm_program* p, int32_t first, int32_t last, void* stream);
int aldm_program_capture(aldm_program* p, void* stream);        /* build + instantiate a CUDA graph */
int aldm_program_replay(aldm_program* p, void* stream);         /* cudaGraphLaunch */
int aldm_program_is_captured(aldm_program* p);                  /* 1 once aldm_program_capture succeeded */
int aldm_program_num_launches(aldm_program* p);                 /* kernels launched per run */
void aldm_program_destroy(aldm_program* p);

/* ---- engine: the reference's seams as single calls (SURVEY.md 8b) --------------------------
 * An engine ties the programs of one model instance to their fixed I/O slots (device addresses inside the
 * workspace the programs were resolved against) so that a caller who is not the Python host -- or the Python
 * host itself -- drives the hot path with the calls the reference makes:
 *   aldm_engine_set_conditioning  <- DiffusionWrapper.forward's cond-dict unpacking (ddpm.py:1821-1879), once per call
 *   aldm_engine_unet_eps          <- the two self.model.apply_model(x, t, c) calls of p_sample_ddim (ddim.py:293-296)
 *   aldm_engine_ddim_step         <- DDIMSampler.p_sample_ddim as a whole (ddim.py:265-355): UNet x2 + CFG + update
 *   aldm_engine_plms_step         <- one get_model_output + get_x_prev_and_pred_x0 of PLMSSampler.p_sample_plms
 *                                    (plms.py:281-358): UNet x2 + CFG + e' + update; the first step is two calls
 *   aldm_engine_vae_decode        <- LatentDiffusion.decode_first_stage (ddpm.py:922-926)
 *   aldm_engine_vocoder           <- first_stage_model.vocoder(mel) in mel_spectrogram_to_waveform (ddpm.py:928-939)
 *   aldm_engine_vae_encode        <- encode_first_stage (ddpm.py:941-943), moments out
 * The engine borrows the programs (it never destroys them) and owns its descriptor copy plus the step graph
 * (all lanes as parallel branches) and the side streams / events used to capture it.  All
 * pointers are device pointers, fp32 contiguous NCHW as in the reference; everything is enqueued on `stream`;
 * nothing synchronises.  Single caller thread per engine. */
typedef struct aldm_engine aldm_engine;

#define ALDM_MAX_LANES 8

/* One UNet lane: an independent copy of the step / conditioning programs planned for B / n_lanes latent rows, with
 * its own workspace (the weight arena is shared).  Lanes are replayed as PARALLEL branches of one CUDA graph: the
 * UNet's deep levels are chains of short kernels that each fill a fraction of the SMs, so independent
 * sub-batches overlap there while the large layers simply share the machine.  Samples are independent through the
 * whole path (SURVEY.md 8e), so results do not depend on the lane count (up to split-K / tile-shape choices). */
typedef struct aldm_unet_lane {
  aldm_program* cond;           /* cross-attention K/V precompute (may be NULL: no cross-attention) */
  aldm_program* step;           /* one UNet evaluation of 2*Bl rows: rows [0,Bl) unconditional, [Bl,2Bl) conditional */
  float* x_slot;                /* [Bl, C, T, F] latent read by `step` */
  int64_t* t_slot;              /* [2Bl] DDPM timestep */
  float* eps_slot;              /* [2Bl, C, T, F] */
  float* ctx_slot[2];           /* [2Bl, ctx_len[i], ctx_dim[i]] zero-padded context i */
  float* mask_slot[2];          /* [2Bl, ctx_len[i]] 1 = attend */
  float* film_slot;             /* [2Bl, film_dim] or NULL */
} aldm_unet_lane;

typedef struct aldm_engine_desc {
  aldm_unet_lane lane[ALDM_MAX_LANES];   /* lane l owns latent rows [l*B/n_lanes, (l+1)*B/n_lanes) */
  int32_t n_lanes;              /* 1..ALDM_MAX_LANES, B % n_lanes == 0 */
  aldm_program* vae_dec;        /* may be NULL */
  aldm_program* vocoder;        /* may be NULL */
  aldm_program* vae_enc;        /* may be NULL */
  float* z_slot;                /* vae_dec input [B, C, T, F] */
  float* mel_slot;              /* vae_dec output [B, 1, T', F'] */
  float* voc_mel_slot;          /* vocoder input [B, T', F'] */
  float* wave_slot;             /* vocoder output [B, 1, L] */
  float* enc_mel_slot;          /* vae_enc input [B, 1, T', F'] */
  float* moments_slot;          /* vae_enc output [B, T, F, 2C] (channels-last) */
  int32_t B;                    /* latent batch the programs were planned for (all lanes together) */
  int32_t latent_elems;         /* C*T*F */
  int32_t mel_elems;            /* T'*F' */
  int32_t wave_len;             /* L */
  int32_t n_ctx;                /* 0..2 */
  int32_t ctx_len[2];
  int32_t ctx_dim[2];
  int32_t film_dim;
  int32_t use_graph;            /* 1: the lanes' step programs are captured into one graph on first use and replayed */
} aldm_engine_desc;

int aldm_engine_create(const aldm_engine_desc* d, aldm_engine** out);
void aldm_engine_destroy(aldm_engine* e);
/* which: 0 = unconditional half, 1 = conditional half.  ctx_i [B, len_i, ctx_dim[i]], mask_i [B, len_i] (fp32 0/1),
 * len_i <= ctx_len[i]; film_y [B, film_dim] or NULL.  Call for both halves, then aldm_engine_precompute once. */
int aldm_engine_set_conditioning(aldm_engine* e, int32_t which, const float* ctx0, const float* mask0, int32_t len0,
                                 const float* ctx1, const float* mask1, int32_t len1, const float* film_y, void* stream);
int aldm_engine_precompute(aldm_engine* e, void* stream);
int aldm_engine_unet_eps(aldm_engine* e, const float* x, int64_t t, float* eps_uncond, float* eps_cond, void* stream);
/* x_prev (and pred_x0 unless NULL) [B, C, T, F]; scalars as in aldm_ddim_step */
int aldm_engine_ddim_step(aldm_engine* e, const float* x, int64_t t, const float* noise, float a_t, float a_prev,
                          float sigma_t, float sqrt_one_minus_at, float guidance, float* x_prev, float* pred_x0,
                          void* stream);
/* UNet pair on x_in at t, then aldm_plms_step per lane with x = x_base (x_in itself except for the first step's
 * second evaluation, whose update starts again from that step's input).  held*, e_t_out, x_prev, pred_x0: [B, C, T, F]
 * caller buffers (the e_t history ring is the caller's); x_prev may alias x_in but not x_base. */
int aldm_engine_plms_step(aldm_engine* e, const float* x_in, int64_t t, const float* x_base, const float* held1,
                          const float* held2, const float* held3, int32_t order, float* e_t_out, float a_t,
                          float a_prev, float sqrt_one_minus_at, float guidance, float* x_prev, float* pred_x0,
                          void* stream);
int aldm_engine_vae_decode(aldm_engine* e, const float* z, float* mel, void* stream);
int aldm_engine_vocoder(aldm_engine* e, const float* mel, float* wave, void* stream);
int aldm_engine_vae_encode(aldm_engine* e, const float* mel, float* moments, void* stream);

/* ---- misc ---------------------------------------------------------------------------------- */

int aldm_abi_version(void);
size_t aldm_sizeof_op(void);
size_t aldm_sizeof_gemm_desc(void);
size_t aldm_sizeof_engine_desc(void);
size_t aldm_offsetof_gemm(int32_t field);     /* 0:B 1:ntaps 2:dy 3:N 4:ldo 5:act 6:alpha 7:n_split (layout self-check) */
const char* aldm_last_error(void);
int aldm_device_check(int32_t device);   /* 0 if `device` is sm_90 and kernels can load */
int aldm_debug_timeline(long long* host_out, int32_t n);   /* profiling aid: per-stage clock64 stamps of CTA 0 (scripts/prof_ops.py --timeline) */
int aldm_debug_store_rate(int32_t n_cta, int32_t iters, int32_t mode, long long region_bytes, long long* host_out);   /* profiling aid: SM -> L2 store throughput, STG.128 (0) vs TMA bulk store (1) (scripts/store_rate.py) */

#ifdef __cplusplus
}
#endif
#endif /* ALDM_B200_H_ */
