// K1/K2/K7/K8: implicit-GEMM convolution / linear layer on Hopper tensor cores (wgmma).
//
//   out[row(m), n] = epilogue( sum_k A[m,k] * W[n,k] )        (aldm_gemm_desc, include/aldm_b200.h)
//
// Precision: split-fp16 operands, fp32 accumulation in registers.  Weights are packed as two fp16 planes (w ~= hi + lo,
// 22 significand bits).  Activations arrive as fp16 planes written by the prep kernels / producer epilogues:
//   * two planes (a_lo != NULL): the products hi*hi + hi*lo_w + lo*hi_w, ~2^-22 operand precision, three wgmma per
//     K step -- the convolutions, where the 200-step waveform budget goes (DESIGN.md section 3, scripts/precision_study.py);
//   * one plane (a_lo == NULL): two wgmma (hi*lo_w, hi*hi_w) and half the A bytes -- the token-side linear layers.
// (SURVEY.md 7 H1: plain single-pass bf16 / TF32-class rounding of BOTH operands misses or crowds the 1e-3 waveform
// tolerance; rounding only the activations to 11 bits costs 2e-4 at 200 steps.)
//
// Structure of one CTA (persistent: 512 threads = four warpgroups, one CTA per SM looping over 128 x BN output tiles /
// split-K slices):
//   warps 0-7   two consumer warpgroups: wgmma on 64-row halves of the tile, then the accumulator is handed to the
//               epilogue warpgroup as an fp32 tile in shared memory and the consumers go on to the next tile.
//   warps 8-11  producers: gather A in 16-byte chunks (8 channels of one tap of one pixel) with cp.async + zero fill into
//               128B-swizzled K-major tiles; completion is signalled on the stage's mbarrier (cp.async.mbarrier.arrive).
//               One ELECTED lane (elect.sync) of warp 8 also issues a TMA bulk copy (cp.async.bulk) of the host-packed,
//               pre-swizzled weight tile image (hi|lo) per stage.
//   warps 12-15 epilogue warpgroup: warp w finishes rows [32 w, 32 w + 32) of the tile, all BN columns, while the
//               consumers already run the next tile's MMAs.
// Halo A path (HALO = 1, aldm_gemm_a_mode): for a 3x3, stride-1 convolution (nearest x2 upsample folded in or not) an M
// tile is an 8 x 16 or 16 x 8 pixel block.
// Warps 8-10 copy its 180-pixel input halo once per 64-channel block into a slab (cp.async, zero fill = the padding), one
// lane of warp 11 streams one tap's weight tile per stage, and the consumers issue the nine taps from the slab through
// shifted descriptors: the A bytes per tile drop from 9 x 128 to 180 pixel rows.  The K loop runs (channel block, tap).
#include <stdlib.h>

#include "common.cuh"

namespace aldm {

// ------------------------------------------------------------------------------------------
// row decoding + epilogue shared by the tensor-core kernel, the SIMT checker and split-K
// ------------------------------------------------------------------------------------------
struct RowInfo {
  int m, b, oh, ow;
  bool valid;
  long long orow;
};

__device__ __forceinline__ RowInfo decode_row(const aldm_gemm_desc& d, int m, int M) {
  RowInfo r;
  r.m = m;
  r.valid = m < M;
  int mm = r.valid ? m : 0;
  r.ow = mm % d.OW;
  int t = mm / d.OW;
  r.oh = t % d.OH;
  r.b = t / d.OH;
  r.orow = ((long long)r.b * d.OHF + (long long)r.oh * d.osy + d.ooy) * d.OWF + r.ow;
  return r;
}

// v[0..cnt) are post-activation values for output columns [n0, n0+cnt) of row r.
__device__ __forceinline__ void epi_finish(const aldm_gemm_desc& d, const RowInfo& r, int n0, int cnt, float* v,
                                           int n_out) {
  if (!r.valid) return;
  if (n0 >= n_out) return;
  if (n0 + cnt > n_out) cnt = n_out - n0;
  if (d.res) {
    const float* rp = d.res + r.orow * d.ld_res + n0;
    for (int i = 0; i < cnt; ++i) v[i] += __ldg(rp + i);
  }
  if (d.alpha != 1.0f)
    for (int i = 0; i < cnt; ++i) v[i] *= d.alpha;
  if (d.out_mode == ALDM_OUT_F32) {
    float* op = d.out + r.orow * d.ldo + n0;
    if (d.accumulate)
      for (int i = 0; i < cnt; ++i) v[i] += op[i];
    if (cnt == 32 && ((reinterpret_cast<uintptr_t>(op) & 15u) == 0)) {
#pragma unroll
      for (int i = 0; i < 32; i += 4) *reinterpret_cast<float4*>(op + i) = make_float4(v[i], v[i + 1], v[i + 2], v[i + 3]);
    } else {
      for (int i = 0; i < cnt; ++i) op[i] = v[i];
    }
    if (d.out_hi) {   // dual output: the same values also as operand planes for the next GEMM
      aldm_plane_t* hp = reinterpret_cast<aldm_plane_t*>(d.out_hi) + r.orow * d.ldo + n0;
      aldm_plane_t* lp = d.out_lo ? reinterpret_cast<aldm_plane_t*>(d.out_lo) + r.orow * d.ldo + n0 : nullptr;
      for (int i = 0; i < cnt; ++i) store_split1(hp, lp, i, v[i]);
    }
  } else if (d.out_mode == ALDM_OUT_QKV && n0 >= d.n_split) {
    // V projection: transposed planes [(b*Cv + c), ld_t] with the token index contiguous
    const int b = r.m / d.tok_per_batch, tok = r.m - b * d.tok_per_batch;
    const long long base = ((long long)b * (d.N - d.n_split) + (n0 - d.n_split)) * d.ld_t + tok;
    aldm_plane_t* hp = reinterpret_cast<aldm_plane_t*>(d.out2_hi) + base;
    aldm_plane_t* lp = d.out2_lo ? reinterpret_cast<aldm_plane_t*>(d.out2_lo) + base : nullptr;
    for (int i = 0; i < cnt; ++i) store_split1(hp, lp, (long long)i * d.ld_t, v[i]);
    // keys in [tok_per_batch, ld_t) are padding the attention kernel multiplies by P = 0: they must
    // be finite (stale workspace bytes reinterpreted as fp16 could be NaN), so the last token zeroes them
    if (tok == d.tok_per_batch - 1) {
      for (int t = 1; tok + t < d.ld_t; ++t)
        for (int i = 0; i < cnt; ++i) store_split1(hp, lp, (long long)i * d.ld_t + t, 0.f);
    }
  } else if (d.out_mode == ALDM_OUT_PLANES || d.out_mode == ALDM_OUT_QKV) {
    aldm_plane_t* hp = reinterpret_cast<aldm_plane_t*>(d.out_hi) + r.orow * d.ldo + n0;
    aldm_plane_t* lp = d.out_lo ? reinterpret_cast<aldm_plane_t*>(d.out_lo) + r.orow * d.ldo + n0 : nullptr;
    if (cnt == 32 && ((reinterpret_cast<uintptr_t>(hp) & 15u) == 0)) {
#pragma unroll
      for (int i = 0; i < 32; i += 8) {
        uint4 h, l;
        split8(v + i, h, l);
        *reinterpret_cast<uint4*>(hp + i) = h;
        if (lp) *reinterpret_cast<uint4*>(lp + i) = l;
      }
    } else {
      for (int i = 0; i < cnt; ++i) store_split1(hp, lp, i, v[i]);
    }
  } else {  // NCHW
    for (int i = 0; i < cnt; ++i)
      d.out[(((long long)r.b * d.N + (n0 + i)) * d.OH + r.oh) * d.OW + r.ow] = v[i];
  }
}

// Bias / rowvec / activation for one 32-column chunk whose packed column base is pc0.
// For GEGLU `g` holds the gate chunk (packed columns pc0 + bn/2 ...).
__device__ __forceinline__ void add_vec32(float* v, const float* __restrict__ p) {
  if ((reinterpret_cast<uintptr_t>(p) & 15u) == 0) {
#pragma unroll
    for (int i = 0; i < 32; i += 4) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(p + i));
      v[i] += t.x; v[i + 1] += t.y; v[i + 2] += t.z; v[i + 3] += t.w;
    }
  } else {
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] += __ldg(p + i);
  }
}

__device__ __forceinline__ void epi_activate(const aldm_gemm_desc& d, const RowInfo& r, int pc0, float* v, float* g) {
  if (d.bias) {
    add_vec32(v, d.bias + pc0);
    if (d.act == ALDM_ACT_GEGLU) add_vec32(g, d.bias + pc0 + d.bn / 2);
  }
  if (d.rowvec) add_vec32(v, d.rowvec + (long long)r.b * d.ld_rowvec + pc0);
  if (d.act == ALDM_ACT_GEGLU) {
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] *= gelu_f(g[i]);
  } else if (d.act == ALDM_ACT_TANH) {
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = tanhf(v[i]);
  } else if (d.act == ALDM_ACT_SILU) {
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = silu_f(v[i]);
  } else if (d.act == ALDM_ACT_GELU_TANH) {
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = gelu_tanh_f(v[i]);
  }
}

// Coalesced finish: the 32x32 chunk (lane == row) is transposed through a per-warp shared-memory
// staging tile (stride 33: conflict-free both ways) so that 8 lanes cover one 128-byte output row
// segment: residual loads and output stores are full-line float4 transactions instead of 32
// scattered 16-byte pieces.  Handles fp32 and operand-plane outputs; returns false if the layout
// does not allow it (caller falls back to the row-owner path).
__device__ __forceinline__ bool epi_coalescable(const aldm_gemm_desc& d, int n_out) {
  if (n_out % 4 != 0 || d.ldo % 4 != 0) return false;
  if (d.res && d.ld_res % 4 != 0) return false;
  return d.out_mode == ALDM_OUT_F32 || d.out_mode == ALDM_OUT_PLANES || d.out_mode == ALDM_OUT_QKV;
}

// Per-tile row bookkeeping of the coalesced path: lane (rs = lane>>3, c4 = (lane&7)*4) handles rows
// it*4+rs, it = 0..7; orow[it] / valid bits are fetched once per tile from the row-owner lanes.
struct CoRows {
  long long orow[8];
  unsigned vmask;
};

__device__ __forceinline__ CoRows co_rows(const RowInfo& r, int lane) {
  CoRows cr;
  cr.vmask = __ballot_sync(0xffffffffu, r.valid);
  const int rs = lane >> 3;
#pragma unroll
  for (int it = 0; it < 8; ++it) cr.orow[it] = __shfl_sync(0xffffffffu, r.orow, it * 4 + rs);
  return cr;
}

// issue the residual loads of one 32-column chunk (they are consumed after the accumulator read + transpose,
// and the next chunk's loads are issued before the current chunk is processed: latency hidden)
__device__ __forceinline__ void co_load_res(const aldm_gemm_desc& d, const CoRows& cr, int n0, int n_out, int lane, float4 (&rv)[8]) {
  const int rs = lane >> 3, n = n0 + (lane & 7) * 4;
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const bool ok = ((cr.vmask >> (it * 4 + rs)) & 1u) && n < n_out;
    rv[it] = ok ? __ldg(reinterpret_cast<const float4*>(d.res + cr.orow[it] * d.ld_res + n)) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

__device__ __forceinline__ void epi_finish_coalesced(const aldm_gemm_desc& d, const CoRows& cr, int n0, const float* v,
                                                     int n_out, float* stg, int lane, const float4 (&rv)[8], bool has_rv) {
#pragma unroll
  for (int i = 0; i < 32; ++i) stg[lane * 33 + i] = v[i];
  __syncwarp();
  const int rs = lane >> 3, c4 = (lane & 7) * 4;
  const int n = n0 + c4;
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int rr = it * 4 + rs;
    if (!((cr.vmask >> rr) & 1u) || n >= n_out) continue;
    const long long orow = cr.orow[it];
    float x[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) x[i] = stg[rr * 33 + c4 + i];
    if (has_rv) { x[0] += rv[it].x; x[1] += rv[it].y; x[2] += rv[it].z; x[3] += rv[it].w; }
    if (d.alpha != 1.0f) {
#pragma unroll
      for (int i = 0; i < 4; ++i) x[i] *= d.alpha;
    }
    if (d.out_mode == ALDM_OUT_F32) {
      float4* op = reinterpret_cast<float4*>(d.out + orow * d.ldo + n);
      if (d.accumulate) {
        const float4 t = *op;
        x[0] += t.x; x[1] += t.y; x[2] += t.z; x[3] += t.w;
      }
      *op = make_float4(x[0], x[1], x[2], x[3]);
    }
    if (d.out_mode != ALDM_OUT_F32 || d.out_hi) {
      uint2 h, l;
      split2(x[0], x[1], h.x, l.x);
      split2(x[2], x[3], h.y, l.y);
      *reinterpret_cast<uint2*>(reinterpret_cast<aldm_plane_t*>(d.out_hi) + orow * d.ldo + n) = h;
      if (d.out_lo) *reinterpret_cast<uint2*>(reinterpret_cast<aldm_plane_t*>(d.out_lo) + orow * d.ldo + n) = l;
    }
  }
  __syncwarp();
}

// ---- compact coalesced finish (EPI_F32N / EPI_PLN / EPI_GEGLU) -----------------------------------
// Same idea as above with a quarter of the instructions: the staging tile is 32 rows x 128 bytes with the
// 16-byte chunk index XOR-swizzled by (row & 7), so both the row-owner writes and the transposed reads are
// conflict-free 128-bit accesses (8 STS.128 + 8 LDS.128 per lane instead of 32 + 32 scalar ones); bias is
// added after the transpose (one float4 per lane and chunk, fetched before the accumulator is ready), the
// output mode is a template parameter, and alpha / accumulate / rowvec are not supported (host-checked).
struct CoRows32 {       // host guarantees rows * max(ldo, ld_res) < 2^31 on this path
  int orow[8];
  unsigned vmask;
};

__device__ __forceinline__ CoRows32 co_rows32(const RowInfo& r, int lane) {
  CoRows32 cr;
  cr.vmask = __ballot_sync(0xffffffffu, r.valid);
  const int rs = lane >> 3;
  const int o = (int)r.orow;
#pragma unroll
  for (int it = 0; it < 8; ++it) cr.orow[it] = __shfl_sync(0xffffffffu, o, it * 4 + rs);
  return cr;
}

__device__ __forceinline__ void co_load_res32(const aldm_gemm_desc& d, const CoRows32& cr, int n0, int n_out, int lane, float4 (&rv)[8]) {
  const int rs = lane >> 3, n = n0 + (lane & 7) * 4;
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const bool ok = ((cr.vmask >> (it * 4 + rs)) & 1u) && n < n_out;
    rv[it] = ok ? __ldg(reinterpret_cast<const float4*>(d.res + (cr.orow[it] * d.ld_res + n))) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

__device__ __forceinline__ void stage_rows(uint8_t* stg, int lane, const float* v) {
  uint8_t* wr = stg + lane * 128;
  const int sw = lane & 7;
#pragma unroll
  for (int j = 0; j < 8; ++j)
    *reinterpret_cast<float4*>(wr + ((j ^ sw) << 4)) = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
  __syncwarp();
}

template <bool PLANES_ONLY, typename CR>
__device__ __forceinline__ void emit_rows(const aldm_gemm_desc& d, const CR& cr, int n0, int n_out, const uint8_t* stg,
                                          int lane, const float4 (&rv)[8], bool has_rv, float4 b4) {
  const int rs = lane >> 3, c8 = lane & 7;
  const int n = n0 + c8 * 4;
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int rr = it * 4 + rs;
    float4 x = *reinterpret_cast<const float4*>(stg + rr * 128 + ((c8 ^ (rr & 7)) << 4));
    if (!((cr.vmask >> rr) & 1u) || n >= n_out) continue;
    x.x += b4.x; x.y += b4.y; x.z += b4.z; x.w += b4.w;
    if (has_rv) { x.x += rv[it].x; x.y += rv[it].y; x.z += rv[it].z; x.w += rv[it].w; }
    const auto o = cr.orow[it] * d.ldo + n;      // 32-bit on the compact path, 64-bit for GEGLU (CoRows)
    if (!PLANES_ONLY) *reinterpret_cast<float4*>(d.out + o) = x;
    if (PLANES_ONLY || d.out_hi) {
      uint2 h, l;
      split2(x.x, x.y, h.x, l.x);
      split2(x.z, x.w, h.y, l.y);
      *reinterpret_cast<uint2*>(reinterpret_cast<aldm_plane_t*>(d.out_hi) + o) = h;
      if (d.out_lo) *reinterpret_cast<uint2*>(reinterpret_cast<aldm_plane_t*>(d.out_lo) + o) = l;
    }
  }
  __syncwarp();
}

// ---- full-line finish for single-plane fp16 outputs (EPI_PLN, EPI_GEGLU -> planes, Q|K planes) --------------------------
// A 32 x 32 chunk is only 64 bytes per row in fp16: stored by itself it is a stream of half-line transactions, and the
// SM's store port moves one transaction per clock whatever its size (scripts/store_rate.py measures it), so half-line
// stores halve the store bandwidth of the epilogue.  The warp therefore packs the two 32-column chunks of one 64-column
// group (part 0 / 1) into its staging tile (rows of 128 bytes, 16-byte chunks XOR-swizzled by the row) and then stores the
// 32 x 64 fp16 block as 32 complete 128-byte rows: 8 STG.128 per block instead of 16 STG.64.
__device__ __forceinline__ void line_put_hi(uint8_t* tile, int lane, int part, const float* v) {
  uint8_t* wr = tile + lane * 128;
  const int sw = lane & 7;
#pragma unroll
  for (int j = 0; j < 4; ++j) *reinterpret_cast<uint4*>(wr + (((part * 4 + j) ^ sw) << 4)) = pack8_hi(v + 8 * j);
}
template <typename CR>
__device__ __forceinline__ void line_store_hi(const aldm_gemm_desc& d, const CR& cr, int n_group0, const uint8_t* tile, int lane) {
  __syncwarp();
  const int rs = lane >> 3, c8 = lane & 7;
  aldm_plane_t* out = reinterpret_cast<aldm_plane_t*>(d.out_hi);
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int rr = it * 4 + rs;
    const uint4 x = *reinterpret_cast<const uint4*>(tile + rr * 128 + ((c8 ^ (rr & 7)) << 4));
    if ((cr.vmask >> rr) & 1u) *reinterpret_cast<uint4*>(out + (cr.orow[it] * d.ldo + n_group0 + c8 * 8)) = x;
  }
  __syncwarp();
}

// ------------------------------------------------------------------------------------------
// tensor-core kernel
// ------------------------------------------------------------------------------------------
// Shared memory, in order: [halo slab (HALO only)] [STAGES stages] [fp32 accumulator] [barriers] [epilogue staging].
// Gather (HALO = 0): a stage is [a_hi | a_lo (AP == 2)] [b_hi | b_lo].  BN = 128: 2 stages (AP 2) / 3 (AP 1); BN = 64:
// 3 / 4; BN = 32: 4.
// Halo (HALO = 1, BN = 64 only): the A operand of one 64-channel block is a slab of the tile's (th + 2) x (tw + 2) = 180
// input pixels, 128 bytes each, per plane, rounded up to the 1024-byte swizzle atom: 23,552 B.  Two slabs, so that the
// next channel block loads while the MMAs run on this one; a stage holds one tap's weight tile [b_hi | b_lo] (16 KB).
// Budget (bytes): 232,448 - 32,768 accumulator - 16,896 staging - 1,280 alignment and barriers = 181,504 =
// 2 x AP x 23,552 slabs + 4 x 16,384 stages + 21,760 (AP 2) / 68,864 (AP 1) spare.  At BN = 128 the 64 KB accumulator
// leaves room for one slab only (148,736 = 2 x 23,552 + 3 x 32,768 + 3,328): every channel block then waits for its
// slab with the tensor cores idle, and that variant was slower (DESIGN.md section 5b).
template <int BN, int AP, int HALO = 0>
struct Tc3Cfg {
  static constexpr int BM = 128;
  static constexpr int BK = 64;                       // fp16 elements = 128 bytes per row
  static constexpr int A_BYTES = BM * 128;            // one plane
  static constexpr int B_BYTES = BN * 128;            // one plane
  static constexpr int HALO_PIX = 180;                // (8 + 2) x (16 + 2) or (16 + 2) x (8 + 2)
  static constexpr int SLAB_PLANE = HALO ? (HALO_PIX * 128 + 1023) / 1024 * 1024 : 0;
  static constexpr int NSLAB = HALO ? 2 : 0;
  static constexpr int SLAB_SET = AP * SLAB_PLANE;     // one slab: [a_hi | a_lo (AP == 2)]
  static constexpr int SLAB_BYTES = NSLAB * SLAB_SET;
  static constexpr int STAGE_BYTES = (HALO ? 0 : AP * A_BYTES) + 2 * B_BYTES;
  static constexpr int B_OFF = HALO ? 0 : AP * A_BYTES;
  static constexpr int ACC_BYTES = BM * BN * 4;       // fp32 accumulator tile handed from the warpgroups to the epilogue
  static constexpr int STG_BYTES = 4 * 32 * 33 * 4;   // one 32x33 fp32 transpose tile per epilogue warp
  static constexpr int SMEM_MAX = 227 * 1024;
  static constexpr int FIT = (SMEM_MAX - 1024 - 256 - STG_BYTES - ACC_BYTES - SLAB_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = FIT > 4 ? 4 : FIT;
  static constexpr int SMEM_BYTES = SLAB_BYTES + STAGES * STAGE_BYTES + ACC_BYTES + 1024 /*align slack*/ + 256 /*barriers*/ + STG_BYTES;
  static_assert(STAGES >= 2, "pipeline needs two stages");
  static_assert(SMEM_BYTES <= SMEM_MAX, "shared memory");
  static_assert(!HALO || BN == 64, "the halo path is built for BN = 64");
};

// Accumulator tile in shared memory: row-major fp32 [BM][BN], the 16-byte chunk index XOR-swizzled by (row & 7), so that
// the wgmma fragment stores and the row-per-lane reads of the epilogue (acc_ld32) are both free of bank conflicts.
// The fragment's rows g and g + 8 land in tile rows row0 + g and row0 + g + hstep (row0 a multiple of 8).
template <int BN>
__device__ __forceinline__ void acc_st_frag(float* accb, int row0, int hstep, int lane, const float* d) {
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row0 + g + hstep * h;
    float* rp = accb + row * BN + 2 * (t & 1);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
      *reinterpret_cast<float2*>(rp + (((2 * j + (t >> 1)) ^ (row & 7)) << 2)) = make_float2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
  }
}
// columns [c0, c0 + 32) of accumulator row `row`
template <int BN>
__device__ __forceinline__ void acc_ld32(const float* accb, int row, int c0, uint32_t* r) {
  const float* rp = accb + row * BN;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 x = *reinterpret_cast<const float4*>(rp + ((((c0 >> 2) + j) ^ (row & 7)) << 2));
    r[4 * j] = __float_as_uint(x.x); r[4 * j + 1] = __float_as_uint(x.y);
    r[4 * j + 2] = __float_as_uint(x.z); r[4 * j + 3] = __float_as_uint(x.w);
  }
}
// Register split of the persistent kernel (setmaxnreg, per thread).  Its four warpgroups put one warp of each role on
// every scheduler sub-partition: 80 (producer) + 2 x 136 (consumers) + 160 (epilogue) = 512 registers x 32 lanes, the
// sub-partition's 16,384.  The kernel is compiled for 512 threads at 128 registers, which is the same total.  80 is the
// least that holds the producers' per-row state without spilling; no instance spills at this split (ptxas -v).
constexpr int kProdRegs = 80, kConsRegs = 136, kEpiRegs = 160;
static_assert(kProdRegs + 2 * kConsRegs + kEpiRegs == 4 * 128, "register split must use exactly the launch allocation");
// wgmma_desc_sw128 with a stride byte offset of `sbo` bytes between 8-row groups (the halo slab's row pitch).
__device__ __forceinline__ uint64_t wgmma_desc_sw128_sbo(uint32_t smem_addr, uint32_t sbo) {
  return static_cast<uint64_t>((smem_addr >> 4) & 0x3FFFu) | (1ull << 16) | (static_cast<uint64_t>((sbo >> 4) & 0x3FFFu) << 32) |
         (1ull << 62);
}
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// Debug timeline (profiling aid, dbg bit 128): CTA 0 records clock64() at pipeline events.
// layout: [role 0..3][iteration 0..255][phase 0..1]
__device__ long long g_timeline[4 * 256 * 2];
#define ALDM_TL(role, i, ph)                                                      \
  do {                                                                            \
    if ((dbg & 128) && blockIdx.x == 0 && (i) < 256) g_timeline[((role) * 256 + (i)) * 2 + (ph)] = clock64(); \
  } while (0)

// ------------------------------------------------------------------------------------------
// persistent variant (default): one CTA per SM loops over output tiles; 512 threads = four warpgroups:
//   WG0, WG1 (warps 0-7)   consumers: wgmma into register accumulators, rows [64 wg, 64 wg + 64) of the tile;
//   WG2      (warps 8-11)  producers: the A gather, and the weight TMA from one elected lane of warp 8;
//   WG3      (warps 12-15) epilogue: warp ew finishes rows [32 ew, 32 ew + 32) of the tile, all BN columns.
// Accumulator hand-off, one 64 KB fp32 tile in shared memory (16-byte chunks swizzled by row, so that each epilogue lane
// reads a whole row) and two mbarriers that both complete once per tile, so that their phase is the parity of the CTA's
// tile counter: after the main loop of tile t the consumers wait acc_empty (the epilogue of t-1 is done reading the
// buffer), store the accumulator, arrive acc_full (one arrival per consumer warp) and start tile t+1.  The epilogue
// warpgroup walks the same tile sequence: it decodes the rows and fetches bias / residual of tile t, waits acc_full,
// finishes the tile and arrives acc_empty (one arrival per warp).  One buffer is enough: the consumers only need it
// again after a whole main loop, and the epilogue of tile t runs under the MMAs of tile t+1.
// The producers' per-stage work is one add + one bit test per row: row bases and per-row tap-validity masks are
// computed once per tile.  EPI selects a specialised epilogue body at compile time (0: linear/conv with optional
// bias, row vector, residual, dual/QKV plane outputs; 1: GEGLU; 2: everything else; 3/4: compact fp32 / planes).
// Tile order: split-K slice fastest, then n-tile, then m-tile, so CTAs running concurrently share the
// same activation rows in L2.
// ------------------------------------------------------------------------------------------
enum { EPI_FAST = ALDM_EPI_FAST, EPI_GEGLU = ALDM_EPI_GEGLU, EPI_GENERIC = ALDM_EPI_GENERIC, EPI_F32N = ALDM_EPI_F32N,
       EPI_PLN = ALDM_EPI_PLN };

// Division by a launch-time constant as multiply + shift (n < 2^31, d < 2^31): q = (n * M) >> (32 + l),
// M = floor(2^(32+l) / d) + 1, l = ceil(log2 d).  The persistent roles run one warp per scheduler, so a
// hardware-emulated integer division (~100 dependent instructions) per row per tile stalls the pipeline.
struct FastDiv {
  unsigned long long M;
  int sh;
  int d;
  __device__ __forceinline__ int div(int n) const {
    return (int)(((unsigned long long)(unsigned)n * M) >> sh);   // n >= 0
  }
  __device__ __forceinline__ void divmod(int n, int& q, int& r) const { q = div(n); r = n - q * d; }
};
static FastDiv make_fastdiv(int d) {
  FastDiv f;
  int l = 0;
  while ((1ll << l) < d) ++l;
  f.M = (unsigned long long)((((unsigned __int128)1) << (32 + l)) / (unsigned)d) + 1ull;
  f.sh = 32 + l;
  f.d = d;
  if (d == 1) { f.M = 1ull << 32; f.sh = 32; }
  return f;
}
struct Tc3Divs {
  FastDiv ow, oh, cp, tn, bmod;
  int plain;      // 1x1 tap, unit stride, no upsample / batch-modulo: input row == output row (linear layers)
  int store;      // ALDM_STORE_*: decided once on the host (gemm_select), so aldm_gemm_variant reports what runs
  // halo path: an M tile is a th x tw pixel block of one image (tw = 16, th = 8 or tw = 8, th = 16); tiles are numbered
  // image, then block row, then block column
  FastDiv tpi, tx;    // tiles per image, tiles per block row
  int tw_sh;          // log2(tw)
};

// AP = number of A planes (2: hi + lo, three MMAs per K step; 1: hi only, two MMAs and half the A bytes).
// HALO = 1 (BN = 64; aldm_gemm_a_mode): the A operand of each 64-channel block is one halo slab per plane and the
// consumers issue the nine taps of a 3x3 convolution from it (see the halo branches below).
template <int BN, int EPI, int AP, int HALO>
__global__ void __launch_bounds__(512, 1) gemm_tc3_kernel(const __grid_constant__ aldm_gemm_desc d, int tiles_m, int tiles_n,
                                                           const __grid_constant__ Tc3Divs fd) {
  using C = Tc3Cfg<BN, AP, HALO>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const uint32_t slab = base;                                  // HALO: C::NSLAB slabs of C::SLAB_SET bytes
  auto stage_base = [&](int s) { return base + C::SLAB_BYTES + s * C::STAGE_BYTES; };
  const uint32_t acc_base = base + C::SLAB_BYTES + C::STAGES * C::STAGE_BYTES;
  const uint32_t bar_base = acc_base + C::ACC_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (C::STAGES + s); };
  const uint32_t acc_full = bar_base + 8u * (2 * C::STAGES);
  const uint32_t acc_empty = acc_full + 8u;
  auto slab_full = [&](int i) { return acc_empty + 8u + 8u * i; };                 // HALO only
  auto slab_empty = [&](int i) { return acc_empty + 8u + 8u * (C::NSLAB + i); };
  float* accb = reinterpret_cast<float*>(smem_raw + (acc_base - raw));

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  const int M = d.B * d.OH * d.OW;
  const int nkb_total = d.Kpad / C::BK;
  const int total = tiles_m * tiles_n * d.splitk;
  const int dbg = d.impl >> 8;     // profiling aids (scripts/prof_ops.py --dbg): 1 skip A, 2 skip B, 4 skip MMA, 8 skip epilogue, 128 timeline

  if (tid == 0) {
    for (int s = 0; s < C::STAGES; ++s) {
      // gather: 128 cp.async producers (completion-triggered arrivals) + B expect_tx; halo: the B expect_tx alone
      mbar_init(full_bar(s), HALO ? 1 : 128 + 1);
      mbar_init(empty_bar(s), 8);        // one arrival per consumer warp once its MMAs on the stage have completed
    }
    mbar_init(acc_full, 8);              // one arrival per consumer warp: its rows of the accumulator are in shared memory
    mbar_init(acc_empty, 4);             // one arrival per epilogue warp: done reading the accumulator tile
    for (int i = 0; i < C::NSLAB; ++i) {
      mbar_init(slab_full(i), 96);       // the 96 halo producers' cp.async completions
      mbar_init(slab_empty(i), 8);       // one arrival per consumer warp once its MMAs on the slab have completed
    }
    fence_barrier_init();
  }
  __syncthreads();
  // Everything above overlapped the predecessor's tail; nothing below may touch its outputs before the wait.  Each role
  // waits inside its branch: the producers after the (memory-free) row decode of their first tile, and after the first
  // weight stages when those do not depend on the predecessor (ALDM_GEMM_STATIC_B).

  auto tile_coords = [&](int id, int& mt, int& nt, int& z, int& kb0, int& nkb) {
    int r = id;
    z = 0; kb0 = 0; nkb = nkb_total;
    if (d.splitk > 1) {
      z = id % d.splitk;
      r = id / d.splitk;
      kb0 = (int)(((long long)z * nkb_total) / d.splitk);
      nkb = (int)(((long long)(z + 1) * nkb_total) / d.splitk) - kb0;
    }
    fd.tn.divmod(r, mt, nt);
  };

  if (warp >= 8 && warp < 12) {
    // ===================== producers: A gather + weight TMA =====================
    setmaxnreg_dec<kProdRegs>();
    if constexpr (HALO) {
      // Halo: warps 8-10 load one slab per 64-channel block, one elected lane of warp 11 streams the weight tiles.  The K
      // loop runs channel block cb outer, tap inner; the weight tile of (tap, cb) is the packed k-block tap * Cp / 64 + cb.
      // The weights may be packed in d.bn = 128-row tiles: N tile nt is then rows [64 (nt % 2), + 64) of packed tile nt / 2,
      // one 8 KB run in each plane (a packed plane is 128-byte rows in N order, swizzled by row & 7).
      const int ncb = d.Cp >> 6;
      const int tw = 1 << fd.tw_sh, th = C::BM >> fd.tw_sh, hw = tw + 2;
      if (warp == 11) {
        if (!(d.impl & ALDM_GEMM_STATIC_B)) pdl_wait();       // the weights are the only global memory this lane reads
        if (elect_one()) {
          uint32_t cnt = 0;
          for (int id = blockIdx.x; id < total; id += gridDim.x) {
            int mt, nt, z, kb0, nkb;
            tile_coords(id, mt, nt, z, kb0, nkb);
            const int per = d.bn / BN;
            const long long wtile = 2ll * d.bn * 128;          // bytes of one packed (n tile, k-block) image
            const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(d.w_packed) + (long long)(nt / per) * nkb_total * wtile +
                                  (nt % per) * C::B_BYTES;
            for (int cb = 0; cb < ncb; ++cb)
              for (int tap = 0; tap < 9; ++tap, ++cnt) {
                const int s = cnt % C::STAGES;
                mbar_wait(empty_bar(s), ((cnt / C::STAGES) & 1) ^ 1);
                if (dbg & 2) { mbar_arrive(full_bar(s)); continue; }
                const uint8_t* src = wsrc + (long long)(tap * ncb + cb) * wtile;
                mbar_arrive_expect_tx(full_bar(s), 2 * C::B_BYTES);
                bulk_g2s(stage_base(s), src, C::B_BYTES, full_bar(s));
                bulk_g2s(stage_base(s) + C::B_BYTES, src + wtile / 2, C::B_BYTES, full_bar(s));
              }
          }
        }
        return;
      }
      // 180 halo pixels x 8 chunks of 16 bytes = 96 threads x 15 copies per plane: thread pt copies chunk j = pt & 7 of halo
      // pixels hr0 + 12 i (i < 15), into the slab row hr with the 128-byte swizzle (chunk j ^ (hr & 7)), the layout the
      // wgmma descriptors read.  12 i changes hr & 7 by 4 i: even and odd i have one destination base each.
      const int pt = tid - 256;
      const int j = pt & 7, hr0 = pt >> 3;
      // up = 1 (nearest x2 upsample folded in): halo pixel (hy, hx) at full resolution is source pixel
      // ((y0 - 1 + hy) >> 1, (x0 - 1 + hx) >> 1) = (y0 / 2 + ((hy - 1) >> 1), x0 / 2 + ((hx - 1) >> 1)), y0 and x0 being even
      const int Ws = d.W >> d.up;
      int relc[15];                              // element offset of each pixel from source pixel (y0 >> up, x0 >> up)
      uint32_t e_top = 0, e_bot = 0, e_lft = 0, e_rgt = 0;     // bit i: pixel i is on that edge of the halo
#pragma unroll
      for (int i = 0; i < 15; ++i) {
        const int hr = hr0 + 12 * i, hy = hr / hw, hx = hr - hy * hw;
        relc[i] = (((hy - 1) >> d.up) * Ws + ((hx - 1) >> d.up)) * d.Cp;
        e_top |= (uint32_t)(hy == 0) << i;
        e_bot |= (uint32_t)(hy == th + 1) << i;
        e_lft |= (uint32_t)(hx == 0) << i;
        e_rgt |= (uint32_t)(hx == tw + 1) << i;
      }
      const uint32_t d_even = slab + hr0 * 128 + ((j ^ (hr0 & 7)) << 4);
      const uint32_t d_odd = slab + hr0 * 128 + ((j ^ ((hr0 + 4) & 7)) << 4);
      const aldm_plane_t* ahi = reinterpret_cast<const aldm_plane_t*>(d.a_hi);
      const aldm_plane_t* alo = reinterpret_cast<const aldm_plane_t*>(d.a_lo);
      uint32_t cnt = 0;
      pdl_wait();
      for (int id = blockIdx.x; id < total; id += gridDim.x) {
        int mt, nt, z, kb0, nkb, b, t, ty, tx;
        tile_coords(id, mt, nt, z, kb0, nkb);
        fd.tpi.divmod(mt, b, t);
        fd.tx.divmod(t, ty, tx);
        const int y0 = ty * th, x0 = tx * tw;
        int bs = b;
        if (d.bmod > 0) { int q; fd.bmod.divmod(b, q, bs); }
        // the border pixels outside the image are the convolution's zero padding (cp.async zero fill)
        uint32_t valid = 0x7fffu;
        if (y0 == 0) valid &= ~e_top;
        if (y0 + th == d.H) valid &= ~e_bot;
        if (x0 == 0) valid &= ~e_lft;
        if (x0 + tw == d.W) valid &= ~e_rgt;
        const long long pix0 = ((long long)(bs * (d.H >> d.up) + (y0 >> d.up)) * Ws + (x0 >> d.up)) * d.Cp + j * 8;
        for (int cb = 0; cb < ncb; ++cb, ++cnt) {
          const int sl = cnt % C::NSLAB;
          mbar_wait(slab_empty(sl), ((cnt / C::NSLAB) & 1) ^ 1);
          const uint32_t de = d_even + sl * C::SLAB_SET, dod = d_odd + sl * C::SLAB_SET;
          if (!(dbg & 1)) {
            const aldm_plane_t* ab = ahi + pix0 + cb * 64;
            const aldm_plane_t* abl = alo + pix0 + cb * 64;
#define ALDM_HALO_PIX(i)                                                                                   \
            {                                                                                                \
              const uint32_t nb = ((valid >> (i)) & 1u) << 4;                                                \
              cp_async_16_off<(i) * 1536>((i) & 1 ? dod : de, ab + relc[i], nb);                             \
              if (AP == 2) cp_async_16_off<(i) * 1536 + C::SLAB_PLANE>((i) & 1 ? dod : de, abl + relc[i], nb); \
            }
            ALDM_HALO_PIX(0) ALDM_HALO_PIX(1) ALDM_HALO_PIX(2) ALDM_HALO_PIX(3) ALDM_HALO_PIX(4) ALDM_HALO_PIX(5)
            ALDM_HALO_PIX(6) ALDM_HALO_PIX(7) ALDM_HALO_PIX(8) ALDM_HALO_PIX(9) ALDM_HALO_PIX(10) ALDM_HALO_PIX(11)
            ALDM_HALO_PIX(12) ALDM_HALO_PIX(13) ALDM_HALO_PIX(14)
#undef ALDM_HALO_PIX
          }
          cp_async_mbar_arrive_noinc(slab_full(sl));
        }
      }
      return;
    }
    const int ptid = tid - 256;
    const int j = ptid & 7;                 // 16-byte chunk (8 channels) inside the 64-wide K block
    const int rbase = ptid >> 3;            // rows rbase + 16*i
    const uint32_t swz = (uint32_t)((j ^ (rbase & 7)) << 4);
    const int Hs = d.H >> d.up, Ws = d.W >> d.up;
    const aldm_plane_t* ahi = reinterpret_cast<const aldm_plane_t*>(d.a_hi);
    const aldm_plane_t* alo = reinterpret_cast<const aldm_plane_t*>(d.a_lo);
    uint32_t cnt = 0;
    int last_mt = -1;
    // Per-row state, kept small: the producers run at kProdRegs registers.
    int rowoff[8];            // element offset of tap (0,0) / channel 0 of each row (valid rows only); up = 1: b * Hs
    uint32_t tapmask[8];      // bit (t + 4) set <=> tap t of this row is inside the input (pre-shifted: (mask >> t) & 16 = bytes to copy)
    uint32_t yx0[8];          // up = 1 only: first input row | column << 16 (before the nearest-upsample shift)
    // Row decode of one M tile.  A single warp per scheduler runs this dependent integer chain slowly and the tensor
    // core idles meanwhile at every tile boundary of the short-K linear layers: linear layers take the trivial branch,
    // and the first tile is decoded before the programmatic-dependency wait (under the previous kernel's tail).
    auto decode_rows = [&](int mt) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int m = mt * C::BM + rbase + 16 * i;
        uint32_t msk = 0, yx = 0;
        int off = 0;
        if (fd.plain) {
          if (m < M) { msk = 16u; off = m * d.Cp; }
        } else if (m < M) {
          int t, ow, b, oh;
          fd.ow.divmod(m, t, ow);
          fd.oh.divmod(t, b, oh);
          const int y0 = oh * d.sy, x0 = ow * d.sx;
          int bs = b;
          if (d.bmod > 0) { int q; fd.bmod.divmod(b, q, bs); }
          const int pb = bs * Hs;
          yx = (uint32_t)y0 | ((uint32_t)x0 << 16);
          for (int tp = 0; tp < d.ntaps; ++tp) {
            const int ih = y0 + d.dy[tp], iw = x0 + d.dx[tp];
            if (ih >= 0 && ih < d.H && iw >= 0 && iw < d.W) msk |= 16u << tp;
          }
          off = d.up ? pb : ((pb + y0) * Ws + x0) * d.Cp;
        }
        tapmask[i] = msk;
        rowoff[i] = off;
        yx0[i] = yx;
      }
    };
    // The weight tile of every stage: one elected lane of warp 8 issues the bulk copy after the same empty-slot wait.
    const bool b_lane = warp == 8 && elect_one();
    auto w_tile = [&](int nt, int kb0) {
      return reinterpret_cast<const uint8_t*>(d.w_packed) + ((long long)nt * nkb_total + kb0) * (2 * C::B_BYTES);
    };
    auto issue_b = [&](uint32_t n, int s, const uint8_t* src) {
      ALDM_TL(1, n, 0);
      if (dbg & 2) { mbar_arrive(full_bar(s)); return; }
      mbar_arrive_expect_tx(full_bar(s), 2 * C::B_BYTES);
      bulk_g2s(base + s * C::STAGE_BYTES + C::B_OFF, src, 2 * C::B_BYTES, full_bar(s));
    };
    uint32_t b_pre = 0;       // weight stages issued before the dependency wait
    if ((int)blockIdx.x < total) {
      int mt, nt, z, kb0, nkb;
      tile_coords(blockIdx.x, mt, nt, z, kb0, nkb);
      decode_rows(mt);
      last_mt = mt;
      if (b_lane && (d.impl & ALDM_GEMM_STATIC_B)) {     // the weights do not depend on the predecessor: fill the free stages now
        b_pre = (uint32_t)(nkb < C::STAGES ? nkb : C::STAGES);
        for (uint32_t it = 0; it < b_pre; ++it) issue_b(it, (int)it, w_tile(nt, kb0) + (long long)it * (2 * C::B_BYTES));
      }
    }
    pdl_wait();
    for (int id = blockIdx.x; id < total; id += gridDim.x) {
      int mt, nt, z, kb0, nkb;
      tile_coords(id, mt, nt, z, kb0, nkb);
      if (mt != last_mt) {
        last_mt = mt;
        decode_rows(mt);
      }
      const uint8_t* wsrc = w_tile(nt, kb0);
      // (tap, c) of this thread's 8-channel chunk at the first k-block of the tile, then advanced by 64 per block
      const int k = kb0 * C::BK + j * 8;
      int tap, c;
      fd.cp.divmod(k, tap, c);
      for (int it = 0; it < nkb; ++it, ++cnt) {
        const int s = cnt % C::STAGES;
        mbar_wait(empty_bar(s), ((cnt / C::STAGES) & 1) ^ 1);
        if (ptid == 0) ALDM_TL(0, cnt, 0);
        if (b_lane && cnt >= b_pre) issue_b(cnt, s, wsrc + (long long)it * (2 * C::B_BYTES));
        const bool kvalid = tap < d.ntaps;
        const int tp = kvalid ? tap : 0;
        const uint32_t sa = base + s * C::STAGE_BYTES + swz;
        // Per 16-byte copy the producers issue 3 (linear) / 4 (conv) instructions: the destination is one register + an
        // immediate, the byte count (16 or 0 = zero fill) is a shift + mask of the per-row tap mask, and the source is one
        // 64-bit add on a per-k-block base.  The four producer warps run one per scheduler with every dependent instruction
        // exposed, so this count paces the pipeline.  A source address whose byte count is 0 is never dereferenced
        // (cp.async zero-fill), so it needs no clamping.
        if (fd.plain) {
          const uint32_t kb = (kvalid && c < d.Cp) ? 16u : 0u;
          const aldm_plane_t* ab = ahi + (kb ? c : 0);
          const aldm_plane_t* abl = alo + (kb ? c : 0);
          const uint32_t sa2 = sa + (uint32_t)rbase * 128u;
          if (!(dbg & 1)) {
#define ALDM_A_ROW(i)                                                                            \
            {                                                                                      \
              const uint32_t nb = tapmask[i] & kb;                                                 \
              cp_async_16_off<(i) * 2048>(sa2, ab + rowoff[i], nb);                                \
              if (AP == 2) cp_async_16_off<(i) * 2048 + C::A_BYTES>(sa2, abl + rowoff[i], nb);     \
            }
            ALDM_A_ROW(0) ALDM_A_ROW(1) ALDM_A_ROW(2) ALDM_A_ROW(3) ALDM_A_ROW(4) ALDM_A_ROW(5) ALDM_A_ROW(6) ALDM_A_ROW(7)
#undef ALDM_A_ROW
          }
        } else if (d.up == 0) {
          const int tapoff = (d.dy[tp] * Ws + d.dx[tp]) * d.Cp + c;
          const aldm_plane_t* ab = ahi + tapoff;
          const aldm_plane_t* abl = alo + tapoff;
          const int sh = kvalid ? tp : 27;                   // tapmask holds the validity bits pre-shifted by 4: (mask >> tp) & 16
          const uint32_t sa2 = sa + (uint32_t)rbase * 128u;
          if (!(dbg & 1)) {
#define ALDM_A_ROW(i)                                                                            \
            {                                                                                      \
              const uint32_t nb = (tapmask[i] >> sh) & 16u;                                        \
              cp_async_16_off<(i) * 2048>(sa2, ab + rowoff[i], nb);                                \
              if (AP == 2) cp_async_16_off<(i) * 2048 + C::A_BYTES>(sa2, abl + rowoff[i], nb);     \
            }
            ALDM_A_ROW(0) ALDM_A_ROW(1) ALDM_A_ROW(2) ALDM_A_ROW(3) ALDM_A_ROW(4) ALDM_A_ROW(5) ALDM_A_ROW(6) ALDM_A_ROW(7)
#undef ALDM_A_ROW
          }
        } else {      // nearest x2 upsample folded into the gather: source pixel = (ih >> 1, iw >> 1)
          const int dy = d.dy[tp], dx = d.dx[tp];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const bool ok = kvalid && ((tapmask[i] >> (tp + 4)) & 1u);
            long long off = 0;
            const int ih = (int)(yx0[i] & 0xffffu) + dy, iw = (int)(yx0[i] >> 16) + dx;
            if (ok) off = ((long long)(rowoff[i] + (ih >> 1)) * Ws + (iw >> 1)) * d.Cp + c;
            const uint32_t dst = sa + (uint32_t)(rbase + 16 * i) * 128u;
            cp_async_16(dst, ahi + off, ok ? 16u : 0u);
            if (AP == 2) cp_async_16(dst + C::A_BYTES, alo + off, ok ? 16u : 0u);
          }
        }
        cp_async_mbar_arrive_noinc(full_bar(s));
        if (ptid == 0) ALDM_TL(0, cnt, 1);
        c += C::BK;
        while (c >= d.Cp) { c -= d.Cp; ++tap; }
      }
    }
  } else if (warp < 8) {
    // ===================== consumers: warpgroup wg = rows [64 wg, 64 wg + 64) of the tile =====================
    setmaxnreg_inc<kConsRegs>();
    pdl_wait();
    const int wg = warp >> 2;
    if constexpr (HALO) {
      // Warpgroup wg computes 64 pixels of the tile as eight groups of 8 consecutive pixels of one row: tw = 16, columns
      // [8 wg, 8 wg + 8) of the 8 rows; tw = 8, rows [8 wg, 8 wg + 8).  In the slab the groups start one halo row (hw x 128
      // bytes, the descriptor's stride byte offset) apart, and tap (dy, dx) moves the start by dy hw + dx whole 128-byte
      // rows.  The hardware applies the 128-byte swizzle to the address it computes, and the slab is written swizzled by
      // its absolute row, so a window that starts at any row reads the slab as written.
      const int ncb = d.Cp >> 6;
      const int tw = 1 << fd.tw_sh, hw = tw + 2;
      const int row_c = (tw == 8 ? 8 * wg + 1 : 1) * hw + (tw == 16 ? 8 * wg : 0) + 1;     // tap (0, 0)
      const uint32_t sbo = (uint32_t)hw * 128u;
      uint32_t cnt = 0, scnt = 0, tl = 0;
      float acc[BN / 2];
      for (int id = blockIdx.x; id < total; id += gridDim.x, ++tl) {
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        for (int cb = 0; cb < ncb; ++cb, ++scnt) {
          const int sl = scnt % C::NSLAB;
          if (cb > 0) {     // the previous block's last weight stage and its slab, once their MMAs have completed
            wgmma_wait<0>();
            if (lane == 0) { mbar_arrive(empty_bar((cnt - 1) % C::STAGES)); mbar_arrive(slab_empty((scnt - 1) % C::NSLAB)); }
          }
          mbar_wait(slab_full(sl), (scnt / C::NSLAB) & 1);
          fence_proxy_async();        // cp.async-written slab -> visible to the tensor core (async proxy)
#pragma unroll 1
          for (int tap = 0; tap < 9; ++tap, ++cnt) {
            const int s = cnt % C::STAGES;
            if (tap > 0) {
              wgmma_wait<0>();
              if (lane == 0) mbar_arrive(empty_bar((cnt - 1) % C::STAGES));
            }
            mbar_wait(full_bar(s), (cnt / C::STAGES) & 1);
            const uint32_t sa = slab + sl * C::SLAB_SET + (uint32_t)(row_c + d.dy[tap] * hw + d.dx[tap]) * 128u;
            const uint64_t da_hi = wgmma_desc_sw128_sbo(sa, sbo);
            const uint64_t da_lo = wgmma_desc_sw128_sbo(sa + C::SLAB_PLANE, sbo);      // only used when AP == 2
            const uint64_t db_hi = wgmma_desc_sw128(stage_base(s));
            const uint64_t db_lo = wgmma_desc_sw128(stage_base(s) + C::B_BYTES);
            wgmma_fence();
            if (!(dbg & 4)) {
#pragma unroll
              for (int ks = 0; ks < 4; ++ks) {
                const uint64_t o = (uint64_t)(ks * 2);
                wgmma_ss<BN>(acc, da_hi + o, db_lo + o, 1);
                if (AP == 2) wgmma_ss<BN>(acc, da_lo + o, db_hi + o, 1);
                wgmma_ss<BN>(acc, da_hi + o, db_hi + o, 1);
              }
            }
            wgmma_commit();
          }
        }
        wgmma_wait<0>();
        wgmma_fence_regs<BN / 2>(acc);
        if (lane == 0) { mbar_arrive(empty_bar((cnt - 1) % C::STAGES)); mbar_arrive(slab_empty((scnt - 1) % C::NSLAB)); }
        if (tid == 0 && id + (int)gridDim.x >= total) pdl_launch();
        mbar_wait(acc_empty, (tl & 1) ^ 1);
        // tile row of pixel (y, x) = y tw + x.  tw = 16: this warp's fragment rows g and g + 8 are pixel groups
        // 2 (warp & 3) and 2 (warp & 3) + 1, i.e. tile rows 32 (warp & 3) + 8 wg + g and 16 further; tw = 8: the gather's order.
        if (tw == 16) acc_st_frag<BN>(accb, 32 * (warp & 3) + 8 * wg, 16, lane, acc);
        else acc_st_frag<BN>(accb, wg * 64 + (warp & 3) * 16, 8, lane, acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(acc_full);
      }
      return;
    }
    uint32_t cnt = 0, tl = 0;
    float acc[BN / 2];
    for (int id = blockIdx.x; id < total; id += gridDim.x, ++tl) {
      int mt, nt, z, kb0, nkb;
      tile_coords(id, mt, nt, z, kb0, nkb);
      // (the asm operands are read-write: a defined start value keeps the accumulator dead between tiles)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      for (int it = 0; it < nkb; ++it, ++cnt) {
        const int s = cnt % C::STAGES;
        // Release the previous stage as soon as its MMAs have completed, BEFORE waiting for this one.  Released after
        // this stage's wait, a slot whose MMAs are long done stays held while the consumers wait for data, so one load
        // fewer is in flight: with two stages (BN = 128, two A planes: the convolutions) only one.
        if (it > 0) {
          wgmma_wait<0>();
          if (lane == 0) mbar_arrive(empty_bar((cnt - 1) % C::STAGES));
        }
        mbar_wait(full_bar(s), (cnt / C::STAGES) & 1);
        if (tid == 0) ALDM_TL(2, cnt, 0);
        fence_proxy_async();          // cp.async-written A tiles -> visible to the tensor core (async proxy)
        const uint32_t sa = base + s * C::STAGE_BYTES;
        const uint64_t da_hi = wgmma_desc_sw128(sa + wg * 64 * 128);
        const uint64_t da_lo = wgmma_desc_sw128(sa + C::A_BYTES + wg * 64 * 128);      // only used when AP == 2
        const uint64_t db_hi = wgmma_desc_sw128(sa + C::B_OFF);
        const uint64_t db_lo = wgmma_desc_sw128(sa + C::B_OFF + C::B_BYTES);
        wgmma_fence();
        if (!(dbg & 4)) {
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) {            // 4 x K=16 (32 bytes) inside the 128B swizzle row
            const uint64_t o = (uint64_t)(ks * 2);
            wgmma_ss<BN>(acc, da_hi + o, db_lo + o, 1);      // small terms first
            if (AP == 2) wgmma_ss<BN>(acc, da_lo + o, db_hi + o, 1);
            wgmma_ss<BN>(acc, da_hi + o, db_hi + o, 1);
          }
        }
        wgmma_commit();
        if (tid == 0) ALDM_TL(2, cnt, 1);
      }
      wgmma_wait<0>();
      wgmma_fence_regs<BN / 2>(acc);
      if (lane == 0) mbar_arrive(empty_bar((cnt - 1) % C::STAGES));
      // all MMAs of this CTA are done: let the next kernel's blocks be scheduled under the last epilogue
      if (tid == 0 && id + (int)gridDim.x >= total) pdl_launch();
      // hand the accumulator over once the epilogue is done reading the previous tile's
      mbar_wait(acc_empty, (tl & 1) ^ 1);
      acc_st_frag<BN>(accb, wg * 64 + (warp & 3) * 16, 8, lane, acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(acc_full);
    }
  } else {
    // ===================== epilogue: warp ew = rows [32 ew, 32 ew + 32) of the tile, all BN columns =====================
    setmaxnreg_inc<kEpiRegs>();
    pdl_wait();
    const int ew = warp - 12;
    const int trow_in_tile = ew * 32 + lane;
    float* stg = reinterpret_cast<float*>(smem_raw + (bar_base + 256 - raw)) + ew * (32 * 33);
    uint8_t* stg8 = reinterpret_cast<uint8_t*>(stg);
    constexpr bool kCompact = EPI == EPI_F32N || EPI == EPI_PLN;
    constexpr int NCH = BN / 32;              // 32-column chunks per row
    constexpr int NRV = NCH > 1 ? 2 : 1;      // residual prefetch buffers (rotating)
    constexpr int NGV = BN >= 64 ? BN / 64 : 1;   // GEGLU: 32-column value chunks per row
    // full-line stores (line_store_hi): single fp16 plane out, no residual, whole 64-column groups (conditions: gemm_select)
    const bool pair_pln = EPI == EPI_PLN && BN >= 64 && fd.store == ALDM_STORE_PAIR_PLN;
    const bool pair_geglu = EPI == EPI_GEGLU && BN == 128 && fd.store == ALDM_STORE_PAIR_GEGLU;
    const bool pair_qk = EPI == EPI_FAST && BN >= 64 && fd.store == ALDM_STORE_PAIR_QK;
    const bool has_res = kCompact && d.res != nullptr;
    uint32_t tl = 0;
    for (int id = blockIdx.x; id < total; id += gridDim.x, ++tl) {
      int mt, nt, z, kb0, nkb;
      tile_coords(id, mt, nt, z, kb0, nkb);
      const int m = mt * C::BM + trow_in_tile;
      RowInfo r;
      if (HALO) {        // tile mt = (image, block row, block column), tile row = y tw + x; every row is inside the image
        int t, ty, tx;
        fd.tpi.divmod(mt, r.b, t);
        fd.tx.divmod(t, ty, tx);
        r.oh = ty * (C::BM >> fd.tw_sh) + (trow_in_tile >> fd.tw_sh);
        r.ow = (tx << fd.tw_sh) + (trow_in_tile & ((1 << fd.tw_sh) - 1));
        r.m = (r.b * d.OH + r.oh) * d.OW + r.ow;
        r.valid = true;
        r.orow = ((long long)r.b * d.OHF + (long long)r.oh * d.osy + d.ooy) * d.OWF + r.ow;
      } else {
        r.m = m; r.valid = m < M;
        const int mm = r.valid ? m : 0;
        int t;
        fd.ow.divmod(mm, t, r.ow);
        fd.oh.divmod(t, r.b, r.oh);
        r.orow = ((long long)r.b * d.OHF + (long long)r.oh * d.osy + d.ooy) * d.OWF + r.ow;
      }
      CoRows cr;
      CoRows32 cr32;
      if (kCompact) cr32 = co_rows32(r, lane); else cr = co_rows(r, lane);
      // bias and the first residual chunks are fetched while the consumers still accumulate the tile
      float4 pb4[NCH], prv[NRV][8];
      if (kCompact) {
#pragma unroll
        for (int ch = 0; ch < NCH; ++ch) {
          const int n = nt * BN + 32 * ch + (lane & 7) * 4;
          pb4[ch] = (d.bias && n < d.N) ? __ldg(reinterpret_cast<const float4*>(d.bias + n)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int ch = 0; ch < NRV; ++ch)
          if (has_res) co_load_res32(d, cr32, nt * BN + 32 * ch, d.N, lane, prv[ch]);
      }
      float pln_b[NCH];      // bias of each chunk's columns (lane = column), distributed by shuffles in full-line mode
#pragma unroll
      for (int ch = 0; ch < NCH; ++ch) {
        const int n = nt * BN + 32 * ch + lane;
        pln_b[ch] = (pair_pln && d.bias && n < d.N) ? __ldg(d.bias + n) : 0.f;
      }
      float gb_v[NGV], gb_g[NGV];       // GEGLU bias of each value / gate chunk (lane = column)
#pragma unroll
      for (int c = 0; c < NGV; ++c) {
        gb_v[c] = 0.f; gb_g[c] = 0.f;
        if (EPI == EPI_GEGLU && d.bias && d.splitk == 1) {
          gb_v[c] = __ldg(d.bias + nt * BN + 32 * c + lane);
          gb_g[c] = __ldg(d.bias + nt * BN + BN / 2 + 32 * c + lane);
        }
      }
      if (ew == 0 && lane == 0) ALDM_TL(3, 64 + tl * 8, 0);      // tile prologue (row decode, bias / residual prefetch) done
      mbar_wait(acc_full, tl & 1);
      if (ew == 0 && lane == 0) ALDM_TL(3, tl, 0);
      if (dbg & 8) {
        // skip
      } else if (d.splitk > 1) {
        // raw partial sums -> ws[z][m][n], coalesced through the staging tile
        const int Mpad = tiles_m * C::BM, Npad = tiles_n * BN;
        const int rs = lane >> 3, c4 = (lane & 7) * 4;
#pragma unroll 1
        for (int c0 = 0; c0 < BN; c0 += 32) {
          uint32_t v[32];
          acc_ld32<BN>(accb, trow_in_tile, c0, v);
#pragma unroll
          for (int i = 0; i < 32; ++i) stg[lane * 33 + i] = __uint_as_float(v[i]);
          __syncwarp();
#pragma unroll
          for (int it = 0; it < 8; ++it) {
            const int rr = it * 4 + rs;
            float* wp = d.ws + ((long long)z * Mpad + mt * C::BM + ew * 32 + rr) * Npad + nt * BN + c0 + c4;
            *reinterpret_cast<float4*>(wp) = make_float4(stg[rr * 33 + c4], stg[rr * 33 + c4 + 1], stg[rr * 33 + c4 + 2], stg[rr * 33 + c4 + 3]);
          }
          __syncwarp();
        }
      } else if (EPI == EPI_GEGLU) {
        // tile columns [0,BN/2) values, [BN/2,BN) gates; output width N/2, coalescable and without residual (host-checked)
        const int n_out = d.N / 2;
        float4 rv[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) rv[i] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll      // full unroll: the bias registers gb_v / gb_g are indexed by the chunk
        for (int c = 0; c < NGV; ++c) {
          const int c0 = 32 * c;
          const int n0 = nt * (BN / 2) + c0;
          uint32_t vr[32], gr[32];
          acc_ld32<BN>(accb, trow_in_tile, c0, vr);
          acc_ld32<BN>(accb, trow_in_tile, BN / 2 + c0, gr);
          if (c == 0 && ew == 0 && lane == 0) ALDM_TL(3, 64 + tl * 8 + 1, 0);
          float* v = reinterpret_cast<float*>(vr);
          float* g = reinterpret_cast<float*>(gr);
          // bias: fetched (one coalesced load per warp) BEFORE the accumulator wait, distributed by shuffles
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            v[i] += __shfl_sync(0xffffffffu, gb_v[c], i);
            g[i] += __shfl_sync(0xffffffffu, gb_g[c], i);
          }
#pragma unroll      // full unroll: v/g must stay in registers (a partial unroll indexes them dynamically -> local memory)
          for (int i = 0; i < 32; i += 8) geglu_mul<8>(v + i, g + i);
          if (c == 0 && ew == 0 && lane == 0) ALDM_TL(3, 64 + tl * 8 + 1, 1);
          if (pair_geglu) {                         // the FF1 case: one fp16 plane for FF2, stored as full lines
            line_put_hi(stg8, lane, c & 1, v);
            if (c & 1) line_store_hi(d, cr, nt * (BN / 2), stg8, lane);
          } else if (d.out_mode == ALDM_OUT_PLANES) {
            stage_rows(stg8, lane, v);
            emit_rows<true>(d, cr, n0, n_out, stg8, lane, rv, false, make_float4(0.f, 0.f, 0.f, 0.f));
          } else {
            epi_finish_coalesced(d, cr, n0, v, n_out, stg, lane, rv, false);
          }
        }
      } else if (kCompact && pair_pln) {
#pragma unroll
        for (int ch = 0; ch < NCH; ++ch) {
          uint32_t vr[32];
          acc_ld32<BN>(accb, trow_in_tile, 32 * ch, vr);
          float* v = reinterpret_cast<float*>(vr);
          if (d.bias) {
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] += __shfl_sync(0xffffffffu, pln_b[ch], i);
          }
          line_put_hi(stg8, lane, ch & 1, v);
          if (ch & 1) line_store_hi(d, cr32, nt * BN + 64 * (ch >> 1), stg8, lane);
        }
      } else if (kCompact) {
#pragma unroll
        for (int ch = 0; ch < NCH; ++ch) {
          const int c0 = 32 * ch;
          const int n0 = nt * BN + c0;
          const bool tl_on = ch < 2 && ew == 0 && lane == 0;
          uint32_t vr[32];
          acc_ld32<BN>(accb, trow_in_tile, c0, vr);
          if (tl_on) ALDM_TL(3, 64 + tl * 8 + 1 + 2 * ch, 0);
          stage_rows(stg8, lane, reinterpret_cast<const float*>(vr));
          if (tl_on) ALDM_TL(3, 64 + tl * 8 + 1 + 2 * ch, 1);
          if (tl_on) ALDM_TL(3, 64 + tl * 8 + 2 + 2 * ch, 0);
          emit_rows<EPI == EPI_PLN>(d, cr32, n0, d.N, stg8, lane, prv[ch % NRV], has_res, pb4[ch]);
          if (tl_on) ALDM_TL(3, 64 + tl * 8 + 2 + 2 * ch, 1);
          // the buffer just consumed takes the residual of the chunk NRV ahead
          if (has_res && ch + NRV < NCH) co_load_res32(d, cr32, n0 + 32 * NRV, d.N, lane, prv[ch % NRV]);
        }
      } else if (EPI == EPI_FAST) {
        // no activation; fp32 / planes / dual / QKV outputs, all through the coalesced path (host-checked)
        float4 rv[8];
#pragma unroll 1
        for (int c0 = 0; c0 < BN; c0 += 32) {
          const int n0 = nt * BN + c0;
          const bool vpart = d.out_mode == ALDM_OUT_QKV && n0 >= d.n_split;
          const bool pre = d.res != nullptr && !vpart;
          if (pre) co_load_res(d, cr, n0, d.N, lane, rv);
          uint32_t vr[32];
          acc_ld32<BN>(accb, trow_in_tile, c0, vr);
          float* v = reinterpret_cast<float*>(vr);
          if (d.bias) add_vec32(v, d.bias + n0);
          if (d.rowvec) add_vec32(v, d.rowvec + (long long)r.b * d.ld_rowvec + n0);
          if (!vpart && pair_qk) {
            // Q | K planes (one fp16 plane, 64 bytes per row and chunk): full-line stores per 64-column group
            line_put_hi(stg8, lane, (c0 >> 5) & 1, v);
            if (c0 & 32) line_store_hi(d, cr, nt * BN + (c0 & ~63), stg8, lane);
          } else if (!vpart) {
            epi_finish_coalesced(d, cr, n0, v, d.N, stg, lane, rv, pre);
          } else if (r.valid) {
            // V projection: transposed planes, lane == token -> consecutive lanes write consecutive bf16
            const int b = r.m / d.tok_per_batch, tok = r.m - b * d.tok_per_batch;
            const long long tb = ((long long)b * (d.N - d.n_split) + (n0 - d.n_split)) * d.ld_t + tok;
            aldm_plane_t* hp = reinterpret_cast<aldm_plane_t*>(d.out2_hi) + tb;
            aldm_plane_t* lp = d.out2_lo ? reinterpret_cast<aldm_plane_t*>(d.out2_lo) + tb : nullptr;
            const bool last = tok == d.tok_per_batch - 1;
#pragma unroll      // full unroll keeps v[] in registers
            for (int i = 0; i < 32; ++i) {
              if (n0 + i < d.N) store_split1(hp, lp, (long long)i * d.ld_t, v[i]);
            }
            if (last) {       // zero the padding keys [tok_per_batch, ld_t) (the attention kernel multiplies them by P = 0)
              for (int i = 0; i < 32 && n0 + i < d.N; ++i)
                for (int t = 1; tok + t < d.ld_t; ++t) store_split1(hp, lp, (long long)i * d.ld_t + t, 0.f);
            }
          }
        }
      } else {
        // generic: any activation / output mode, row-owner stores
#pragma unroll 1
        for (int c0 = 0; c0 < BN; c0 += 32) {
          if (d.act == ALDM_ACT_GEGLU) {
            if (c0 >= BN / 2) break;
            uint32_t vr[32], gr[32];
            acc_ld32<BN>(accb, trow_in_tile, c0, vr);
            acc_ld32<BN>(accb, trow_in_tile, BN / 2 + c0, gr);
            epi_activate(d, r, nt * BN + c0, reinterpret_cast<float*>(vr), reinterpret_cast<float*>(gr));
            epi_finish(d, r, nt * (BN / 2) + c0, 32, reinterpret_cast<float*>(vr), d.N / 2);
          } else {
            uint32_t vr[32];
            acc_ld32<BN>(accb, trow_in_tile, c0, vr);
            epi_activate(d, r, nt * BN + c0, reinterpret_cast<float*>(vr), nullptr);
            epi_finish(d, r, nt * BN + c0, 32, reinterpret_cast<float*>(vr), d.N);
          }
        }
      }
      if (ew == 0 && lane == 0) ALDM_TL(3, tl, 1);
      // every lane's reads of the accumulator tile are done: the consumers may overwrite it
      __syncwarp();
      if (lane == 0) mbar_arrive(acc_empty);
    }
  }
}

// ------------------------------------------------------------------------------------------
// split-K reduction + epilogue
// ------------------------------------------------------------------------------------------
__global__ void splitk_epilogue_kernel(const __grid_constant__ aldm_gemm_desc d, int Mpad, int Npad) {
  pdl_wait();
  const int M = d.B * d.OH * d.OW;
  const int chunks_per_row = (d.act == ALDM_ACT_GEGLU) ? (Npad / d.bn) * (d.bn / 64) : Npad / 32;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)M * chunks_per_row) return;
  const int m = (int)(idx / chunks_per_row);
  const int ch = (int)(idx % chunks_per_row);
  const RowInfo r = decode_row(d, m, M);
  float v[32], g[32];
  int pc0, n0, n_out;
  if (d.act == ALDM_ACT_GEGLU) {
    const int per_tile = d.bn / 64;
    const int tile = ch / per_tile, sub = ch % per_tile;
    pc0 = tile * d.bn + sub * 32;
    n0 = tile * (d.bn / 2) + sub * 32;
    n_out = d.N / 2;
  } else {
    pc0 = ch * 32; n0 = pc0; n_out = d.N;
  }
#pragma unroll
  for (int i = 0; i < 32; ++i) { v[i] = 0.f; g[i] = 0.f; }
  for (int z = 0; z < d.splitk; ++z) {
    const float* wp = d.ws + ((long long)z * Mpad + m) * Npad + pc0;
#pragma unroll
    for (int i = 0; i < 32; i += 4) {
      float4 t = *reinterpret_cast<const float4*>(wp + i);
      v[i] += t.x; v[i + 1] += t.y; v[i + 2] += t.z; v[i + 3] += t.w;
    }
    if (d.act == ALDM_ACT_GEGLU) {
#pragma unroll
      for (int i = 0; i < 32; i += 4) {
        float4 t = *reinterpret_cast<const float4*>(wp + d.bn / 2 + i);
        g[i] += t.x; g[i + 1] += t.y; g[i + 2] += t.z; g[i + 3] += t.w;
      }
    }
  }
  epi_activate(d, r, pc0, v, g);
  epi_finish(d, r, n0, 32, v, n_out);
}

// Coalesced variant for the cases the planner actually splits (no activation, alpha = 1, no accumulate; fp32,
// planes or dual output; bias / row vector / residual): one thread per (row, 4 columns), so the partial sums,
// the residual and the outputs are all full-line float4 streams, where the row-owner kernel above issues scattered
// per-row accesses for a few MB of traffic.
__global__ void __launch_bounds__(256) splitk_reduce4_kernel(const __grid_constant__ aldm_gemm_desc d, int Mpad, int Npad) {
  pdl_wait();
  const int M = d.B * d.OH * d.OW;
  const int q_per_row = (d.N + 3) >> 2;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)M * q_per_row) return;
  const int m = (int)(idx / q_per_row);
  const int n = (int)(idx % q_per_row) * 4;
  const RowInfo r = decode_row(d, m, M);
  float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int z = 0; z < d.splitk; ++z) {          // fixed order: deterministic
    const float4 t = *reinterpret_cast<const float4*>(d.ws + ((long long)z * Mpad + m) * Npad + n);
    x.x += t.x; x.y += t.y; x.z += t.z; x.w += t.w;
  }
  pdl_launch();
  if (d.bias) { const float4 t = __ldg(reinterpret_cast<const float4*>(d.bias + n)); x.x += t.x; x.y += t.y; x.z += t.z; x.w += t.w; }
  if (d.rowvec) {
    const float4 t = __ldg(reinterpret_cast<const float4*>(d.rowvec + (long long)r.b * d.ld_rowvec + n));
    x.x += t.x; x.y += t.y; x.z += t.z; x.w += t.w;
  }
  if (d.res) {
    const float4 t = __ldg(reinterpret_cast<const float4*>(d.res + r.orow * d.ld_res + n));
    x.x += t.x; x.y += t.y; x.z += t.z; x.w += t.w;
  }
  const long long o = r.orow * d.ldo + n;
  if (d.out_mode == ALDM_OUT_F32) *reinterpret_cast<float4*>(d.out + o) = x;
  if (d.out_mode == ALDM_OUT_PLANES || d.out_hi) {
    uint2 h, l;
    split2(x.x, x.y, h.x, l.x);
    split2(x.z, x.w, h.y, l.y);
    *reinterpret_cast<uint2*>(reinterpret_cast<aldm_plane_t*>(d.out_hi) + o) = h;
    if (d.out_lo) *reinterpret_cast<uint2*>(reinterpret_cast<aldm_plane_t*>(d.out_lo) + o) = l;
  }
}

// ------------------------------------------------------------------------------------------
// SIMT checker: obviously-correct restatement of the same descriptor on CUDA cores (fp32 FMA).
// One warp per output row, lanes over 32 packed columns.  Validation / debugging only.
// ------------------------------------------------------------------------------------------
__global__ void gemm_simt_kernel(const __grid_constant__ aldm_gemm_desc d, int Npad) {
  const int M = d.B * d.OH * d.OW;
  const int lane = threadIdx.x & 31;
  const int m = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (m >= M) return;
  const RowInfo r = decode_row(d, m, M);
  const int Hs = d.H >> d.up, Ws = d.W >> d.up;
  const int bsrc = d.bmod > 0 ? r.b % d.bmod : r.b;
  const aldm_plane_t* ahi = reinterpret_cast<const aldm_plane_t*>(d.a_hi);
  const aldm_plane_t* alo = reinterpret_cast<const aldm_plane_t*>(d.a_lo);      // NULL: single-plane operand
  const bool geglu = d.act == ALDM_ACT_GEGLU;
  const int nchunks = geglu ? (Npad / d.bn) * (d.bn / 64) : Npad / 32;
  for (int ch = blockIdx.y; ch < nchunks; ch += gridDim.y) {
    int pc0, n0, n_out;
    if (geglu) {
      const int per_tile = d.bn / 64;
      const int tile = ch / per_tile, sub = ch % per_tile;
      pc0 = tile * d.bn + sub * 32; n0 = tile * (d.bn / 2) + sub * 32; n_out = d.N / 2;
    } else {
      pc0 = ch * 32; n0 = pc0; n_out = d.N;
    }
    const float* wv = d.w_plain + (long long)(pc0 + lane) * d.Kpad;
    const float* wg = wv + (long long)(d.bn / 2) * d.Kpad;
    float acc = 0.f, accg = 0.f;
    for (int tap = 0; tap < d.ntaps; ++tap) {
      const int ih = r.oh * d.sy + d.dy[tap], iw = r.ow * d.sx + d.dx[tap];
      if (ih < 0 || ih >= d.H || iw < 0 || iw >= d.W) continue;
      const long long off = ((long long)(bsrc * Hs + (ih >> d.up)) * Ws + (iw >> d.up)) * d.Cp;
      const float* wt = wv + tap * d.Cp;
      const float* wgt = wg + tap * d.Cp;
      for (int c = 0; c < d.Cp; ++c) {
        const float a = plane_to_f(ahi[off + c]) + (alo ? plane_to_f(alo[off + c]) : 0.f);
        acc = fmaf(a, __ldg(wt + c), acc);
        if (geglu) accg = fmaf(a, __ldg(wgt + c), accg);
      }
    }
    // gather the 32 lanes' results into every lane's registers via shuffles, lane 0.. stores
    float v[32], g[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      v[i] = __shfl_sync(0xffffffffu, acc, i);
      g[i] = __shfl_sync(0xffffffffu, accg, i);
    }
    if (lane == 0) {
      epi_activate(d, r, pc0, v, g);
      epi_finish(d, r, n0, 32, v, n_out);
    }
  }
}

// ------------------------------------------------------------------------------------------
// host launch
// ------------------------------------------------------------------------------------------
// The kernel variant a descriptor runs: template parameters (BN, EPI, AP), split-K reduction kernel and store mode.  One
// function decides it for the launch and for aldm_gemm_variant, so what the query reports is what runs.
struct GemmVariant {
  int bn, epi, ap, red, store, amode;
};

// The halo A path (aldm_gemm_a_mode): a 3x3, stride-1 convolution whose pixels tile into 8 x 16 or 16 x 8 blocks.
static bool halo_ok(const aldm_gemm_desc& d) {
  static const bool on = [] { const char* e = getenv("ALDM_CONV_HALO"); return !(e && e[0] == '0'); }();   // A/B switch
  if (!on || (d.bn != 64 && d.bn != 128) || d.act == ALDM_ACT_GEGLU || d.splitk != 1 || d.ntaps != 9 || d.sy != 1 ||
      d.sx != 1 || d.Cp % 64 != 0 || d.OH != d.H || d.OW != d.W)
    return false;
  for (int t = 0; t < d.ntaps; ++t)
    if (d.dy[t] < -1 || d.dy[t] > 1 || d.dx[t] < -1 || d.dx[t] > 1) return false;
  return (d.W % 16 == 0 && d.H % 8 == 0) || (d.W == 8 && d.H % 16 == 0);
}

static GemmVariant gemm_select(const aldm_gemm_desc& d) {
  const bool halo = halo_ok(d);
  // the halo kernel runs 64-wide N tiles (two of them per 128-wide packed weight tile)
  GemmVariant v{halo ? 64 : d.bn, EPI_GENERIC, d.a_lo ? 2 : 1, ALDM_RED_NONE, ALDM_STORE_ROW, halo ? ALDM_AMODE_HALO : ALDM_AMODE_GATHER};
  const int BN = v.bn;
  // pick the specialised epilogue: the planner's dominant cases take the compact bodies
  const bool geglu = d.act == ALDM_ACT_GEGLU;
  const int n_out = geglu ? d.N / 2 : d.N;
  const bool co = d.splitk == 1 && n_out % 4 == 0 && d.ldo % 4 == 0 && (!d.res || d.ld_res % 4 == 0) &&
                  (d.out_mode == ALDM_OUT_F32 || d.out_mode == ALDM_OUT_PLANES || d.out_mode == ALDM_OUT_QKV);
  const long long out_rows = (long long)d.B * d.OHF * d.OWF;
  const int ld_max = d.ldo > d.ld_res ? d.ldo : d.ld_res;
  static const bool compact_on = [] { const char* e = getenv("ALDM_EPI_COMPACT"); return !(e && e[0] == '0'); }();   // A/B switch
  const bool plain = compact_on && co && d.act == ALDM_ACT_NONE && d.alpha == 1.0f && !d.accumulate && !d.rowvec &&
                     out_rows * ld_max < (1ll << 31) &&
                     (!d.bias || aligned16(d.bias)) && (!d.res || aligned16(d.res));
  if (co && geglu && !d.res && d.out_mode != ALDM_OUT_QKV && BN >= 64) v.epi = EPI_GEGLU;
  else if (plain && d.out_mode == ALDM_OUT_F32 && aligned16(d.out) && (!d.out_hi || d.ldo % 4 == 0)) v.epi = EPI_F32N;
  else if (plain && d.out_mode == ALDM_OUT_PLANES) v.epi = EPI_PLN;
  else if (co && d.act == ALDM_ACT_NONE) v.epi = EPI_FAST;
  if (v.epi == EPI_F32N || v.epi == EPI_PLN) v.store = ALDM_STORE_COMPACT;
  // full-line pair stores (emit_pair_hi): one fp16 plane out, no residual, whole 64-column groups, and every tile's columns
  // inside the output (emit_pair_hi does not check them: N % BN == 0 for the planes form)
  const bool pair_ok = d.out_lo == nullptr && d.splitk == 1 && d.ldo % 8 == 0 && aligned16(d.out_hi);
  if (v.epi == EPI_PLN && BN >= 64 && pair_ok && d.res == nullptr && d.N % BN == 0) v.store = ALDM_STORE_PAIR_PLN;
  if (v.epi == EPI_GEGLU && BN == 128 && pair_ok && d.out_mode == ALDM_OUT_PLANES && (d.N / 2) % 64 == 0) v.store = ALDM_STORE_PAIR_GEGLU;
  if (v.epi == EPI_FAST && BN >= 64 && pair_ok && d.out_mode == ALDM_OUT_QKV && d.res == nullptr && d.n_split % 64 == 0)
    v.store = ALDM_STORE_PAIR_QK;
  if (d.splitk > 1) {
    // coalesced reduction for the cases the planner actually splits; the row-owner kernel for everything else
    const bool fast = d.act == ALDM_ACT_NONE && d.alpha == 1.0f && !d.accumulate && d.N % 4 == 0 && d.ldo % 4 == 0 &&
                      (d.out_mode == ALDM_OUT_F32 || d.out_mode == ALDM_OUT_PLANES) && (!d.res || (d.ld_res % 4 == 0 && aligned16(d.res))) &&
                      (!d.bias || aligned16(d.bias)) && (!d.rowvec || (d.ld_rowvec % 4 == 0 && aligned16(d.rowvec))) &&
                      (d.out_mode != ALDM_OUT_F32 || aligned16(d.out));
    v.red = fast ? ALDM_RED_REDUCE4 : ALDM_RED_GENERIC;
  }
  return v;
}

template <int BN, int EPI, int AP, int HALO>
static int launch_tc3_mode(const aldm_gemm_desc& d, int M, const GemmVariant& v, cudaStream_t st) {
  using C = Tc3Cfg<BN, AP, HALO>;
  static bool configured = false;
  if (!configured) {
    ALDM_CHECK_CUDA(cudaFuncSetAttribute(gemm_tc3_kernel<BN, EPI, AP, HALO>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
    configured = true;
  }
  const int tiles_m = cdiv(M, C::BM), tiles_n = cdiv(d.N, BN);
  const long long total = (long long)tiles_m * tiles_n * d.splitk;
  const int grid = (int)(total < num_sms() ? total : num_sms());
  Tc3Divs fd;
  fd.ow = make_fastdiv(d.OW); fd.oh = make_fastdiv(d.OH); fd.cp = make_fastdiv(d.Cp); fd.tn = make_fastdiv(tiles_n);
  fd.bmod = make_fastdiv(d.bmod > 0 ? d.bmod : 1);
  fd.plain = d.ntaps == 1 && d.dy[0] == 0 && d.dx[0] == 0 && d.sy == 1 && d.sx == 1 && d.up == 0 && d.bmod <= 0 &&
             d.OH == d.H && d.OW == d.W;
  fd.store = v.store;
  fd.tw_sh = d.W == 8 ? 3 : 4;
  const int tw = 1 << fd.tw_sh, th = C::BM / tw;
  fd.tx = make_fastdiv(HALO ? d.W / tw : 1);
  fd.tpi = make_fastdiv(HALO ? (d.H / th) * (d.W / tw) : 1);
  ALDM_CHECK_CUDA(launch_pdl(gemm_tc3_kernel<BN, EPI, AP, HALO>, dim3(grid), dim3(512), C::SMEM_BYTES, st, d, tiles_m, tiles_n, fd));
  ALDM_CHECK_CUDA(cudaGetLastError());
  if (d.splitk > 1) {
    const int Mpad = tiles_m * C::BM, Npad = tiles_n * BN;
    const int chunks = (d.act == ALDM_ACT_GEGLU) ? (Npad / BN) * (BN / 64) : Npad / 32;
    const long long tot = (long long)M * chunks;
    // plain launches (full serialisation): early-scheduled reduction blocks only disturbed the GEMM's last epilogue
    if (v.red == ALDM_RED_REDUCE4) {
      const long long q = (long long)M * ((d.N + 3) / 4);
      splitk_reduce4_kernel<<<(unsigned)((q + 255) / 256), 256, 0, st>>>(d, Mpad, Npad);
    } else {
      splitk_epilogue_kernel<<<(unsigned)((tot + 127) / 128), 128, 0, st>>>(d, Mpad, Npad);
    }
    ALDM_CHECK_CUDA(cudaGetLastError());
  }
  return ALDM_OK;
}

template <int BN, int EPI, int AP>
static int launch_tc3_ap(const aldm_gemm_desc& d, int M, const GemmVariant& v, cudaStream_t st) {
  if constexpr (BN == 64)
    if (v.amode == ALDM_AMODE_HALO) return launch_tc3_mode<BN, EPI, AP, 1>(d, M, v, st);
  return launch_tc3_mode<BN, EPI, AP, 0>(d, M, v, st);
}

template <int BN, int EPI>
static int launch_tc3_epi(const aldm_gemm_desc& d, int M, const GemmVariant& v, cudaStream_t st) {
  return v.ap == 2 ? launch_tc3_ap<BN, EPI, 2>(d, M, v, st) : launch_tc3_ap<BN, EPI, 1>(d, M, v, st);
}

template <int BN>
static int launch_tc2(const aldm_gemm_desc& d, int M, const GemmVariant& v, cudaStream_t st) {
  switch (v.epi) {
    case EPI_GEGLU: return launch_tc3_epi<BN, EPI_GEGLU>(d, M, v, st);
    case EPI_F32N: return launch_tc3_epi<BN, EPI_F32N>(d, M, v, st);
    case EPI_PLN: return launch_tc3_epi<BN, EPI_PLN>(d, M, v, st);
    case EPI_FAST: return launch_tc3_epi<BN, EPI_FAST>(d, M, v, st);
    default: return launch_tc3_epi<BN, EPI_GENERIC>(d, M, v, st);
  }
}

int gemm_num_launches(const aldm_gemm_desc& d) { return ((d.impl & 0xff) != ALDM_GEMM_SIMT && d.splitk > 1) ? 2 : 1; }

// descriptor checks shared by the launch and the variant query (no CUDA calls)
static int gemm_check(const aldm_gemm_desc& d) {
  const long long Mll = (long long)d.B * d.OH * d.OW;
  ALDM_REQUIRE(Mll > 0 && Mll < (1ll << 31), ALDM_E_SHAPE, "gemm: bad M=%lld", Mll);
  ALDM_REQUIRE(d.bn == 32 || d.bn == 64 || d.bn == 128, ALDM_E_UNSUPPORTED, "gemm: bn=%d unsupported", d.bn);
  ALDM_REQUIRE(d.Cp % 8 == 0 && d.Cp > 0, ALDM_E_SHAPE, "gemm: Cp=%d must be a positive multiple of 8", d.Cp);
  ALDM_REQUIRE(d.ntaps >= 1 && d.ntaps <= ALDM_MAX_TAPS, ALDM_E_SHAPE, "gemm: ntaps=%d", d.ntaps);
  ALDM_REQUIRE(d.K == d.ntaps * d.Cp, ALDM_E_SHAPE, "gemm: K=%d != ntaps*Cp=%d", d.K, d.ntaps * d.Cp);
  ALDM_REQUIRE(d.Kpad % 64 == 0 && d.Kpad >= d.K, ALDM_E_SHAPE, "gemm: Kpad=%d (K=%d)", d.Kpad, d.K);
  ALDM_REQUIRE(d.N >= 1, ALDM_E_SHAPE, "gemm: N=%d", d.N);
  ALDM_REQUIRE(d.a_hi, ALDM_E_ARG, "gemm: null A plane");      // a_lo == NULL: single-plane activations
  ALDM_REQUIRE(aligned16(d.a_hi) && aligned16(d.a_lo), ALDM_E_ALIGN, "gemm: A planes not 16B aligned");
  ALDM_REQUIRE(d.up == 0 || d.up == 1, ALDM_E_ARG, "gemm: up=%d", d.up);
  ALDM_REQUIRE(d.up == 0 || (d.H < 65536 && d.W < 65536), ALDM_E_SHAPE, "gemm: upsampled input %dx%d too large", d.H, d.W);
  ALDM_REQUIRE(d.splitk >= 1 && d.splitk <= d.Kpad / 64, ALDM_E_ARG, "gemm: splitk=%d", d.splitk);
  ALDM_REQUIRE(d.splitk == 1 || d.ws, ALDM_E_ARG, "gemm: split-K needs a workspace");
  if (d.act == ALDM_ACT_GEGLU) {
    ALDM_REQUIRE(d.bn >= 64 && d.N % d.bn == 0, ALDM_E_SHAPE, "gemm: GEGLU needs N %% bn == 0 and bn >= 64");
    ALDM_REQUIRE(!d.rowvec, ALDM_E_UNSUPPORTED, "gemm: GEGLU with rowvec");
  }
  if (d.out_mode == ALDM_OUT_QKV) {
    ALDM_REQUIRE(d.out2_hi && d.n_split > 0 && d.n_split < d.N && d.n_split % d.bn == 0 && d.n_split % 32 == 0,
                 ALDM_E_ARG, "gemm: bad QKV split (n_split=%d, N=%d, bn=%d)", d.n_split, d.N, d.bn);
    ALDM_REQUIRE(d.tok_per_batch > 0 && d.ld_t >= d.tok_per_batch && d.act != ALDM_ACT_GEGLU, ALDM_E_ARG,
                 "gemm: bad QKV token layout");
  }
  if (d.out_mode == ALDM_OUT_F32 || d.out_mode == ALDM_OUT_NCHW) {
    ALDM_REQUIRE(d.out, ALDM_E_ARG, "gemm: null out");
  } else {
    ALDM_REQUIRE(d.out_hi, ALDM_E_ARG, "gemm: null out plane");      // out_lo == NULL: single-plane output
    ALDM_REQUIRE(!d.accumulate, ALDM_E_UNSUPPORTED, "gemm: accumulate into planes");
  }
  if ((d.impl & 0xff) == ALDM_GEMM_SIMT) {
    ALDM_REQUIRE(d.w_plain, ALDM_E_ARG, "gemm: SIMT path needs w_plain");
  } else {
    ALDM_REQUIRE(d.w_packed && aligned16(d.w_packed), ALDM_E_ARG, "gemm: w_packed null/unaligned");
  }
  return ALDM_OK;
}

int gemm_launch(const aldm_gemm_desc& d, cudaStream_t st) {
  const int rc = gemm_check(d);
  if (rc) return rc;
  const int M = d.B * d.OH * d.OW;
  if ((d.impl & 0xff) == ALDM_GEMM_SIMT) {
    const int Npad = cdiv(d.N, d.bn) * d.bn;
    const bool geglu = d.act == ALDM_ACT_GEGLU;
    const int nchunks = geglu ? (Npad / d.bn) * (d.bn / 64) : Npad / 32;
    dim3 grid(cdiv(M, 4), nchunks < 64 ? nchunks : 64);
    gemm_simt_kernel<<<grid, 128, 0, st>>>(d, Npad);
    ALDM_CHECK_CUDA(cudaGetLastError());
    return ALDM_OK;
  }
  // ALDM_GEMM_TC_V1 (the round-1 one-tile-per-CTA kernel) is retired: the value selects the persistent kernel
  const GemmVariant v = gemm_select(d);
  switch (v.bn) {
    case 128: return launch_tc2<128>(d, M, v, st);
    case 64: return launch_tc2<64>(d, M, v, st);
    default: return launch_tc2<32>(d, M, v, st);
  }
}

}  // namespace aldm

extern "C" int aldm_debug_timeline(long long* host_out, int32_t n) {
  using namespace aldm;
  ALDM_REQUIRE(host_out && n > 0 && n <= 4 * 256 * 2, ALDM_E_ARG, "debug_timeline: bad arguments");
  ALDM_CHECK_CUDA(cudaMemcpyFromSymbol(host_out, g_timeline, sizeof(long long) * n));
  void* sym = nullptr;        // cleared after every read so that stamps of different cases never mix
  ALDM_CHECK_CUDA(cudaGetSymbolAddress(&sym, g_timeline));
  ALDM_CHECK_CUDA(cudaMemset(sym, 0, sizeof(g_timeline)));
  return ALDM_OK;
}

extern "C" int aldm_gemm_variant(const aldm_gemm_desc* d, int32_t out[5]) {
  if (!d || !out) { aldm::set_error("aldm_gemm_variant: null argument"); return ALDM_E_ARG; }
  const int rc = aldm::gemm_check(*d);
  if (rc) return rc;
  if ((d->impl & 0xff) == ALDM_GEMM_SIMT) { aldm::set_error("aldm_gemm_variant: the SIMT checker has no variants"); return ALDM_E_UNSUPPORTED; }
  const aldm::GemmVariant v = aldm::gemm_select(*d);
  out[0] = v.bn; out[1] = v.epi; out[2] = v.ap; out[3] = v.red; out[4] = v.store;
  return ALDM_OK;
}

extern "C" int aldm_gemm_a_mode(const aldm_gemm_desc* d, int32_t* mode) {
  if (!d || !mode) { aldm::set_error("aldm_gemm_a_mode: null argument"); return ALDM_E_ARG; }
  const int rc = aldm::gemm_check(*d);
  if (rc) return rc;
  if ((d->impl & 0xff) == ALDM_GEMM_SIMT) { aldm::set_error("aldm_gemm_a_mode: the SIMT checker has no variants"); return ALDM_E_UNSUPPORTED; }
  *mode = aldm::gemm_select(*d).amode;
  return ALDM_OK;
}

extern "C" int aldm_gemm(const aldm_gemm_desc* d, void* stream) {
  if (!d) { aldm::set_error("aldm_gemm: null desc"); return ALDM_E_ARG; }
  return aldm::gemm_launch(*d, reinterpret_cast<cudaStream_t>(stream));
}
