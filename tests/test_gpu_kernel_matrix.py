"""Conformance matrix: every GEMM kernel variant, both attention kernels and the GroupNorm statistics against float64
references, with guard bands that catch stores outside the output.

GEMM.  GEMM_MATRIX is a table of descriptors that together reach every kernel variant aldm_gemm_variant can report:
N tile 32 / 64 / 128 x A planes 1 / 2 x epilogue body (FAST, GEGLU, GENERIC, F32N, PLN) x split-K reduction (none,
reduce4, generic) x store mode (row, compact, pair_pln, pair_geglu, pair_qk), over the plain, convolution, strided,
nearest-upsample and batch-modulo gathers.  test_gemm_matrix_reaches_every_variant checks that on the CPU, and that every
epilogue body and every pair store runs with at least 3 tiles per persistent CTA and a ragged last M tile (those cases
are sized from the GPU's SM count).  Split-K is forced by editing the planned op.

The reference is float64 and shares nothing with tests/emulator.py or the weight packing: the A operand is gathered from
the operand planes as the kernel reads them (hi + lo, or hi alone) through the tap list, the weight is the fp32 master
matrix [N, taps, Cin] (GEGLU: values then gates, in the module's order), and the epilogue is the one documented in
include/aldm_b200.h, with the erf GELU, tanh and SiLU computed exactly.

Bounds, each checked as relative L2 AND per element (so that one wrong row, column or tile is not diluted):
  * fp32 and two-plane outputs: relative L2 < 2e-5; |err| <= 1e-4 rms(ref).  The kernel's own error is the fp32
    accumulation (about sqrt(K) 2^-24 |partial sum|, < 5e-6 rms(ref) at K = 5760) plus the 2^-22 operand split, so the
    per-element bound leaves a 20x margin over the largest of ~10^7 elements, while a wrong element is off by ~rms(ref).
  * single-plane (fp16) outputs: relative L2 < 3e-4; |err| <= 2^-10 |ref| + 1e-5 rms(ref).  Rounding to fp16 costs at most
    2^-11 |ref|; the compute error can move a value across one rounding boundary, which at most doubles that; the
    absolute term covers results in the fp16 subnormal range.
Attention: Q, K and V^T are single fp16 planes; the reference uses those fp16 values, fills masked scores with
  -finfo(float32).max (a fully masked row then averages V uniformly, as the reference module does) and takes the softmax
  in float64.  The wgmma kernel rounds the probabilities to fp16 (relative error <= 2^-11 each) and both kernels round the
  output to fp16, so per element |err| <= 2^-11 (|ref| + sum_k p_k |v_k|); the test allows twice that (2^-10), plus
  1e-6 for the fp32 score and exponent arithmetic.  Relative L2 < 5e-4.
GroupNorm: inputs whose every (batch, group) has |mean| / std of 30 or 100 (asserted); outputs as the GEMM's
  (two-plane GN+SiLU, single-plane GN), plus 2^-21 |x| rstd |gamma| per element: the fp32 apply y = x sc + sh works on
  terms of that size (x sc and mean sc, ~ratio), and its roundings of sc, mean, mean sc, sh and y cost about five units of
  2^-24 of it (SiLU's slope is below 1.1).  An error in the statistics themselves is not bounded by this: a mean off by
  d shifts every output of the group by d rstd |gamma|, an rstd off by e scales it by 1 + e.

Guard bands.  Every output window has at least 4 KB of guard bytes before and after it, so a stray store lands inside
the test's own workspace.  The workspace is filled with 0xFF bytes (NaN as fp16 and fp32) before the inputs are written,
except the split-K and GroupNorm scratch, which must start at zero; the split-K scratch is followed by GUARD zero bytes that
must stay zero.  After one run every byte outside the declared output windows and the scratch must be unchanged: inputs,
guards, and the padding columns between n_out and ld (fp32, compact, per-warp and pair plane stores).  The V^T padding keys belong to
the QKV window and must be exactly zero."""
import math
from dataclasses import dataclass
from typing import Optional

import numpy as np
import pytest
import torch

from audioldm2_b200 import _lib, engine, plan
from audioldm2_b200.packing import round_up
from audioldm2_b200.plan import F32, VT, Planes, Planner, Ref
from tests.conftest import rel_l2

DEV = "cuda:0"
GUARD = 4096
FLT_MAX = float(np.finfo(np.float32).max)
T3, T3A = plan.TAPS_3x3, plan.TAPS_3x3_ASYM
GEGLU, TANH, SILU = _lib.ACT_GEGLU, _lib.ACT_TANH, _lib.ACT_SILU


def _n_sm() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


# ----------------------------------------------------------------------------------------------
# workspace windows and guards
# ----------------------------------------------------------------------------------------------
@dataclass
class Win:
    """Output window: `rows` (None: all) of a [n_rows, ld] array of `esz`-byte elements at byte `off`, columns [0, cols)."""
    off: int
    n_rows: int
    ld: int
    cols: int
    esz: int
    rows: Optional[torch.Tensor] = None

    def view(self, ws: torch.Tensor) -> torch.Tensor:
        dt = {4: torch.float32, 2: torch.float16}[self.esz]
        full = ws[self.off:self.off + self.n_rows * self.ld * self.esz].view(dt).view(self.n_rows, self.ld)
        return (full if self.rows is None else full[self.rows.to(ws.device)])[:, :self.cols]

    def mark(self, mask: torch.Tensor):
        m = mask[self.off:self.off + self.n_rows * self.ld * self.esz].view(self.n_rows, self.ld * self.esz)
        if self.rows is None:
            m[:, :self.cols * self.esz] = True
        else:
            m[self.rows.to(mask.device), :self.cols * self.esz] = True


def _guarded(P: Planner, nbytes: int) -> Ref:
    """nbytes with GUARD bytes before and at least GUARD bytes after them."""
    return P.raw(GUARD + round_up(nbytes, 256) + GUARD) + GUARD


def _guarded_planes(P: Planner, rows: int, ld: int, n: int) -> Planes:
    hi = _guarded(P, rows * ld * 2)
    return Planes(hi, _guarded(P, rows * ld * 2) if n == 2 else None, rows, ld)


def _run_guarded(pl: plan.Plan, writes, wins, zero=(), scratch=()):
    """0xFF-fill the workspace, zero the `zero` regions (scratch that must start at zero, with any guard after it), write
    the inputs, run once; every byte outside `wins` and the `scratch` regions the kernels may rewrite must be unchanged."""
    prog = engine.DeviceProgram(pl, torch.device(DEV), dict(all=(0, len(pl.ops))))
    ws = prog.ws
    ws.fill_(0xFF)
    for off, n in zero:
        ws[off:off + n].zero_()
    for off, t in writes:
        b = t.contiguous().view(torch.uint8).reshape(-1)
        ws[off:off + b.numel()].copy_(b.to(DEV))
    before = ws.clone()
    prog.run("all")
    torch.cuda.synchronize()
    _assert_unchanged(ws, before, wins, scratch)
    return prog


def _assert_unchanged(ws: torch.Tensor, before: torch.Tensor, wins, scratch=()):
    """Every byte of `ws` outside the windows and the scratch regions equals `before`."""
    inside = torch.zeros_like(ws, dtype=torch.bool)
    for w in wins:
        w.mark(inside)
    for off, n in scratch:
        inside[off:off + n] = True
    stray = ((ws != before) & ~inside).nonzero().flatten()
    if stray.numel():
        first = int(stray[0])
        where = None
        for w in wins:
            rel = first - w.off
            if 0 <= rel < w.n_rows * w.ld * w.esz:        # inside the array but outside the window: a padding column
                where = f"row {rel // (w.ld * w.esz)}, column {rel % (w.ld * w.esz) // w.esz} of the [{w.n_rows}, {w.ld}] " \
                        f"array at {w.off} (window: columns < {w.cols})"
        if where is None:
            near = min(wins, key=lambda w: abs(first - w.off - w.n_rows * w.ld * w.esz))
            where = f"{first - near.off - near.n_rows * near.ld * near.esz:+d} bytes past the end of the array at {near.off}"
        raise AssertionError(f"{stray.numel()} bytes changed outside the output windows; first at workspace byte {first}: "
                             f"{where}; scratch regions (first, last byte): {[(o, o + n - 1) for o, n in scratch]}")


def _check(name: str, got: torch.Tensor, ref: torch.Tensor, planes: int, extra: Optional[torch.Tensor] = None):
    """planes: 0 fp32 output, 2 two-plane output, 1 single fp16 plane; extra: per-element term added to the bound."""
    got, ref = got.double().reshape(-1), ref.double().reshape(-1).to(got.device)
    assert torch.isfinite(got).all(), f"{name}: non-finite output"
    err = (got - ref).abs()
    rms = float(ref.pow(2).mean().sqrt())
    bound = 2.0 ** -10 * ref.abs() + 1e-5 * rms if planes == 1 else torch.full_like(ref, 1e-4 * rms)
    if extra is not None:
        bound = bound + extra.double().reshape(-1).to(got.device)
    rl2 = rel_l2(got, ref)
    assert rl2 < (3e-4 if planes == 1 else 2e-5), f"{name}: relative L2 {rl2:.3e}"
    bad = (err > bound).nonzero().flatten()
    assert bad.numel() == 0, (f"{name}: {bad.numel()} elements over the bound; first flat index {int(bad[0])}: "
                              f"got {float(got[bad[0]]):.6g} want {float(ref[bad[0]]):.6g}")


# ----------------------------------------------------------------------------------------------
# GEMM matrix
# ----------------------------------------------------------------------------------------------
_GEMM_DEFAULTS = dict(B=1, H=None, W=1, Cin=32, N=64, taps=((0, 0),), OH=None, OW=None, sy=1, sx=1, up=0, bmod=0,
                      act=_lib.ACT_NONE, res=False, rowvec=False, alpha=1.0, accumulate=False, out="f32", planes_out=2, dual=0,
                      a_planes=2, bias=True, bn=None, splitk=1, pad_cols=0, phase=False, m3=False, qkv=None)

# name -> descriptor.  m3: M sized for >= 3 tiles per CTA on every SM with a ragged last M tile (B = W = 1);
# qkv = (Cc, Bt): Q|K|V projection of Bt sequences of H tokens (N = 3 Cc, Cin = Cc); dual = planes of the dual output;
# phase: output rows 2 oh + 1 of 2 OH + 1 (a polyphase transposed-convolution phase; the other rows stay untouched).
GEMM_MATRIX = {
    # GEGLU body (N = 2 x output width)
    "geglu_b128_pair_a1": dict(Cin=64, N=256, act=GEGLU, bn=128, out="planes", planes_out=1, a_planes=1, m3=True),
    "geglu_b128_pair_a2": dict(H=300, Cin=48, N=512, act=GEGLU, bn=128, out="planes", planes_out=1, pad_cols=8),
    "geglu_b128_f32_a2": dict(Cin=32, N=256, act=GEGLU, bn=128, m3=True),
    "geglu_b128_p2_a1": dict(H=200, Cin=64, N=256, act=GEGLU, bn=128, out="planes", a_planes=1),
    "geglu_b64_p1_a1": dict(H=333, Cin=64, N=384, act=GEGLU, bn=64, out="planes", planes_out=1, a_planes=1),
    "geglu_b64_f32_a2": dict(B=2, H=10, W=7, Cin=24, N=128, taps=T3, act=GEGLU, bn=64, pad_cols=4),
    # compact fp32 body
    "f32n_b32_a1": dict(Cin=64, N=96, bn=32, res=True, a_planes=1, m3=True),
    "f32n_b32_a2": dict(H=250, Cin=40, N=64, bn=32, dual=2),
    "f32n_b64_a1": dict(B=2, H=40, Cin=32, N=128, taps=plan.taps_1d(3), bn=64, bias=False, a_planes=1, phase=True),
    "f32n_b64_a2": dict(B=2, H=16, W=8, Cin=16, N=64, taps=T3A, OH=8, OW=4, sy=2, sx=2, bn=64, res=True),
    "f32n_b128_a1": dict(H=300, Cin=128, N=256, bn=128, res=True, dual=1, a_planes=1),
    "f32n_b128_a2": dict(B=2, H=16, W=8, Cin=40, N=128, taps=T3, up=1, bn=128, pad_cols=8),
    # compact plane body, per-warp and pair stores
    "pln_b32_a1": dict(H=400, Cin=64, N=96, bn=32, out="planes", planes_out=1, a_planes=1, pad_cols=8),
    "pln_b32_a2": dict(Cin=32, N=64, bn=32, out="planes", res=True, m3=True),
    "pln_b64_a1": dict(H=300, Cin=64, N=128, bn=64, out="planes", planes_out=1, res=True, a_planes=1, pad_cols=8),
    "pln_b64_a2": dict(B=2, H=9, W=11, Cin=16, N=64, taps=T3, bn=64, out="planes"),
    "pln_b128_a1": dict(H=260, Cin=128, N=256, bn=128, out="planes", a_planes=1),
    # N % 128 == 64 with 128-wide tiles: full-line pair stores would write columns 192..255 of every row
    "pln_b128_a2_n192": dict(H=700, Cin=64, N=192, bn=128, out="planes", planes_out=1),
    "pln_b128_a1_n192_pad": dict(H=300, Cin=64, N=192, bn=128, out="planes", planes_out=1, a_planes=1, pad_cols=8),
    "pln_b64_pair_a1": dict(Cin=128, N=192, bn=64, out="planes", planes_out=1, a_planes=1, m3=True),
    "pln_b64_pair_a2": dict(B=4, H=12, W=4, Cin=8, N=64, taps=T3, bmod=2, bn=64, out="planes", planes_out=1, pad_cols=8),
    "pln_b128_pair_a1": dict(Cin=64, N=256, bn=128, out="planes", planes_out=1, a_planes=1, m3=True),
    "pln_b128_pair_a2": dict(H=515, Cin=64, N=128, bn=128, out="planes", planes_out=1, bias=False, pad_cols=8),
    # FAST body: row vector / alpha / accumulate / dual / QKV
    "fast_b32_a1": dict(B=2, H=20, W=6, Cin=24, N=64, taps=T3, bn=32, rowvec=True, res=True, a_planes=1),
    "fast_b32_a2": dict(B=2, H=333, Cin=32, N=32, taps=plan.taps_1d(11, 5), bn=32, res=True, alpha=1 / 3, accumulate=True),
    "fast_b64_a1": dict(H=300, Cin=64, N=128, bn=64, rowvec=True, out="planes", a_planes=1),
    "fast_b64_a2": dict(qkv=(64, 3), H=37, bn=64),
    "fast_b128_a1": dict(Cin=64, N=256, bn=128, rowvec=True, dual=2, a_planes=1, m3=True),
    "fast_b128_a2": dict(qkv=(128, 2), H=50, bn=128),
    "qk_b64_pair_a1": dict(qkv=(64, 3), bn=64, planes_out=1, a_planes=1, m3=True),
    "qk_b64_pair_a2": dict(qkv=(64, 2), H=77, bn=64, planes_out=1),
    "qk_b128_pair_a1": dict(qkv=(128, 2), bn=128, planes_out=1, a_planes=1, m3=True),
    "qk_b128_pair_a2": dict(qkv=(128, 3), H=37, bn=128, planes_out=1),
    # GENERIC body without split-K
    "gen_b32_a1_tanh": dict(Cin=32, N=1, taps=plan.taps_1d(7), bn=32, act=TANH, a_planes=1, m3=True),
    "gen_b32_a2_silu": dict(H=130, Cin=32, N=96, bn=32, act=SILU, out="planes"),
    "gen_b64_a1_geglu_res": dict(H=200, Cin=64, N=256, bn=64, act=GEGLU, res=True, a_planes=1),
    "gen_b64_a2_nchw": dict(B=2, H=16, W=8, Cin=32, N=64, taps=T3, OH=8, OW=4, sy=2, sx=2, bn=64, out="nchw"),
    "gen_b128_a1_silu_rowvec": dict(B=3, H=50, Cin=64, N=128, bn=128, act=SILU, rowvec=True, a_planes=1),
    "gen_b128_a2_geglu_res_planes": dict(H=150, Cin=32, N=256, bn=128, act=GEGLU, res=True, out="planes"),
    # split-K, coalesced reduction (splitk_reduce4_kernel)
    "sk4_b32_a1_f32": dict(B=2, H=8, W=4, Cin=64, N=64, taps=T3, bn=32, res=True, rowvec=True, a_planes=1, splitk=3),
    "sk4_b32_a2_planes": dict(H=100, Cin=256, N=96, bn=32, out="planes", splitk=4),
    "sk4_b64_a1_dual": dict(H=100, Cin=512, N=128, bn=64, res=True, dual=2, a_planes=1, splitk=5),
    "sk4_b64_a2_planes1": dict(B=2, H=6, W=6, Cin=64, N=128, taps=T3, bn=64, out="planes", planes_out=1, splitk=3),
    "sk4_b128_a1_planes": dict(H=90, Cin=640, N=256, bn=128, out="planes", a_planes=1, splitk=10),
    "sk4_b128_a2_f32": dict(B=2, H=8, W=2, Cin=640, N=640, taps=T3, bn=128, res=True, rowvec=True, splitk=16),
    # split-K, row-owner reduction with the full epilogue (splitk_epilogue_kernel)
    "skg_b32_a1_tanh": dict(B=2, H=300, Cin=32, N=32, taps=plan.taps_1d(7), bn=32, act=TANH, a_planes=1, splitk=3),
    "skg_b32_a2_alpha_acc": dict(B=2, H=200, Cin=64, N=64, taps=plan.taps_1d(3, 3), bn=32, res=True, alpha=1 / 3,
                                 accumulate=True, splitk=3),
    "skg_b64_a1_nchw": dict(B=2, H=8, W=8, Cin=64, N=64, taps=T3, bn=64, out="nchw", a_planes=1, splitk=4),
    "skg_b64_a2_geglu": dict(H=130, Cin=256, N=256, bn=64, act=GEGLU, out="planes", splitk=4),
    "skg_b128_a1_geglu_f32": dict(H=100, Cin=512, N=256, bn=128, act=GEGLU, a_planes=1, splitk=8),
    "skg_b128_a2_silu_p1": dict(H=64, Cin=384, N=128, bn=128, act=SILU, out="planes", planes_out=1, splitk=6),
}


@dataclass
class GemmCase:
    pl: plan.Plan
    s: dict
    a: Planes            # operand planes (written by the test)
    wm: torch.Tensor     # fp32 master weight [N, taps, Cp] (natural row order)
    bias: Optional[torch.Tensor]
    refs: dict           # input / output buffers
    M: int
    N: int
    n_out: int
    ldo: int
    geom: dict           # B, H, W, OH, OW, sy, sx, up, bmod, OHF, osy, ooy, taps, Hs, Ws, Bsrc


def plan_gemm(name: str, n_sm: int) -> GemmCase:
    s = dict(_GEMM_DEFAULTS, **GEMM_MATRIX[name])
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    geglu = s["act"] == GEGLU
    B, W, bn, taps = s["B"], s["W"], s["bn"], s["taps"]
    if s["qkv"]:
        Cc, Bt = s["qkv"]
        N, Cin = 3 * Cc, Cc
    else:
        N, Cin = s["N"], s["Cin"]
    n_out = N // 2 if geglu else N
    H = s["H"]
    if s["m3"]:
        tiles_m = math.ceil(3 * n_sm / (math.ceil(N / bn) * s["splitk"]))
        H = (tiles_m - 1) * 128 + 77
        if s["qkv"]:
            H = math.ceil(H / Bt)
            if (Bt * H) % 128 == 0:
                H += 1
    OH = H if s["OH"] is None else s["OH"]
    OW = W if s["OW"] is None else s["OW"]
    up, bmod = s["up"], s["bmod"]
    Hs, Ws = H >> up, W >> up
    Bsrc = bmod or B
    if s["qkv"]:
        B, H, OH = 1, Bt * H, Bt * H
        Hs = H
        Bsrc = 1
    M = B * OH * OW
    OHF, osy, ooy = (2 * OH + 1, 2, 1) if s["phase"] else (OH, 1, 0)
    out_rows = B * OHF * OW
    ldo = n_out + s["pad_cols"]

    P = Planner(splitk=False)
    T = len(taps)
    cp = round_up(Cin, 8)
    a = P.planes(Bsrc * Hs * Ws, Cin, s["a_planes"])
    wm = torch.zeros(N, T, cp)
    wm[:, :, :Cin] = torch.randn(N, T, Cin, generator=g) / math.sqrt(T * Cin)
    bias = 0.1 * torch.randn(N, generator=g) if s["bias"] else None
    w = P.wmat(wm.reshape(N, -1), bias, T, cp, geglu=geglu, bn=bn)
    kw = dict(B=B, H=H, W=W, taps=taps, OH=OH, OW=OW, sy=s["sy"], sx=s["sx"], up=up, bmod=bmod, act=s["act"],
              alpha=s["alpha"], accumulate=s["accumulate"], OHF=OHF, osy=osy, ooy=ooy)
    refs = {}
    if s["res"]:
        refs["res"] = P.raw(out_rows * n_out * 4)
        kw.update(res_ref=refs["res"], ld_res=n_out)
    if s["rowvec"]:
        refs["rowvec"] = P.raw(B * (n_out + 8) * 4)
        kw.update(rowvec=refs["rowvec"] + 16, ld_rowvec=n_out + 8)
    if s["qkv"]:
        ld_t = round_up(H // Bt, 8)
        qk = _guarded_planes(P, M, 2 * Cc, s["planes_out"])
        vhi = _guarded(P, Bt * Cc * ld_t * 2)
        vt = VT(vhi, _guarded(P, Bt * Cc * ld_t * 2) if s["planes_out"] == 2 else None, ld_t)
        refs.update(qk=qk, vt=vt)
        o = P.gemm(a, w, B=1, H=M, qkv=(qk, vt, 2 * Cc, H // Bt))
    elif s["out"] == "planes":
        op = _guarded_planes(P, out_rows, ldo, s["planes_out"])
        refs["planes"] = op
        o = P.gemm(a, w, out_planes=op, ldo=ldo, **kw)
    elif s["out"] == "nchw":
        refs["out"] = _guarded(P, B * N * OH * OW * 4)
        o = P.gemm(a, w, out_ref=refs["out"], out_mode=_lib.OUT_NCHW, **kw)
    else:
        refs["out"] = _guarded(P, out_rows * ldo * 4)
        dual = _guarded_planes(P, out_rows, ldo, s["dual"]) if s["dual"] else None
        refs["dual"] = dual
        o = P.gemm(a, w, out_ref=refs["out"], ldo=ldo, also_planes=dual, **kw)
    if s["splitk"] > 1:          # [splitk][Mpad][Npad] fp32 partial sums, then GUARD bytes that must stay zero
        o["splitk"], o["ws"] = s["splitk"], "SPLITK"
        P.splitk_ws_bytes = s["splitk"] * round_up(M, 128) * round_up(N, bn) * 4 + GUARD
    pl = P.finish({})
    geom = dict(B=B, H=H, W=W, OH=OH, OW=OW, sy=s["sy"], sx=s["sx"], up=up, bmod=bmod, OHF=OHF, osy=osy, ooy=ooy, taps=taps,
                Hs=Hs, Ws=Ws, Bsrc=Bsrc, out_rows=out_rows)
    return GemmCase(pl, s, a, wm, bias, refs, M, N, n_out, ldo, geom)


def _gemm_desc(c: GemmCase):
    """The case's aldm_gemm_desc, resolved against placeholder (aligned) base addresses: enough for the variant query."""
    arr = c.pl.resolve(1 << 32, 1 << 40)
    return arr[len(arr) - 1].u.gemm


# ---- the variant query covers the matrix (CPU) ----------------------------------------------
def _reachable_variants():
    """Every (bn, epi, a_planes, reduction, store) the selection in csrc/gemm.cu can return."""
    out = set()
    for ap in (1, 2):
        for bn in (32, 64, 128):
            out |= {(bn, _lib.EPI_F32N, ap, _lib.RED_NONE, _lib.STORE_COMPACT), (bn, _lib.EPI_PLN, ap, _lib.RED_NONE, _lib.STORE_COMPACT),
                    (bn, _lib.EPI_FAST, ap, _lib.RED_NONE, _lib.STORE_ROW)}
            out |= {(bn, _lib.EPI_GENERIC, ap, red, _lib.STORE_ROW) for red in (_lib.RED_NONE, _lib.RED_REDUCE4, _lib.RED_GENERIC)}
            if bn >= 64:        # GEGLU needs two 32-column halves; pair stores need whole 64-column groups
                out |= {(bn, _lib.EPI_GEGLU, ap, _lib.RED_NONE, _lib.STORE_ROW), (bn, _lib.EPI_PLN, ap, _lib.RED_NONE, _lib.STORE_PAIR_PLN),
                        (bn, _lib.EPI_FAST, ap, _lib.RED_NONE, _lib.STORE_PAIR_QK)}
        out.add((128, _lib.EPI_GEGLU, ap, _lib.RED_NONE, _lib.STORE_PAIR_GEGLU))
    return out


def test_gemm_matrix_reaches_every_variant():
    _lib.build()
    seen, long_epi, long_store = {}, set(), set()
    for name in GEMM_MATRIX:
        c = plan_gemm(name, plan.H100_SMS)
        d = _gemm_desc(c)
        v = _lib.gemm_variant(d)
        assert v[0] == c.s["bn"] and v[2] == c.s["a_planes"], (name, v)
        seen.setdefault(v, name)
        tiles = math.ceil(c.M / 128) * math.ceil(c.N / d.bn) * d.splitk
        if tiles >= 3 * plan.H100_SMS and c.M % 128:
            long_epi.add(v[1]); long_store.add(v[4])
    missing = _reachable_variants() - set(seen)
    assert not missing, f"variants no case reaches: {sorted(missing)}"
    assert set(seen) <= _reachable_variants(), sorted(set(seen) - _reachable_variants())
    assert long_epi == {_lib.EPI_FAST, _lib.EPI_GEGLU, _lib.EPI_GENERIC, _lib.EPI_F32N, _lib.EPI_PLN}, long_epi
    assert {_lib.STORE_PAIR_PLN, _lib.STORE_PAIR_GEGLU, _lib.STORE_PAIR_QK, _lib.STORE_COMPACT, _lib.STORE_ROW} <= long_store
    # pair stores do not check columns: N = 192 with 128-wide tiles must take the per-warp stores
    assert _lib.gemm_variant(_gemm_desc(plan_gemm("pln_b128_a2_n192", plan.H100_SMS)))[4] == _lib.STORE_COMPACT


def test_gemm_variant_rejects_bad_descriptors():
    _lib.build()
    d = _gemm_desc(plan_gemm("pln_b32_a1", plan.H100_SMS))
    d.bn = 48
    with pytest.raises(RuntimeError, match="bn=48"):
        _lib.gemm_variant(d)
    d.bn, d.impl = 32, _lib.GEMM_SIMT
    with pytest.raises(RuntimeError, match="SIMT"):
        _lib.gemm_variant(d)


# ---- float64 reference ------------------------------------------------------------------------
def _gather(a64: torch.Tensor, gm: dict, M: int) -> torch.Tensor:
    """[Bsrc*Hs*Ws, Cp] operand -> [M, taps*Cp], the implicit-GEMM A matrix (zero outside the input)."""
    dev = a64.device
    m = torch.arange(M, device=dev)
    ow, t = m % gm["OW"], m // gm["OW"]
    oh, b = t % gm["OH"], t // gm["OH"]
    bs = b % gm["bmod"] if gm["bmod"] else b
    cols = []
    for dy, dx in gm["taps"]:
        ih, iw = oh * gm["sy"] + dy, ow * gm["sx"] + dx
        ok = (ih >= 0) & (ih < gm["H"]) & (iw >= 0) & (iw < gm["W"])
        src = (bs * gm["Hs"] + (ih.clamp(0, gm["H"] - 1) >> gm["up"])) * gm["Ws"] + (iw.clamp(0, gm["W"] - 1) >> gm["up"])
        cols.append(a64[src] * ok[:, None])
    return torch.stack(cols, 1).reshape(M, -1)


def _gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def _orows(gm: dict, M: int) -> torch.Tensor:
    m = torch.arange(M)
    ow, t = m % gm["OW"], m // gm["OW"]
    oh, b = t % gm["OH"], t // gm["OH"]
    return (b * gm["OHF"] + oh * gm["osy"] + gm["ooy"]) * gm["OW"] + ow


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GEMM_MATRIX))
def test_gemm_matrix(name):
    c = plan_gemm(name, _n_sm())
    s, gm, M, N, n_out, ldo = c.s, c.geom, c.M, c.N, c.n_out, c.ldo
    g = torch.Generator().manual_seed(1000 + sum(map(ord, name)))
    op = c.pl.ops[-1]
    writes, wins, zero, scratch = [], [], [], []
    # operand planes as the kernel reads them (channels [Cin, Cp) are zero, as the prep kernels write them)
    cin = s["qkv"][0] if s["qkv"] else s["Cin"]
    x = torch.zeros(c.a.rows, c.a.Cp)
    x[:, :cin] = torch.randn(c.a.rows, cin, generator=g)
    hi = x.half()
    writes.append((c.a.hi.off, hi))
    a64 = hi.double()
    if c.a.lo is not None:
        lo = (x - hi.float()).half()
        writes.append((c.a.lo.off, lo))
        a64 = a64 + lo.double()
    out_rows = gm["out_rows"]
    res = torch.randn(out_rows, n_out, generator=g) if s["res"] else None
    if res is not None:
        writes.append((c.refs["res"].off, res))
    rv = torch.randn(gm["B"], n_out + 8, generator=g) if s["rowvec"] else None
    if rv is not None:
        writes.append((c.refs["rowvec"].off, rv))
    orow = _orows(gm, M)
    old = None
    if s["accumulate"]:
        old = torch.randn(out_rows, ldo, generator=g)
        writes.append((c.refs["out"].off, old))
    if op["splitk"] > 1:
        part = s["splitk"] * round_up(M, 128) * round_up(N, c.s["bn"]) * 4
        zero.append((op["ws"].off, part + GUARD))
        scratch.append((op["ws"].off, part))

    # reference (float64, on the device)
    d64 = dict(device=DEV, dtype=torch.float64)
    acc = _gather(a64.to(DEV), gm, M) @ c.wm.reshape(N, -1).to(**d64).t()
    if c.bias is not None:
        acc = acc + c.bias.to(**d64)
    if s["rowvec"]:
        b_of_m = torch.arange(M, device=DEV) // (gm["OH"] * gm["OW"])
        acc = acc + rv.to(**d64)[b_of_m, 4:4 + n_out]          # the descriptor points 16 bytes into each row
    if s["act"] == GEGLU:
        acc = acc[:, :n_out] * _gelu(acc[:, n_out:])
    elif s["act"] == TANH:
        acc = torch.tanh(acc)
    elif s["act"] == SILU:
        acc = acc * torch.sigmoid(acc)
    if res is not None:
        acc = acc + res.to(**d64)[orow.to(DEV)]
    acc = acc * float(np.float32(s["alpha"]))
    if old is not None:
        acc = acc + old.to(**d64)[orow.to(DEV), :n_out]

    checks = []           # (what, [hi window, lo window or None], reference, planes)

    def planes_check(what, p: Planes, n_rows, ld, cols, rows, want, n):
        wh = Win(p.hi.off, n_rows, ld, cols, 2, rows)
        wl = Win(p.lo.off, n_rows, ld, cols, 2, rows) if p.lo is not None else None
        wins.extend(w for w in (wh, wl) if w is not None)
        checks.append((what, [wh, wl], want, n))

    if s["qkv"]:
        Cc, Bt = s["qkv"]
        tpb = M // Bt
        vt = c.refs["vt"]
        want_v = torch.zeros(Bt, Cc, vt.ld_t, **d64)          # padding keys [tpb, ld_t) must come out exactly zero
        want_v[:, :, :tpb] = acc[:, 2 * Cc:].reshape(Bt, tpb, Cc).permute(0, 2, 1)
        planes_check("qk", c.refs["qk"], M, 2 * Cc, 2 * Cc, None, acc[:, :2 * Cc], s["planes_out"])
        planes_check("vt", Planes(vt.hi, vt.lo, Bt * Cc, vt.ld_t), Bt * Cc, vt.ld_t, vt.ld_t, None,
                     want_v.reshape(Bt * Cc, vt.ld_t), s["planes_out"])
    elif s["out"] == "planes":
        planes_check("planes", c.refs["planes"], out_rows, ldo, n_out, orow, acc, s["planes_out"])
    elif s["out"] == "nchw":
        n = gm["B"] * N * gm["OH"] * gm["OW"]
        wn = Win(c.refs["out"].off, 1, n, n, 4)
        wins.append(wn)
        checks.append(("nchw", [wn, None], acc.reshape(gm["B"], gm["OH"], gm["OW"], N).permute(0, 3, 1, 2), 0))
    else:
        wf = Win(c.refs["out"].off, out_rows, ldo, n_out, 4, orow)
        wins.append(wf)
        checks.append(("f32", [wf, None], acc, 0))
        if c.refs["dual"] is not None:
            planes_check("dual", c.refs["dual"], out_rows, ldo, n_out, orow, acc, s["dual"])

    prog = _run_guarded(c.pl, writes, wins, zero, scratch)
    for what, (wh, wl), want, planes in checks:
        got = wh.view(prog.ws).double()
        if wl is not None:
            got = got + wl.view(prog.ws).double()
        _check(f"{name}/{what}", got, want, planes)
    if s["qkv"]:
        Cc, Bt = s["qkv"]
        vt = c.refs["vt"]
        for p in (vt.hi, vt.lo):
            if p is not None:
                pad = Win(p.off, Bt * Cc, vt.ld_t, vt.ld_t, 2).view(prog.ws)[:, M // Bt:]
                assert bool((pad == 0).all()), f"{name}: V^T padding keys are not zero"


# ----------------------------------------------------------------------------------------------
# attention
# ----------------------------------------------------------------------------------------------
# name -> (B, heads, Nq, Nk, mask, kv_bmod, sigma of the Q / K entries).  mask: None; "rand" (~40 % of keys masked, key 0
# kept); "row" (kv batch 1 fully masked); "tile0" / "tile1" (keys [0, 64) / [64, 128) masked for every batch, the rest
# random).  sigma 6 gives scaled scores of magnitude ~50-100.  Nk <= 32 runs the short kernel; "_tc" forces the wgmma one.
ATTN_CASES = {
    "nk77_mask": (2, 2, 100, 77, "rand", 0, 1.0),
    "nk130_mask": (2, 2, 150, 130, "rand", 0, 1.0),
    "nk200_mask": (2, 2, 129, 200, "rand", 0, 1.0),
    "nk64_nq127": (2, 2, 127, 64, None, 0, 1.0),
    "nk65_nq128": (2, 2, 128, 65, None, 0, 1.0),
    "nk127_nq129": (2, 2, 129, 127, None, 0, 1.0),
    "nk128_mask": (2, 2, 128, 128, "rand", 0, 1.0),
    "nk129_nq127": (2, 2, 127, 129, "rand", 0, 1.0),
    "allmasked_row_nk40": (3, 2, 70, 40, "row", 0, 1.0),
    "allmasked_row_nk150": (3, 2, 70, 150, "row", 0, 1.0),
    "masked_tile0_nk150": (2, 2, 90, 150, "tile0", 0, 1.0),
    "masked_tile1_nk200": (2, 2, 90, 200, "tile1", 0, 1.0),
    "bmod_mask_nk90": (4, 2, 100, 90, "rand", 2, 1.0),
    "big_scores_nk256": (2, 2, 200, 256, None, 0, 6.0),
    "big_scores_mask_nk200": (2, 2, 130, 200, "rand", 0, 6.0),
    "big_scores_tile0_nk150": (2, 2, 130, 150, "tile0", 0, 6.0),
    "short8_mask": (2, 2, 150, 8, "rand", 0, 1.0),
    "short13_mask_bmod": (4, 2, 150, 13, "rand", 2, 1.0),
    "short32_row": (3, 2, 150, 32, "row", 0, 1.0),
    "short27_big": (2, 2, 140, 27, "rand", 0, 6.0),
    "short8_tc": (2, 2, 150, 8, "rand", 0, 1.0),
    "short16_tc_row": (3, 2, 150, 16, "row", 0, 1.0),
    "short32_tc_big": (2, 2, 150, 32, "rand", 0, 6.0),
    "self_nk150": (2, 2, 150, 150, None, 0, 1.0),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(ATTN_CASES))
def test_attention_matrix(name, monkeypatch):
    B, heads, Nq, Nk, mk, kv_bmod, sigma = ATTN_CASES[name]
    if name.endswith("_tc") or "_tc_" in name:
        monkeypatch.setenv("ALDM_ATTN_SHORT", "0")
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    Bkv = kv_bmod or B
    Cc = heads * 32
    selfattn = name.startswith("self")
    P = Planner()
    writes = []
    if selfattn:          # Q | K in one buffer (the QKV projection's layout): K at column offset Cc
        q = P.planes(B * Nq, 2 * Cc, 1)
        k, q_col, k_col = q, 0, Cc
        qk = (torch.randn(B * Nq, 2 * Cc, generator=g) * sigma).half()
        writes.append((q.hi.off, qk))
        qv, kv = qk[:, :Cc], qk[:, Cc:]
    else:
        q = P.planes(B * Nq, Cc, 1)
        k = P.planes(Bkv * Nk, Cc, 1)
        q_col = k_col = 0
        qv = (torch.randn(B * Nq, Cc, generator=g) * sigma).half()
        kv = (torch.randn(Bkv * Nk, Cc, generator=g) * sigma).half()
        writes += [(q.hi.off, qv), (k.hi.off, kv)]
    vt = P.vt(Bkv, Cc, Nk, 1)
    v = torch.zeros(Bkv, Cc, vt.ld_t)
    v[:, :, :Nk] = torch.randn(Bkv, Cc, Nk, generator=g)
    vh = v.half()
    writes.append((vt.hi.off, vh))
    mask_ref, keep = None, torch.ones(Bkv, Nk, dtype=torch.bool)
    if mk is not None:
        m = (torch.rand(Bkv, Nk, generator=g) > 0.4).float()
        m[:, 0] = 1
        if mk == "row":
            m[1] = 0
        elif mk == "tile0":
            m[:, :64] = 0
        elif mk == "tile1":
            m[:, 64:128] = 0
        mask_ref = P.raw(Bkv * Nk * 4)
        writes.append((mask_ref.off, m))
        keep = m == 1
    out = _guarded_planes(P, B * Nq, Cc, 1)
    P.attn(q, q_col, k, k_col, vt, out, B=B, heads=heads, Nq=Nq, Nk=Nk, mask=mask_ref, scale=32 ** -0.5, kv_bmod=kv_bmod)
    pl = P.finish({})
    win = Win(out.hi.off, B * Nq, Cc, Cc, 2)
    prog = _run_guarded(pl, writes, [win])
    got = win.view(prog.ws).double()

    # float64 softmax over the fp16 operands
    d64 = dict(device=DEV, dtype=torch.float64)
    bkv = torch.arange(B) % Bkv
    q4 = qv.to(**d64).reshape(B, Nq, heads, 32)
    k4 = kv.to(**d64).reshape(Bkv, Nk, heads, 32)[bkv]
    v4 = vh.to(**d64)[:, :, :Nk].reshape(Bkv, heads, 32, Nk)[bkv]                  # [B, h, d, k]
    sc = torch.einsum("bqhd,bkhd->bhqk", q4, k4) * float(np.float32(32 ** -0.5))
    sc = torch.where(keep.to(DEV)[bkv][:, None, None, :], sc, torch.full_like(sc, -FLT_MAX))
    p = torch.softmax(sc, dim=-1)
    want = torch.einsum("bhqk,bhdk->bqhd", p, v4).reshape(B * Nq, Cc)
    pv = torch.einsum("bhqk,bhdk->bqhd", p, v4.abs()).reshape(B * Nq, Cc)
    assert torch.isfinite(got).all(), f"{name}: non-finite output"
    err = (got - want).abs()
    bound = 2.0 ** -10 * (want.abs() + pv) + 1e-6
    rl2 = rel_l2(got, want)
    assert rl2 < 5e-4, f"{name}: relative L2 {rl2:.3e}"
    bad = (err > bound).nonzero()
    assert bad.numel() == 0, (f"{name}: {bad.shape[0]} elements over the bound; first (row, col) {bad[0].tolist()}: "
                              f"got {float(got[tuple(bad[0])]):.6g} want {float(want[tuple(bad[0])]):.6g}")


# ----------------------------------------------------------------------------------------------
# GroupNorm statistics on offset inputs
# ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("ratio", [30, 100])
@pytest.mark.parametrize("B,HW,C,c1", [(2, 4096, 128, 0), (80, 2048, 128, 0), (16, 64, 640, 256), (3, 1000, 256, 0),
                                       (2, 300, 1280, 0), (4, 1024, 640, 0), (3, 50, 96, 32)])
def test_groupnorm_offset(B, HW, C, c1, ratio):
    """GN+SiLU (two planes) and GN (one plane) of x = std * (z + ratio), z standardised over every (batch, group), so that
    each group has |mean| / std = ratio (asserted), through the
    single-pass, column-owner and generic statistics kernels (C = 96: 3 channels per group); c1 > 0 reads the concat of two
    sources.  Statistics in float64 over each (batch, group)."""
    g = torch.Generator().manual_seed(ratio + C + B)
    P = Planner()
    c0 = C - c1
    a = F32(P.raw(B * HW * c0 * 4), B * HW, c0)
    a2 = F32(P.raw(B * HW * c1 * 4), B * HW, c1) if c1 else None
    gam_t = 1 + 0.1 * torch.randn(C, generator=g)
    bet_t = 0.1 * torch.randn(C, generator=g)
    gam, bet = P.vec(gam_t), P.vec(bet_t)
    o1 = _guarded_planes(P, B * HW, C, 2)
    o2 = _guarded_planes(P, B * HW, C, 1)
    P.prep(_lib.PREP_GN_SILU, a, a2, gam, bet, eps=1e-5, B=B, HW=HW, out=o1)
    P.prep(_lib.PREP_GN, a, a2, gam, bet, eps=1e-6, B=B, HW=HW, out=o2)
    pl = P.finish({})
    std = 2.0
    z = torch.randn(B, HW, 32, C // 32, generator=g, dtype=torch.float64)
    z = (z - z.mean(dim=(1, 3), keepdim=True)) / z.std(dim=(1, 3), correction=0, keepdim=True)       # per (batch, group)
    x = (std * (z + ratio)).float().reshape(B * HW, C)
    xg = x.double().reshape(B, HW, 32, C // 32)
    reached = xg.mean(dim=(1, 3)).abs() / xg.std(dim=(1, 3), correction=0)
    assert float(reached.min()) > 0.99 * ratio, f"offset ratio reached {float(reached.min()):.1f} < {ratio}"
    writes = [(a.ref.off, x[:, :c0].contiguous())]
    if c1:
        writes.append((a2.ref.off, x[:, c0:].contiguous()))
    scr = sorted({op["scratch"].off for op in pl.ops if op.get("scratch") is not None})
    zero = [(off, Planner.gn_scratch_bytes(B)) for off in scr]
    wins = [Win(o1.hi.off, B * HW, C, C, 2), Win(o1.lo.off, B * HW, C, C, 2), Win(o2.hi.off, B * HW, C, C, 2)]
    prog = _run_guarded(pl, writes, wins, zero, zero)

    xd = x.to(DEV, torch.float64).reshape(B, HW, 32, C // 32)
    mean = xd.mean(dim=(1, 3), keepdim=True)
    var = (xd - mean).pow(2).mean(dim=(1, 3), keepdim=True)
    gd, bd = gam_t.to(DEV, torch.float64), bet_t.to(DEV, torch.float64)
    for eps, act, w_hi, w_lo, planes in ((1e-5, True, wins[0], wins[1], 2), (1e-6, False, wins[2], None, 1)):
        rstd = 1.0 / torch.sqrt(var + float(np.float32(eps)))
        y = ((xd - mean) * rstd).reshape(B * HW, C) * gd + bd
        if act:
            y = y * torch.sigmoid(y)
        apply_err = 2.0 ** -21 * (xd.abs() * rstd).reshape(B * HW, C) * gd.abs()
        got = w_hi.view(prog.ws).double() + (w_lo.view(prog.ws).double() if w_lo is not None else 0)
        _check(f"GN B={B} HW={HW} C={C} ratio={ratio} planes={planes}", got, y, planes, apply_err)
    first = [w.view(prog.ws).clone() for w in wins]
    prog.run("all")           # the self-resetting tickets: a second run computes the same
    torch.cuda.synchronize()
    for w, f in zip(wins, first):
        assert torch.equal(w.view(prog.ws), f), "second run differs"
