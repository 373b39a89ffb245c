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
  * fp32 and two-plane outputs: relative L2 < 2e-5 + ||T|| / ||ref||; |err| <= 1e-4 rms(ref) + T.  The 2^-22 operand split and the
    rounding of the fp32 partial sums cost about sqrt(K) 2^-24 |partial sum| (< 1e-5 rms(ref) at K = 11520).  T is the
    accumulation in the tensor cores, which truncates instead of rounding (Fasi, Higham, Mikaitis and Pranesh, "Numerical
    behavior of NVIDIA tensor cores", PeerJ CS 2021): every k16 wgmma step of every pass (3 passes with two A planes,
    2 with one) may drop up to one ulp, 2^-23 |partial sum|, always towards zero, so the error grows with K, not sqrt(K).
    The partial sums of a product sum are on the scale of |g| + rms(g) (g the GEMM sum, rms over the rows compared
    together), so T = steps 2^-23 (|g| + rms(g)) with steps = passes * Kpad / (16 splitk), times the epilogue's slope
    (SiLU 1.1, tanh 1, GEGLU |gelu(gate)| for the value and 1.13 |value| for the gate) and |alpha|.  Measured on an H100
    at K = 4224 to 11520 (fp32 outputs, values up to 5 rms): errors of up to 0.21 T, all towards zero, and relative L2
    of up to 4e-5 at K = 11520, where ||T|| / ||ref|| is about 5e-4; a wrong element is off by ~rms(ref), while
    T <= 2e-3 (|g| + rms(g)) at K = 11520.  (The single-plane bounds below are unchanged, plus T.)
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
CHECK_CHUNK = 1 << 28      # workspace bytes compared at a time: a whole-workspace copy and masks would not fit beside a 2 GB output


@dataclass
class Win:
    """Output window: `rows` (None: all) of a [n_rows, ld] array of `esz`-byte elements at byte `off`, columns [0, cols)."""
    off: int
    n_rows: int
    ld: int
    cols: int
    esz: int
    rows: Optional[torch.Tensor] = None

    def full(self, ws: torch.Tensor) -> torch.Tensor:
        dt = {4: torch.float32, 2: torch.float16}[self.esz]
        return ws[self.off:self.off + self.n_rows * self.ld * self.esz].view(dt).view(self.n_rows, self.ld)

    def view(self, ws: torch.Tensor) -> torch.Tensor:
        full = self.full(ws)
        return (full if self.rows is None else full[self.rows.to(ws.device)])[:, :self.cols]

    def mark(self, mask: torch.Tensor, c0: int = 0):
        """mask holds workspace bytes [c0, c0 + mask.numel()): set those inside the window."""
        rb = self.ld * self.esz
        a, b = max(c0, self.off), min(c0 + mask.numel(), self.off + self.n_rows * rb)
        if a >= b:
            return
        r0, r1 = (a - self.off) // rb, (b - self.off + rb - 1) // rb
        t = torch.zeros(r1 - r0, rb, dtype=torch.bool, device=mask.device)
        if self.rows is None:
            t[:, :self.cols * self.esz] = True
        else:
            sel = torch.zeros(self.n_rows, dtype=torch.bool, device=mask.device)
            sel[self.rows.to(mask.device)] = True
            t[sel[r0:r1], :self.cols * self.esz] = True
        s = self.off + r0 * rb
        mask[a - c0:b - c0] |= t.reshape(-1)[a - s:b - s]


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
    prog.run("all")
    torch.cuda.synchronize()

    def before(c0: int, c1: int) -> torch.Tensor:      # the workspace as it was before the run, rebuilt chunk by chunk
        exp = torch.full((c1 - c0,), 0xFF, dtype=torch.uint8, device=ws.device)
        for off, n in zero:
            if max(off, c0) < min(off + n, c1):
                exp[max(off, c0) - c0:min(off + n, c1) - c0] = 0
        for off, t in writes:
            b = t.contiguous().view(torch.uint8).reshape(-1)
            lo, hi = max(off, c0), min(off + b.numel(), c1)
            if lo < hi:
                exp[lo - c0:hi - c0] = b[lo - off:hi - off].to(ws.device)
        return exp

    _assert_unchanged(ws, before, wins, scratch)
    return prog


def _assert_unchanged(ws: torch.Tensor, before, wins, scratch=()):
    """Every byte of `ws` outside the windows and the scratch regions equals `before` (a tensor of the same size, or a
    function (c0, c1) -> its bytes [c0, c1)).  Compared in chunks of CHECK_CHUNK bytes."""
    n_stray, first = 0, None
    for c0 in range(0, ws.numel(), CHECK_CHUNK):
        c1 = min(ws.numel(), c0 + CHECK_CHUNK)
        inside = torch.zeros(c1 - c0, dtype=torch.bool, device=ws.device)
        for w in wins:
            w.mark(inside, c0)
        for off, n in scratch:
            if max(off, c0) < min(off + n, c1):
                inside[max(off, c0) - c0:min(off + n, c1) - c0] = True
        exp = before[c0:c1] if isinstance(before, torch.Tensor) else before(c0, c1)
        stray = ((ws[c0:c1] != exp) & ~inside).nonzero().flatten()
        if stray.numel():
            n_stray += stray.numel()
            first = c0 + int(stray[0]) if first is None else first
    if n_stray:
        where = None
        for w in wins:
            rel = first - w.off
            if 0 <= rel < w.n_rows * w.ld * w.esz:        # inside the array but outside the window: a padding column
                where = f"row {rel // (w.ld * w.esz)}, column {rel % (w.ld * w.esz) // w.esz} of the [{w.n_rows}, {w.ld}] " \
                        f"array at {w.off} (window: columns < {w.cols})"
        if where is None:
            near = min(wins, key=lambda w: abs(first - w.off - w.n_rows * w.ld * w.esz))
            where = f"{first - near.off - near.n_rows * near.ld * near.esz:+d} bytes past the end of the array at {near.off}"
        raise AssertionError(f"{n_stray} bytes changed outside the output windows; first at workspace byte {first}: "
                             f"{where}; scratch regions (first, last byte): {[(o, o + n - 1) for o, n in scratch]}")


class _Errors:
    """The bounds of _check, accumulated over an output compared in chunks: the per-element bound's rms(ref) term is
    known only at the end, so each chunk keeps its largest error in excess of the |ref|-proportional terms."""

    def __init__(self, name: str, planes: int, extra_in_rl2: bool = False):
        """extra_in_rl2: the per-element extra term is an error the kernel may make everywhere, so its norm over
        the reference's is added to the relative L2 budget as well."""
        self.name, self.planes, self.extra_in_rl2 = name, planes, extra_in_rl2
        self.se = self.sr = self.sx = 0.0
        self.n = 0
        self.worst = None          # (excess, flat index, got, want, |ref|-proportional bound)

    def add(self, got: torch.Tensor, ref: torch.Tensor, extra: Optional[torch.Tensor] = None):
        got, ref = got.double().reshape(-1), ref.double().reshape(-1).to(got.device)
        assert torch.isfinite(got).all(), f"{self.name}: non-finite output"
        err = (got - ref).abs()
        rel = 2.0 ** -10 * ref.abs() if self.planes == 1 else torch.zeros_like(ref)
        if extra is not None:
            extra = extra.double().reshape(-1).to(got.device)
            rel = rel + extra
            self.sx += float(extra.pow(2).sum())
        ex = err - rel
        i = int(ex.argmax())
        if self.worst is None or float(ex[i]) > self.worst[0]:
            self.worst = (float(ex[i]), self.n + i, float(got[i]), float(ref[i]), float(rel[i]))
        self.se += float(err.pow(2).sum())
        self.sr += float(ref.pow(2).sum())
        self.n += ref.numel()

    def finish(self):
        rl2 = math.sqrt(self.se) / (math.sqrt(self.sr) + 1e-30)
        tol = (3e-4 if self.planes == 1 else 2e-5) + (math.sqrt(self.sx / self.sr) if self.extra_in_rl2 else 0.0)
        assert rl2 < tol, f"{self.name}: relative L2 {rl2:.3e} >= {tol:.3e}"
        absb = (1e-5 if self.planes == 1 else 1e-4) * math.sqrt(self.sr / self.n)
        ex, i, got, want, rel = self.worst
        assert ex <= absb, f"{self.name}: element over the bound; worst flat index {i}: got {got:.6g} want {want:.6g} " \
                           f"bound {rel + absb:.3g}"


def _check(name: str, got: torch.Tensor, ref: torch.Tensor, planes: int, extra: Optional[torch.Tensor] = None):
    """planes: 0 fp32 output, 2 two-plane output, 1 single fp16 plane; extra: per-element term added to the bound."""
    e = _Errors(name, planes)
    e.add(got, ref, extra)
    e.finish()


# ----------------------------------------------------------------------------------------------
# GEMM matrix
# ----------------------------------------------------------------------------------------------
_GEMM_DEFAULTS = dict(B=1, H=None, W=1, Cin=32, N=64, taps=((0, 0),), OH=None, OW=None, sy=1, sx=1, up=0, bmod=0,
                      act=_lib.ACT_NONE, res=False, rowvec=False, alpha=1.0, accumulate=False, out="f32", planes_out=2, dual=0,
                      a_planes=2, bias=True, bn=None, splitk=1, pad_cols=0, phase=False, m3=False, qkv=None,
                      n_split=None, ophase=None, res_pad=0, ld_rowvec=None, rowvec_col=4, static_b=True)

# name -> descriptor.  m3: M sized for >= 3 tiles per CTA on every SM with a ragged last M tile (B = W = 1);
# qkv = (Cc, Bt): Q|K|V projection of Bt sequences of H tokens (N = 3 Cc, Cin = Cc; with n_split set, N and Cin are the
# spec's and columns >= n_split are the transposed part: the K|V projection of a cross-attention context);
# dual = planes of the dual output;
# phase: output rows 2 oh + 1 of 2 OH + 1 (a polyphase transposed-convolution phase; the other rows stay untouched);
# ophase = (OHF, osy, ooy): the general form, output rows osy oh + ooy of OHF;
# rowvec: a row vector per batch image, read at column rowvec_col of a row of ld_rowvec floats (default n_out + 8);
# res_pad: ld_res = n_out + res_pad; static_b = False: the weights are planned as a dynamic operand (no GEMM_STATIC_B).
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


def plan_gemm(name: str, n_sm: int, spec: Optional[dict] = None) -> GemmCase:
    """The case `name` of GEMM_MATRIX (or `spec`, under that name)."""
    s = dict(_GEMM_DEFAULTS, **(GEMM_MATRIX[name] if spec is None else spec))
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    geglu = s["act"] == GEGLU
    B, W, bn, taps = s["B"], s["W"], s["bn"], s["taps"]
    n_split = None
    if s["qkv"]:
        Cc, Bt = s["qkv"]
        N, Cin, n_split = (3 * Cc, Cc, 2 * Cc) if s["n_split"] is None else (s["N"], s["Cin"], s["n_split"])
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
    OHF, osy, ooy = (2 * OH + 1, 2, 1) if s["phase"] else (s["ophase"] or (OH, 1, 0))
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
    ld_res = n_out + s["res_pad"]
    ld_rowvec = n_out + 8 if s["ld_rowvec"] is None else s["ld_rowvec"]
    if s["res"]:
        refs["res"] = P.raw(out_rows * ld_res * 4)
        kw.update(res_ref=refs["res"], ld_res=ld_res)
    if s["rowvec"]:
        assert s["rowvec_col"] + n_out <= ld_rowvec
        refs["rowvec"] = P.raw(B * ld_rowvec * 4)
        kw.update(rowvec=refs["rowvec"] + 4 * s["rowvec_col"], ld_rowvec=ld_rowvec)
    if s["qkv"]:
        ld_t = round_up(H // Bt, 8)
        Cv = N - n_split
        qk = _guarded_planes(P, M, n_split, s["planes_out"])
        vhi = _guarded(P, Bt * Cv * ld_t * 2)
        vt = VT(vhi, _guarded(P, Bt * Cv * ld_t * 2) if s["planes_out"] == 2 else None, ld_t)
        refs.update(qk=qk, vt=vt)
        o = P.gemm(a, w, B=1, H=M, qkv=(qk, vt, n_split, H // Bt))
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
    if not s["static_b"]:
        o["impl"] &= ~_lib.GEMM_STATIC_B
    pl = P.finish({})
    geom = dict(B=B, H=H, W=W, OH=OH, OW=OW, sy=s["sy"], sx=s["sx"], up=up, bmod=bmod, OHF=OHF, osy=osy, ooy=ooy, taps=taps,
                Hs=Hs, Ws=Ws, Bsrc=Bsrc, out_rows=out_rows, Cin=Cin, n_split=n_split, ld_res=ld_res, ld_rowvec=ld_rowvec)
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
REF_CHUNK_BYTES = 1 << 30        # float64 A rows gathered at a time: a whole 2M-row, K = 2304 operand would be 38 GB


def _gather(hi: torch.Tensor, lo: Optional[torch.Tensor], gm: dict, m0: int, m1: int) -> torch.Tensor:
    """Rows [m0, m1) of the implicit-GEMM A matrix [M, taps*Cp] in float64, from the operand planes [Bsrc*Hs*Ws, Cp] as
    the kernel reads them (hi + lo, or hi alone; zero outside the input)."""
    m = torch.arange(m0, m1, device=hi.device)
    ow, t = m % gm["OW"], m // gm["OW"]
    oh, b = t % gm["OH"], t // gm["OH"]
    bs = b % gm["bmod"] if gm["bmod"] else b
    cols = []
    for dy, dx in gm["taps"]:
        ih, iw = oh * gm["sy"] + dy, ow * gm["sx"] + dx
        ok = (ih >= 0) & (ih < gm["H"]) & (iw >= 0) & (iw < gm["W"])
        src = (bs * gm["Hs"] + (ih.clamp(0, gm["H"] - 1) >> gm["up"])) * gm["Ws"] + (iw.clamp(0, gm["W"] - 1) >> gm["up"])
        v = hi[src].double()
        if lo is not None:
            v += lo[src].double()
        cols.append(v * ok[:, None])
    return torch.stack(cols, 1).reshape(m1 - m0, -1)


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
    x = torch.zeros(c.a.rows, c.a.Cp)
    x[:, :gm["Cin"]] = torch.randn(c.a.rows, gm["Cin"], generator=g)
    hi = x.half()
    writes.append((c.a.hi.off, hi))
    if c.a.lo is not None:
        writes.append((c.a.lo.off, (x - hi.float()).half()))
    del x, hi
    out_rows = gm["out_rows"]
    res = torch.randn(out_rows, gm["ld_res"], generator=g) if s["res"] else None
    if res is not None:
        writes.append((c.refs["res"].off, res))
    rv = torch.randn(gm["B"], gm["ld_rowvec"], generator=g) if s["rowvec"] else None
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

    checks = []           # (what, hi window, lo window or None, planes)

    def planes_win(what, p: Planes, n_rows, ld, cols, rows, n):
        checks.append((what, Win(p.hi.off, n_rows, ld, cols, 2, rows), Win(p.lo.off, n_rows, ld, cols, 2, rows)
                       if p.lo is not None else None, n))

    if s["qkv"]:
        Bt, n_split = s["qkv"][1], gm["n_split"]
        Cv, tpb, vt = N - n_split, M // Bt, c.refs["vt"]
        planes_win("qk", c.refs["qk"], M, n_split, n_split, None, s["planes_out"])
        planes_win("vt", Planes(vt.hi, vt.lo, Bt * Cv, vt.ld_t), Bt * Cv, vt.ld_t, vt.ld_t, None, s["planes_out"])
    elif s["out"] == "planes":
        planes_win("planes", c.refs["planes"], out_rows, ldo, n_out, orow, s["planes_out"])
    elif s["out"] == "nchw":
        n = gm["B"] * N * gm["OH"] * gm["OW"]
        checks.append(("nchw", Win(c.refs["out"].off, 1, n, n, 4), None, 0))
    else:
        checks.append(("f32", Win(c.refs["out"].off, out_rows, ldo, n_out, 4, orow), None, 0))
        if c.refs["dual"] is not None:
            planes_win("dual", c.refs["dual"], out_rows, ldo, n_out, orow, s["dual"])
    wins = [w for _, wh, wl, _ in checks for w in (wh, wl) if w is not None]
    prog = _run_guarded(c.pl, writes, wins, zero, scratch)
    del writes
    ws = prog.ws

    def got_rows(what, rows):
        _, wh, wl, _ = next(ch for ch in checks if ch[0] == what)
        r = rows.to(DEV)
        v = wh.full(ws)[r, :wh.cols].double()
        return v + wl.full(ws)[r, :wl.cols].double() if wl is not None else v

    # reference (float64, on the device) in chunks of output rows: whole V^T batches for QKV, whole images for NCHW
    d64 = dict(device=DEV, dtype=torch.float64)
    a_hi = Win(c.a.hi.off, c.a.rows, c.a.Cp, c.a.Cp, 2).full(ws)
    a_lo = Win(c.a.lo.off, c.a.rows, c.a.Cp, c.a.Cp, 2).full(ws) if c.a.lo is not None else None
    wt = c.wm.reshape(N, -1).to(**d64).t()
    bias = c.bias.to(**d64) if c.bias is not None else None
    unit = M // s["qkv"][1] if s["qkv"] else (gm["OH"] * gm["OW"] if s["out"] == "nchw" else 1)
    step = max(unit, REF_CHUNK_BYTES // (8 * (wt.shape[0] + 4 * N)) // unit * unit)
    errs = {what: _Errors(f"{name}/{what}", planes, extra_in_rl2=True) for what, _, _, planes in checks}
    steps = 4 * math.ceil(op["Kpad"] // 64 / op["splitk"]) * (3 if a_lo is not None else 2)
    for m0 in range(0, M, step):
        m1 = min(M, m0 + step)
        acc = _gather(a_hi, a_lo, gm, m0, m1) @ wt
        trunc = steps * 2.0 ** -23 * (acc.abs() + float(acc.pow(2).mean().sqrt()))   # T of the docstring
        if bias is not None:
            acc += bias
        if s["rowvec"]:
            b_of_m = torch.arange(m0, m1) // (gm["OH"] * gm["OW"])
            acc += rv[b_of_m, s["rowvec_col"]:s["rowvec_col"] + n_out].to(**d64)
        if s["act"] == GEGLU:
            trunc = trunc[:, :n_out] * _gelu(acc[:, n_out:]).abs() + 1.13 * acc[:, :n_out].abs() * trunc[:, n_out:]
            acc = acc[:, :n_out] * _gelu(acc[:, n_out:])
        elif s["act"] == TANH:
            acc = torch.tanh(acc)
        elif s["act"] == SILU:
            trunc *= 1.1
            acc = acc * torch.sigmoid(acc)
        trunc *= abs(float(np.float32(s["alpha"])))
        rows = orow[m0:m1]
        if res is not None:
            acc += res[rows, :n_out].to(**d64)
        acc *= float(np.float32(s["alpha"]))
        if old is not None:
            acc += old[rows, :n_out].to(**d64)
        if s["qkv"]:
            b0, b1 = m0 // tpb, m1 // tpb
            errs["qk"].add(got_rows("qk", torch.arange(m0, m1)), acc[:, :n_split], trunc[:, :n_split])
            want_v = torch.zeros(b1 - b0, Cv, vt.ld_t, **d64)          # padding keys [tpb, ld_t) must come out exactly zero
            want_v[:, :, :tpb] = acc[:, n_split:].reshape(b1 - b0, tpb, Cv).permute(0, 2, 1)
            t_v = torch.zeros_like(want_v)
            t_v[:, :, :tpb] = trunc[:, n_split:].reshape(b1 - b0, tpb, Cv).permute(0, 2, 1)
            errs["vt"].add(got_rows("vt", torch.arange(b0 * Cv, b1 * Cv)), want_v, t_v)
        elif s["out"] == "nchw":
            img = gm["OH"] * gm["OW"]
            got = checks[0][1].full(ws).view(gm["B"], N, gm["OH"], gm["OW"])[m0 // img:m1 // img]
            nchw = lambda t: t.reshape(-1, gm["OH"], gm["OW"], N).permute(0, 3, 1, 2)
            errs["nchw"].add(got, nchw(acc), nchw(trunc))
        else:
            for what, _, _, _ in checks:
                errs[what].add(got_rows(what, rows), acc, trunc)
        del acc, trunc
    for e in errs.values():
        e.finish()
    if s["qkv"]:
        for p in (vt.hi, vt.lo):
            if p is not None:
                pad = Win(p.off, Bt * Cv, vt.ld_t, vt.ld_t, 2).view(ws)[:, tpb:]
                assert bool((pad == 0).all()), f"{name}: V^T padding keys are not zero"


# ----------------------------------------------------------------------------------------------
# attention
# ----------------------------------------------------------------------------------------------
# name -> (B, heads, Nq, Nk, mask, kv_bmod, sigma of the Q / K entries).  mask: None; "rand" (~40 % of keys masked, key 0
# kept); "row" (kv batch 1 fully masked); "tile0" / "tile1" (keys [0, 64) / [64, 128) masked for every batch, the rest
# random); "tail" (the keys after a per-batch length masked, as in a padded context).  sigma 6 gives scaled scores of magnitude ~50-100.  Nk <= 32 runs the short kernel; "_tc" forces the wgmma one.
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
        elif mk == "tail":            # lengths 1 .. Nk, both ends included
            n = torch.randint(1, Nk + 1, (Bkv,), generator=g)
            n[0], n[-1] = Nk, 1
            m = (torch.arange(Nk)[None, :] < n[:, None]).float()
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
    x = torch.empty(B * HW, C)
    for b in range(B):        # image by image: the same draws as one [B, HW, 32, C / 32] tensor
        z = torch.randn(HW, 32, C // 32, generator=g, dtype=torch.float64)
        z = (z - z.mean(dim=(0, 2), keepdim=True)) / z.std(dim=(0, 2), correction=0, keepdim=True)      # per group
        x[b * HW:(b + 1) * HW] = (std * (z + ratio)).float().reshape(HW, C)
        xg = x[b * HW:(b + 1) * HW].double().reshape(HW, 32, C // 32)
        reached = xg.mean(dim=(0, 2)).abs() / xg.std(dim=(0, 2), correction=0)
        assert float(reached.min()) > 0.99 * ratio, f"offset ratio reached {float(reached.min()):.1f} < {ratio}"
    del z, xg
    writes = [(a.ref.off, x[:, :c0].contiguous())]
    if c1:
        writes.append((a2.ref.off, x[:, c0:].contiguous()))
    scr = sorted({op["scratch"].off for op in pl.ops if op.get("scratch") is not None})
    zero = [(off, Planner.gn_scratch_bytes(B)) for off in scr]
    wins = [Win(o1.hi.off, B * HW, C, C, 2), Win(o1.lo.off, B * HW, C, C, 2), Win(o2.hi.off, B * HW, C, C, 2)]
    prog = _run_guarded(pl, writes, wins, zero, zero)
    del writes

    # float64 statistics and outputs, one image at a time
    gd, bd = gam_t.to(DEV, torch.float64), bet_t.to(DEV, torch.float64)
    runs = ((1e-5, True, wins[0], wins[1], 2), (1e-6, False, wins[2], None, 1))
    errs = [_Errors(f"GN B={B} HW={HW} C={C} ratio={ratio} planes={planes}", planes) for *_, planes in runs]
    for b in range(B):
        r = slice(b * HW, (b + 1) * HW)
        xd = x[r].to(DEV, torch.float64).reshape(HW, 32, C // 32)
        mean = xd.mean(dim=(0, 2), keepdim=True)
        var = (xd - mean).pow(2).mean(dim=(0, 2), keepdim=True)
        for (eps, act, w_hi, w_lo, planes), e in zip(runs, errs):
            rstd = 1.0 / torch.sqrt(var + float(np.float32(eps)))
            y = ((xd - mean) * rstd).reshape(HW, C) * gd + bd
            if act:
                y = y * torch.sigmoid(y)
            apply_err = 2.0 ** -21 * (xd.abs() * rstd).reshape(HW, C) * gd.abs()
            got = w_hi.full(prog.ws)[r].double() + (w_lo.full(prog.ws)[r].double() if w_lo is not None else 0)
            e.add(got, y, apply_err)
            del y, apply_err, got
    for e in errs:
        e.finish()
    first = [w.view(prog.ws).clone() for w in wins]
    prog.run("all")           # the self-resetting tickets: a second run computes the same
    torch.cuda.synchronize()
    for w, f in zip(wins, first):
        assert torch.equal(w.view(prog.ws), f), "second run differs"
