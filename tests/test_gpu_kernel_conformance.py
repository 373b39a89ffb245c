"""Conformance of the remaining kernels (LayerNorm, elementwise prep, the VAE attention path, STFT, sampler kernels)
against float64 references, with the guard bands of tests/test_gpu_kernel_matrix.py; an inventory that maps every
__global__ kernel to its test; and PDL bit-identity of whole programs against serialized runs.

References are float64 and share nothing with tests/emulator.py or packing.pack_tiles.  Every case is checked by
relative L2 and by a per-element bound derived in the test's docstring; per-element terms scale with the magnitude the
kernel rounds or cancels (2^-24 per fp32 rounding of that magnitude), so a wrong statistic, index or coefficient is
not absorbed.  Outputs sit in 0xFF-filled workspaces with GUARD bytes around every region, and every byte outside the
declared output windows must be unchanged after one run.

Operand planes (csrc/common.cuh): y is saturated to +-65504, hi = fp16(y), lo = fp16(y - hi).  Two planes carry
|hi + lo - y| <= 2^-22 |y| + 2^-25 (the absolute floor is half the fp16 subnormal spacing: lo of a value below about 2^-3
is subnormal, hi of a value below 2^-14 too); one plane |hi - y| <= 2^-11 |y| + 2^-25.  PLANE_ERR gives both; a compute
error d before the split adds d (two planes) or 2 d (one plane: it can move y across a rounding boundary)."""
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from audioldm2_b200 import _lib, arch, engine, plan  # noqa: E402
from audioldm2_b200.packing import round_up  # noqa: E402
from audioldm2_b200.plan import F32, Planes, Planner  # noqa: E402
from tests.conftest import rel_l2  # noqa: E402
from tests.test_gpu_kernel_matrix import (DEV, GUARD, Win, _assert_unchanged, _check, _guarded, _guarded_planes,  # noqa: E402
                                          _n_sm, _run_guarded)

U = 2.0 ** -24            # unit roundoff of fp32


def _plane_err(ref: torch.Tensor, planes: int) -> torch.Tensor:
    return (2.0 ** -22 if planes == 2 else 2.0 ** -11) * ref.abs() + 2.0 ** -25


def _within(name: str, got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, rl2_tol: float):
    got, ref, bound = (t.double().reshape(-1).to(DEV) for t in (got, ref, bound))
    assert torch.isfinite(got).all(), f"{name}: non-finite output"
    rl2 = rel_l2(got, ref)
    assert rl2 < rl2_tol, f"{name}: relative L2 {rl2:.3e} >= {rl2_tol:.0e}"
    bad = ((got - ref).abs() > bound).nonzero().flatten()
    assert bad.numel() == 0, (f"{name}: {bad.numel()} elements over the bound; first flat index {int(bad[0])}: got "
                              f"{float(got[bad[0]]):.8g} want {float(ref[bad[0]]):.8g} bound {float(bound[bad[0]]):.3g}")


def _planes_of(ws: torch.Tensor, p: Planes, rows: int, cols: int):
    hi = Win(p.hi.off, rows, p.Cp, cols, 2).view(ws)
    lo = Win(p.lo.off, rows, p.Cp, cols, 2).view(ws) if p.lo is not None else None
    return hi, lo


def _planes_wins(p: Planes, rows: int, cols: int):
    return [Win(r.off, rows, p.Cp, cols, 2) for r in (p.hi, p.lo) if r is not None]


def _split_exact(y32: torch.Tensor):
    """The device split of fp32 values, with torch's round-to-nearest conversions."""
    y = y32.float().clamp(-65504.0, 65504.0)
    hi = y.half()
    return hi, (y - hi.float()).half()


class _Slab:
    """Workspace for the stand-alone entry points: regions with GUARD bytes between them, 0xFF-filled."""

    def __init__(self):
        self.top = GUARD
        self.writes = []

    def region(self, nbytes: int) -> int:
        off = self.top
        self.top = off + round_up(max(nbytes, 1), 256) + GUARD
        return off

    def put(self, t: torch.Tensor) -> int:
        off = self.region(t.numel() * t.element_size())
        self.writes.append((off, t))
        return off

    def run(self, fn, wins):
        ws = torch.full((self.top,), 0xFF, dtype=torch.uint8, device=DEV)
        for off, t in self.writes:
            b = t.contiguous().view(torch.uint8).reshape(-1)
            ws[off:off + b.numel()].copy_(b.to(DEV))
        before = ws.clone()
        base = ws.data_ptr()
        fn(lambda off: base + off, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        _assert_unchanged(ws, before, wins)
        return ws


def _flat(ws, off, n, dt=torch.float32):
    esz = torch.empty((), dtype=dt).element_size()
    return ws[off:off + n * esz].view(dt)


# ----------------------------------------------------------------------------------------------
# LayerNorm (ln_kernel<2|4|8, 1>)
# ----------------------------------------------------------------------------------------------
LN_C = [32, 96, 128, 256, 384, 640, 1024]


def _offset_rows(rows: int, C: int, g, ratios=(0, 30, 100)) -> torch.Tensor:
    """Row r: std * (z + ratio) with z standardised over the row and ratio = ratios[r % 3] (sign alternating);
    row 0 (when rows > 1) is the constant 0.75."""
    z = torch.randn(rows, C, generator=g, dtype=torch.float64)
    z = (z - z.mean(1, keepdim=True)) / z.std(1, correction=0, keepdim=True)
    ratio = torch.tensor([ratios[r % len(ratios)] * (-1) ** (r // 3) for r in range(rows)], dtype=torch.float64)
    x = (1.5 * (z + ratio[:, None])).float()
    if rows > 1:
        x[0] = 0.75
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("rows,C", [(1, c) for c in LN_C] + [(8 * 37 + 3, c) for c in LN_C] + [(65539, 128)])
def test_layernorm(rows, C):
    """LayerNorm to two planes (eps 1e-5) and one plane (eps 1e-6) of rows with |mean| / std of 0, 30 and 100 (asserted)
    and a constant row.  Reference: float64 layer_norm with eps rounded to fp32.

    Bound, per element (on top of PLANE_ERR and the 4 roundings of the fp32 apply, 2^-22 |y|):
      * the mean is an fp32 sum of C terms of magnitude |x| (two adds per float4, at most 8 float4 per lane, then a
        5-level shuffle tree: depth <= 15) divided by C, so |d mean| <= 16 u mean|x|; it shifts the output by
        d mean rstd |gamma|: 2^-20 mean|x| rstd |gamma| per element, doubled for margin;
      * rstd is the same kind of sum over (x - mean)^2 plus rsqrtf (2 ulp): relative error <= 2^-19, which scales the
        normalised term: 2^-19 |xhat gamma|.
    A constant row normalises to exactly 0: its output must be the split of beta, bit for bit."""
    g = torch.Generator().manual_seed(C + rows)
    P = Planner()
    a = F32(P.raw(rows * C * 4), rows, C)
    gam_t = 1 + 0.1 * torch.randn(C, generator=g)
    bet_t = 0.1 * torch.randn(C, generator=g)
    gam, bet = P.vec(gam_t), P.vec(bet_t)
    o2 = _guarded_planes(P, rows, C, 2)
    o1 = _guarded_planes(P, rows, C, 1)
    P.prep(_lib.PREP_LN, a, None, gam, bet, eps=1e-5, out=o2)
    P.prep(_lib.PREP_LN, a, None, gam, bet, eps=1e-6, out=o1)
    pl = P.finish({})
    x = _offset_rows(rows, C, g, ratios=(30,) if rows == 1 else (0, 30, 100))
    xd = x.to(DEV, torch.float64)
    mean = xd.mean(1, keepdim=True)
    var = (xd - mean).pow(2).mean(1, keepdim=True)
    if rows > 1:
        for ratio in (30, 100):
            sel = torch.arange(1, rows) % 3 == (1 if ratio == 30 else 2)
            sel = torch.cat([torch.tensor([False]), sel]).to(DEV)
            reached = mean[sel].abs() / var[sel].sqrt()
            assert float(reached.min()) > 0.99 * ratio, f"offset ratio reached {float(reached.min()):.1f} < {ratio}"
    else:
        assert float(mean.abs() / var.sqrt()) > 0.99 * 30
    wins = _planes_wins(o2, rows, C) + _planes_wins(o1, rows, C)
    prog = _run_guarded(pl, [(a.ref.off, x)], wins)
    gd, bd = gam_t.to(DEV, torch.float64), bet_t.to(DEV, torch.float64)
    for eps, o, planes in ((1e-5, o2, 2), (1e-6, o1, 1)):
        rstd = 1.0 / torch.sqrt(var + float(np.float32(eps)))
        xh = (xd - mean) * rstd
        y = xh * gd + bd
        hi, lo = _planes_of(prog.ws, o, rows, C)
        got = hi.double() + (lo.double() if lo is not None else 0)
        comp = 2.0 ** -19 * xd.abs().mean(1, keepdim=True) * rstd * gd.abs() + 2.0 ** -19 * (xh * gd).abs() \
            + 2.0 ** -22 * y.abs()
        bound = _plane_err(y, planes) + (1 if planes == 2 else 2) * comp
        _within(f"LN rows={rows} C={C} planes={planes}", got, y, bound, 2e-5 if planes == 2 else 3e-4)
        if rows > 1:
            bh, bl = _split_exact(bet_t)
            assert torch.equal(hi[0].cpu(), bh), f"LN C={C}: constant row: hi plane is not fp16(beta)"
            if lo is not None:
                assert torch.equal(lo[0].cpu(), bl), f"LN C={C}: constant row: lo plane is not fp16(beta - hi)"


# ----------------------------------------------------------------------------------------------
# elementwise prep (ew_kernel)
# ----------------------------------------------------------------------------------------------
EW_MODES = {"copy": (_lib.PREP_COPY, 0.0), "silu": (_lib.PREP_SILU, 0.0), "lrelu0.1": (_lib.PREP_LRELU, 0.1),
            "lrelu0.01": (_lib.PREP_LRELU, 0.01)}
# name -> (c0, c1, nchw): vector path (C % 8 == 0 and c0 % 8 == 0), scalar path, mixed (vector chunks then a scalar tail)
EW_SHAPES = {"c8": (8, 0, False), "c64": (64, 0, False), "c1": (1, 0, False), "c5": (5, 0, False), "c12": (12, 0, False),
             "c44": (44, 0, False), "cat64_32": (64, 32, False), "cat12_20": (12, 20, False), "cat64_4": (64, 4, False),
             "nchw1": (1, 0, True), "nchw8": (8, 0, True), "nchw5": (5, 0, True)}


def _ew_input(rows: int, C: int, g) -> torch.Tensor:
    """Standard normal * 4 with every 7th element beyond the fp16 range (+-7e4, +-1e5), every 11th below the fp16
    normal range (1e-5 .. 1e-8, both signs), and some exact zeros of both signs."""
    x = 4 * torch.randn(rows, C, generator=g)
    f = x.reshape(-1)
    n = f.numel()
    i = torch.arange(n)
    big = torch.tensor([7e4, -7e4, 1e5, -1e5, 65519.0, -65520.0])
    tiny = torch.tensor([1e-5, -3e-6, 6e-8, -2e-8, 1e-8, 5.9e-5])
    f[i % 7 == 3] = big[(i[i % 7 == 3] // 7) % len(big)]
    f[i % 11 == 5] = tiny[(i[i % 11 == 5] // 11) % len(tiny)]
    f[i % 29 == 17] = 0.0
    f[i % 31 == 19] = -0.0
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("shape", sorted(EW_SHAPES))
@pytest.mark.parametrize("mode", sorted(EW_MODES))
def test_prep_elementwise(mode, shape):
    """ew_kernel: copy / SiLU / leaky ReLU of one source, a concatenation of two, or an NCHW source, to two planes and to
    one plane; padding columns [C, Cp) must be exactly zero in every plane.

    COPY and LRELU are exact in fp32 (the leaky product is one fp32 multiply, as torch computes it): hi and lo must be
    fp16(sat(y)) and fp16(sat(y) - hi) bit for bit.  SiLU is __fdividef(x, 1 + __expf(-x)): __expf has at most
    2 + 1.173 |x| ulp (CUDA C Programming Guide, intrinsic functions), which perturbs the denominator 1 + e by
    e / (1 + e) times that relative error; the add, and __fdividef (2 ulp), add 3 ulp more; an ulp is at most 2^-23
    relative.  So |d silu| <= [(e / (1 + e)) (2 + 1.173 |x|) + 3] 2^-23 |silu|, added to PLANE_ERR (twice on one plane)."""
    m, slope = EW_MODES[mode]
    c0, c1, nchw = EW_SHAPES[shape]
    C = c0 + c1
    g = torch.Generator().manual_seed(sum(map(ord, mode + shape)))
    B, HW = 3, 37
    rows = B * HW
    P = Planner()
    s0 = F32(_guarded(P, rows * c0 * 4), rows, c0)
    s1 = F32(_guarded(P, rows * c1 * 4), rows, c1) if c1 else None
    Cp = round_up(C, 8)
    o2, o1 = _guarded_planes(P, rows, Cp, 2), _guarded_planes(P, rows, Cp, 1)
    for o in (o2, o1):
        P.prep(m, s0, s1, slope=slope, B=B, HW=HW, src_nchw=nchw, out=o)
    pl = P.finish({})
    x = _ew_input(rows, C, g)                         # channels-last view of the input [rows, C]
    if nchw:
        writes = [(s0.ref.off, x.reshape(B, HW, C).permute(0, 2, 1).contiguous())]
    else:
        writes = [(s0.ref.off, x[:, :c0].contiguous())] + ([(s1.ref.off, x[:, c0:].contiguous())] if c1 else [])
    wins = _planes_wins(o2, rows, Cp) + _planes_wins(o1, rows, Cp)
    prog = _run_guarded(pl, writes, wins)
    if mode == "silu":
        xd = x.double()
        y = (xd * torch.sigmoid(xd)).clamp(-65504.0, 65504.0)
        e = torch.exp(-xd)
        w = torch.where(torch.isinf(e), torch.ones_like(e), e / (1 + e))
        comp = (w * (2 + 1.173 * xd.abs()) + 3) * 2.0 ** -23 * y.abs()
    elif mode == "copy":
        y32 = x
    else:
        y32 = torch.where(x > 0, x, x * torch.tensor(slope, dtype=torch.float32))
    for o, planes in ((o2, 2), (o1, 1)):
        hi, lo = _planes_of(prog.ws, o, rows, Cp)
        for p in (hi, lo):
            if p is not None:
                assert bool((p[:, C:].view(torch.int16) == 0).all()), f"{mode}/{shape}: padding columns are not zero"
        hi, lo = hi[:, :C], (lo[:, :C] if lo is not None else None)
        if mode == "silu":
            got = hi.double() + (lo.double() if lo is not None else 0)
            bound = _plane_err(y, planes) + (1 if planes == 2 else 2) * comp
            _within(f"{mode}/{shape}/planes={planes}", got, y, bound, 2e-5 if planes == 2 else 3e-4)
        else:
            wh, wl = _split_exact(y32)
            assert torch.equal(hi.cpu().view(torch.int16), wh.view(torch.int16)), f"{mode}/{shape}: hi plane differs"
            if lo is not None:
                assert torch.equal(lo.cpu().view(torch.int16), wl.view(torch.int16)), f"{mode}/{shape}: lo plane differs"


# ----------------------------------------------------------------------------------------------
# VAE attention path: softmax_rows, pack_b, and the planner's _vae_attn
# ----------------------------------------------------------------------------------------------
def _softmax_bound(s: torch.Tensor, p: torch.Tensor, planes: int) -> torch.Tensor:
    """Per-element bound of softmax_rows_kernel on scaled scores s (float64, as the fp32 product x * scale rounds them:
    that rounding is inside the bound) against the float64 probabilities p.

    The kernel computes e_i = expf(fl(x_i scale) - mx) with mx the row maximum, s = sum e_i in fp32 (a sequential
    per-thread sum of n / 256 terms, a 5-level shuffle tree, 8 warp partials: depth n / 256 + 14), p_i = e_i * (1 / s).
    Relative error of p_i <= 2^-22 (expf, 2 ulp) + 2^-22 (the same in the terms of s) + (n / 256 + 16) u (the sum,
    the reciprocal, the product) + u (|s_i| + |mx| + |s_i - mx|) (rounding of the argument of exp_i) + the largest such
    argument term of the row (it enters through s).  Then PLANE_ERR: at n = 4096 a typical p is 2^-12, whose lo plane is
    an fp16 subnormal, so two planes hold it to 2^-25 absolute, not 2^-22 relative."""
    n = s.shape[-1]
    mx = s.max(-1, keepdim=True).values
    arg = U * (s.abs() + mx.abs() + (s - mx).abs())
    rel = 2.0 ** -21 + (n / 256 + 16) * U + arg + arg.max(-1, keepdim=True).values
    return _plane_err(p, planes) + (1 if planes == 2 else 2) * rel * p


def _softmax_rl2(p: torch.Tensor, planes: int) -> float:
    """Relative L2 budget of a softmax output: the planes' budget (2e-5 / 3e-4) plus the 2^-25 absolute floor over
    rms(p) -- at n = 4096 with flat rows (p ~ 2^-12 everywhere) that floor alone is ~2^-13 relative per element."""
    return (2e-5 if planes == 2 else 3e-4) + 2.0 ** -25 / float(p.pow(2).mean().sqrt())


SOFTMAX_N = [2, 34, 256, 4096]


@pytest.mark.gpu
@pytest.mark.parametrize("scale", [1.0, 0.125])
@pytest.mark.parametrize("n", SOFTMAX_N)
def test_softmax_rows(n, scale):
    """softmax_rows to two planes and to one plane.  Rows: normal scores, scores of magnitude 50-100 (N(0, 1) * 25 +- 75
    before the scale), a constant row, a row with one score 60 above the others.  Reference: float64 softmax of
    fp32 x times the fp32 scale; bound: _softmax_bound."""
    g = torch.Generator().manual_seed(n + int(8 * scale))
    rows = 13
    P = Planner()
    x_ref = _guarded(P, rows * n * 4)
    o2, o1 = _guarded_planes(P, rows, n, 2), _guarded_planes(P, rows, n, 1)
    for o in (o2, o1):
        P.ops.append(dict(kind="softmax", x=x_ref, out_hi=o.hi, out_lo=o.lo, rows=rows, n=n, scale=scale))
    pl = P.finish({})
    x = torch.randn(rows, n, generator=g)
    x[4:9] = x[4:9] * 25 + 75 * torch.sign(torch.randn(5, n, generator=g))
    x[9] = 0.75
    x[10] = torch.randn(n, generator=g)
    x[10, n // 3] += 60 / scale
    x[11] = -x[11].abs() * 40
    prog = _run_guarded(pl, [(x_ref.off, x)], _planes_wins(o2, rows, n) + _planes_wins(o1, rows, n))
    s = x.to(DEV, torch.float64) * float(np.float32(scale))
    assert float(s[4:9].abs().max()) > 50 / (8 if scale < 1 else 1)
    p = torch.softmax(s, dim=-1)
    for o, planes in ((o2, 2), (o1, 1)):
        hi, lo = _planes_of(prog.ws, o, rows, n)
        got = hi.double() + (lo.double() if lo is not None else 0)
        _within(f"softmax n={n} scale={scale} planes={planes}", got, p, _softmax_bound(s, p, planes), _softmax_rl2(p, planes))


def _packed_image(w: torch.Tensor, N: int, K: int, bn: int) -> torch.Tensor:
    """Tile image of the fp32 matrix w [N, K] as packing.py documents it, built element by element:
    packed[n_tile][k_blk][plane (hi, lo)][row r < bn][128 bytes], the 16-byte chunk j of row r (fp16 K-elements
    8 j .. 8 j + 7 of the k block) stored at chunk position j ^ (r & 7); rows >= N and K-elements >= K are zero."""
    Npad, Kpad = round_up(N, bn), round_up(K, 64)
    full = torch.zeros(Npad, Kpad)
    full[:N, :K] = w
    hi, lo = _split_exact(full)
    out = torch.zeros(Npad * Kpad * 2, dtype=torch.int16)
    n = torch.arange(Npad)[:, None].expand(Npad, Kpad)
    k = torch.arange(Kpad)[None, :].expand(Npad, Kpad)
    tile, r, kb, j, e = n // bn, n % bn, k // 64, (k % 64) // 8, k % 8
    for plane, v in ((0, hi), (1, lo)):
        idx = (((tile * (Kpad // 64) + kb) * 2 + plane) * bn + r) * 64 + (j ^ (r & 7)) * 8 + e
        out[idx.reshape(-1)] = v.view(torch.int16).reshape(-1)
    return out


# (N, K, bn, transpose, lds): N and K not multiples of bn or of 64, lds beyond the row length
PACKB_CASES = [(100, 72, 32, 0, 80), (130, 200, 64, 1, 136), (300, 70, 128, 0, 72), (77, 129, 128, 1, 84),
               (33, 65, 64, 0, 68), (1000, 40, 32, 1, 1003)]


@pytest.mark.gpu
@pytest.mark.parametrize("N,K,bn,transpose,lds", PACKB_CASES)
def test_pack_b(N, K, bn, transpose, lds):
    """pack_b_kernel: the tile image must equal _packed_image bit for bit (padding rows and K-elements zero) and the
    plain [Npad, Kpad] copy must be the matrix, exactly, with zero padding.  The source holds values beyond the fp16
    range and below its normal range."""
    g = torch.Generator().manual_seed(N * K + bn)
    P = Planner()
    rows_src = K if transpose else N
    src = _guarded(P, rows_src * lds * 4)
    Npad, Kpad = round_up(N, bn), round_up(K, 64)
    dp, dpl = _guarded(P, Npad * Kpad * 4), _guarded(P, Npad * Kpad * 4)
    P.ops.append(dict(kind="packb", src=src, dst_packed=dp, dst_plain=dpl, lds=lds, transpose=transpose, N=N, K=K, bn=bn))
    pl = P.finish({})
    s = torch.randn(rows_src, lds, generator=g)
    s[::5, ::3] *= 3e4
    s[1::7, ::2] *= 1e-6
    prog = _run_guarded(pl, [(src.off, s)], [Win(dp.off, 1, Npad * Kpad * 2, Npad * Kpad * 2, 2),
                                              Win(dpl.off, Npad, Kpad, Kpad, 4)])
    w = s[:, :N].t() if transpose else s[:, :K]
    want = _packed_image(w, N, K, bn)
    got = Win(dp.off, 1, Npad * Kpad * 2, Npad * Kpad * 2, 2).view(prog.ws).reshape(-1).view(torch.int16).cpu()
    assert torch.equal(got, want), f"tile image differs at {int((got != want).nonzero()[0])} (int16 index)"
    plain = torch.zeros(Npad, Kpad)
    plain[:N, :K] = w
    assert torch.equal(Win(dpl.off, Npad, Kpad, Kpad, 4).view(prog.ws).cpu(), plain), "plain copy differs"


def _attn_block_sd(Cc: int, g):
    n = "mid.attn_1"
    sd = {n + ".norm.weight": 1 + 0.1 * torch.randn(Cc, generator=g), n + ".norm.bias": 0.1 * torch.randn(Cc, generator=g)}
    for k in ("q", "k", "v", "proj_out"):
        sd[f"{n}.{k}.weight"] = torch.randn(Cc, Cc, 1, 1, generator=g) / math.sqrt(Cc)
        sd[f"{n}.{k}.bias"] = 0.1 * torch.randn(Cc, generator=g)
    return n, sd


def _plan_vae_attn(B: int, HW: int, Cc: int, seed: int):
    """The planner's own AttnBlock program (GroupNorm, q/k/v, per-batch pack_b + score GEMM + softmax_rows + pack_b +
    output GEMM, proj_out + residual) behind a leading guard; returns (plan, x, out, the input, the state dict)."""
    g = torch.Generator().manual_seed(seed)
    n, sd = _attn_block_sd(Cc, g)
    P = Planner()
    lead = P.raw(GUARD)
    x = F32(P.raw(B * HW * Cc * 4), B * HW, Cc)
    out = plan._vae_attn(P, sd, n, x, B, HW, Cc)
    pl = P.finish({})
    assert lead.off == 0
    xin = torch.randn(B * HW, Cc, generator=g) + 0.5
    return pl, x, out, xin, sd, n


def _attn_block_ref(xin: torch.Tensor, sd, n: str, B: int, HW: int, Cc: int) -> torch.Tensor:
    """AttnBlock.forward in float64 from the fp32 master weights: GroupNorm(32, eps 1e-6), 1x1 q/k/v, softmax of
    q k^T * Cc^-0.5 (the fp32 alpha of the score GEMM), o = P v, proj_out(o) + x."""
    d64 = dict(device=DEV, dtype=torch.float64)
    x = xin.to(**d64)
    xg = x.reshape(B, HW, 32, Cc // 32)
    mean = xg.mean(dim=(1, 3), keepdim=True)
    var = (xg - mean).pow(2).mean(dim=(1, 3), keepdim=True)
    h = ((xg - mean) / torch.sqrt(var + float(np.float32(1e-6)))).reshape(B * HW, Cc)
    h = h * sd[n + ".norm.weight"].to(**d64) + sd[n + ".norm.bias"].to(**d64)
    lin = {k: (sd[f"{n}.{k}.weight"].reshape(Cc, Cc).to(**d64), sd[f"{n}.{k}.bias"].to(**d64)) for k in ("q", "k", "v", "proj_out")}
    q, k, v = (h @ lin[t][0].t() + lin[t][1] for t in ("q", "k", "v"))
    alpha = float(np.float32(float(int(Cc) ** -0.5)))
    o = torch.empty_like(q)
    for b in range(B):
        sl = slice(b * HW, (b + 1) * HW)
        o[sl] = torch.softmax(q[sl] @ k[sl].t() * alpha, dim=-1) @ v[sl]
    return o @ lin["proj_out"][0].t() + lin["proj_out"][1] + x


@pytest.mark.gpu
@pytest.mark.parametrize("B,HW,Cc", [(2, 4096, 512), (2, 1000, 128)])
def test_vae_attention_block(B, HW, Cc):
    """plan._vae_attn at the production shape (B = 2: the per-batch loop reuses the packed K / V^T, S and P buffers)
    and a ragged one (HW even, not a multiple of 64).  The score and output GEMMs read dynamic B operands: they must be
    planned without GEMM_STATIC_B (their weight producer waits for pack_b).

    Block output: the GEMM bound of the matrix (two-plane operands, fp32 output).  For the last batch element, the
    intermediates are checked against references built from the operands the kernels read back: S (fp32) against
    (q_hi + q_lo) k^T * alpha with the same GEMM bound, P (two planes) against the float64 softmax of that S with
    _softmax_bound.  Everything outside the output lies in the program's own buffers or must be unchanged."""
    pl, x, out, xin, sd, n = _plan_vae_attn(B, HW, Cc, seed=HW + Cc)
    dyn = [o for o in pl.ops if o["kind"] == "gemm" and o["w_packed"].region == "ws"]
    assert len(dyn) == 2 * B and all(not (o["impl"] & _lib.GEMM_STATIC_B) for o in dyn), [o["impl"] for o in dyn]
    packs = [i for i, o in enumerate(pl.ops) if o["kind"] == "packb"]
    assert len(packs) == 2 * B
    last_pv = max(i for i, o in enumerate(pl.ops) if o is dyn[-1])
    sm = [o for o in pl.ops if o["kind"] == "softmax"][-1]
    score = dyn[-2]
    kpack = pl.ops[packs[-2]]
    prog = engine.DeviceProgram(pl, torch.device(DEV), dict(a=(0, last_pv + 1), b=(last_pv + 1, len(pl.ops))))
    ws = prog.ws
    ws.fill_(0xFF)
    scr = sorted({o["scratch"].off for o in pl.ops if o.get("scratch") is not None})
    for off in scr:
        ws[off:off + Planner.gn_scratch_bytes(B)].zero_()
    ws[x.ref.off:x.ref.off + xin.numel() * 4].copy_(xin.reshape(-1).view(torch.uint8).to(DEV))
    before = ws.clone()
    prog.run("a")
    torch.cuda.synchronize()
    # last batch element's intermediates, before the tail of the program reuses their memory
    Cp = round_up(Cc, 8)
    qh = ws[score["a_hi"].off:score["a_hi"].off + HW * Cp * 2].view(torch.float16).reshape(HW, Cp)[:, :Cc].double()
    ql = ws[score["a_lo"].off:score["a_lo"].off + HW * Cp * 2].view(torch.float16).reshape(HW, Cp)[:, :Cc].double()
    kk = ws[kpack["src"].off:kpack["src"].off + HW * Cc * 4].view(torch.float32).reshape(HW, Cc).double()
    S = ws[sm["x"].off:sm["x"].off + HW * HW * 4].view(torch.float32).reshape(HW, HW).double().clone()
    Pd = (ws[sm["out_hi"].off:sm["out_hi"].off + HW * HW * 2].view(torch.float16).double()
          + ws[sm["out_lo"].off:sm["out_lo"].off + HW * HW * 2].view(torch.float16).double()).reshape(HW, HW)
    S_ref = (qh + ql) @ kk.t() * float(np.float32(score["alpha"]))
    _check(f"vae_attn B={B} HW={HW} S", S, S_ref, 0)
    p_ref = torch.softmax(S, dim=-1)
    _within(f"vae_attn B={B} HW={HW} P", Pd, p_ref, _softmax_bound(S, p_ref, 2), _softmax_rl2(p_ref, 2))
    del qh, ql, kk, S, Pd, S_ref, p_ref
    prog.run("b")
    torch.cuda.synchronize()
    wo = Win(out.ref.off, B * HW, Cc, Cc, 4)
    first_internal = x.ref.off + round_up(B * HW * Cc * 4, 256)
    _assert_unchanged(ws, before, [wo], [(first_internal, pl.ws_bytes - first_internal)])
    _check(f"vae_attn B={B} HW={HW} out", wo.view(ws), _attn_block_ref(xin, sd, n, B, HW, Cc), 0)


# ----------------------------------------------------------------------------------------------
# STFT + mel + log (stft_mel_kernel)
# ----------------------------------------------------------------------------------------------
# n_fft -> (sr, hop, n_mels, fmin, fmax)
STFT_CFG = {256: (4000, 37, 16, 0, 2000), 512: (8000, 80, 32, 0, 4000), 1024: (16000, 160, 64, 0, 8000),
            2048: (48000, 480, 256, 20, 24000)}
STFT_KINDS = ["white", "band_limited", "tone", "quiet", "zero"]
STFT_FFT_C = 4.0         # constant of the per-bin FFT error bound (see test_stft_mel)


def _stft_signal(kind: str, B: int, T: int, sr: int, g) -> torch.Tensor:
    if kind == "zero":
        return torch.zeros(B, T)
    if kind == "tone":
        t = torch.arange(T, dtype=torch.float64) / sr
        f = torch.tensor([0.11, 0.23, 0.31])[:B, None] * sr
        return (0.5 * torch.sin(2 * math.pi * f * t + torch.arange(B)[:, None])).float()
    w = torch.rand(B, T, generator=g, dtype=torch.float64) - 0.5
    if kind == "band_limited":          # content below a quarter of the sampling rate
        W = torch.fft.rfft(w, dim=-1)
        W[:, torch.fft.rfftfreq(T, 1 / sr) >= sr / 8] = 0
        w = torch.fft.irfft(W, T, dim=-1)
        w = 0.3 * w / w.abs().amax(-1, keepdim=True)
    if kind == "quiet":
        w = 2e-3 * w
    return w.float()


def _stft_bound(wav: np.ndarray, n_fft: int, hop: int, basis: np.ndarray, logmel: np.ndarray) -> np.ndarray:
    """Per-element bound on |d log-mel| [B, n_mels, frames] (see test_stft_mel)."""
    B, T = wav.shape
    from oracle import mel as OM
    x = np.pad(wav.astype(np.float64), ((0, 0), (n_fft // 2, n_fft // 2)), mode="reflect")
    nfr = (x.shape[1] - n_fft) // hop + 1
    frames = x[:, np.arange(n_fft)[None, :] + hop * np.arange(nfr)[:, None]] * OM.hann_periodic(n_fft)
    norm = np.linalg.norm(frames, axis=-1)                                     # [B, frames]
    mag = np.abs(np.fft.rfft(frames, axis=-1))                                 # [B, frames, bins]
    b64 = basis.astype(np.float64)
    e_bin = (STFT_FFT_C * math.log2(n_fft) + 4) * U * norm                     # per bin, [B, frames]
    mel = np.einsum("mk,bfk->bmf", b64, mag)
    gemv = (n_fft // 2 // 32 + 1 + 5 + 2) * U
    dmel = b64.sum(1)[None, :, None] * e_bin[:, None, :] + gemv * mel
    den = np.maximum(mel - dmel, 1e-5)
    return dmel / den + 2.0 ** -22 * np.abs(logmel) + 1e-6


@pytest.mark.gpu
@pytest.mark.parametrize("kind", STFT_KINDS)
@pytest.mark.parametrize("n_fft", sorted(STFT_CFG))
def test_stft_mel(n_fft, kind):
    """stft_mel for B = 3 clips with out_frames < frames, once with T = 7 hop + 13 and once with T = n_fft / 2 + 1
    (every frame reflects, the middle ones at both ends); hop does not divide T.  Reference: oracle/mel.py (float64,
    returned as float32).

    Bound on |d log-mel|: the fp32 radix-2 FFT of a frame errs in every bin by at most (C log2 N + 4) u ||frame||_2
    (each of the log2 N stages rounds values whose sum of squares is N ||frame||^2 at about u per butterfly; the error
    reaching one bin is a unitary-weighted sum over them, so it grows with log2 N times the frame's L2 norm; the + 4
    covers the window's cospif and product; C = STFT_FFT_C).  The mel row sums basis * bin errors, plus the fp32 GEMV
    (a per-lane chain of N / 64 + 1 terms and a 5-level tree) and sqrtf: (N / 64 + 8) u mel.  log(max(mel, 1e-5)) moves
    by dmel / max(mel - dmel, 1e-5); logf and the oracle's float32 output add 2^-22 |log|."""
    from oracle import mel as OM
    sr, hop, n_mels, fmin, fmax = STFT_CFG[n_fft]
    g = torch.Generator().manual_seed(n_fft + STFT_KINDS.index(kind))
    B = 3
    basis = OM.mel_filterbank(sr, n_fft, n_mels, fmin, fmax)
    slab = _Slab()
    runs = []
    for T in (7 * hop + 13, n_fft // 2 + 1):
        assert T % hop
        wav = _stft_signal(kind, B, T, sr, g)
        frames = T // hop + 1
        of = frames - 1
        runs.append((T, wav, of, slab.put(wav), slab.region(B * of * n_mels * 4)))
    boff = slab.put(torch.from_numpy(basis))
    L = _lib.lib()

    def go(ptr, st):
        for T, wav, of, woff, ooff in runs:
            _lib.check(L.aldm_stft_mel(ptr(woff), B, T, n_fft, hop, ptr(boff), n_mels, ptr(ooff), of, st), "stft_mel")

    ws = slab.run(go, [Win(ooff, 1, B * of * n_mels, B * of * n_mels, 4) for _, _, of, _, ooff in runs])
    for T, wav, of, _, ooff in runs:
        want, _ = OM.stft_mel(wav.numpy(), n_fft, hop, n_mels, sr, fmin, fmax)       # [B, n_mels, frames]
        bound = _stft_bound(wav.numpy(), n_fft, hop, basis, want.astype(np.float64))[:, :, :of]
        want = want[:, :, :of]
        got = _flat(ws, ooff, B * of * n_mels).reshape(B, of, n_mels).permute(0, 2, 1)
        if kind == "zero":
            assert bool((got == float(np.float32(math.log(1e-5)))).all()), "all-zero clip: not log(1e-5)"
        _within(f"stft n_fft={n_fft} {kind} T={T}", got, torch.from_numpy(want), torch.from_numpy(bound), 1e-4)


# ----------------------------------------------------------------------------------------------
# sampler and small kernels
# ----------------------------------------------------------------------------------------------
def _ddim_coef(st: dict, guidance: float):
    """The fp32 coefficients as aldm_ddim_step computes them from its fp32 arguments."""
    f = np.float32
    a_t, a_prev, sig, s1m = f(st["a_t"]), f(st["a_prev"]), f(st["sigma_t"]), f(st["sqrt_one_minus_at"])
    return dict(inv_sqrt_at=float(np.sqrt(a_t)), s1m=float(s1m), sqrt_aprev=float(np.sqrt(a_prev)),
                dir=float(np.sqrt(f(f(f(1.0) - a_prev) - f(sig * sig)))), sigma=float(sig), g=float(f(guidance)))


@pytest.mark.gpu
@pytest.mark.parametrize("with_px0", [True, False])
@pytest.mark.parametrize("guidance", [1.0, 3.5])
@pytest.mark.parametrize("eta", [0.0, 1.0])
@pytest.mark.parametrize("step", [0, 199])
def test_ddim_step(step, eta, guidance, with_px0):
    """ddim_step on n / 4 > 8 * SMs * 256 float4 (the grid is capped there: every thread runs the grid-stride loop
    twice, some three times), first and last step of the 200-step schedule.  Reference: float64 with the launcher's
    fp32 coefficients.  Bound: each fp32 operation rounds at u of its operands' magnitude, with or without FMA
    contraction: |d e| <= 3 u (|U| + g (|C| + |U|)); |d p0| <= (s1m |d e| + 3 u (|X| + s1m |e|)) / sqrt(a_t) + u |p0|;
    |d x'| <= sqrt(a_prev) |d p0| + dir |d e| + 4 u (sqrt(a_prev) |p0| + dir |e| + sigma |Z|).  Without pred_x0 its
    region must stay untouched."""
    from oracle import functional as OF
    st = OF.ddim_schedule(OF.ddpm_tables(), 200, eta)[step]
    c = _ddim_coef(st, guidance)
    n = 4 * (8 * _n_sm() * 256 * 2 + 777)
    g = torch.Generator().manual_seed(step + int(10 * eta) + int(guidance))
    X, Uu, Cn, Z = (torch.randn(n, generator=g) for _ in range(4))
    slab = _Slab()
    offs = [slab.put(t) for t in (X, Uu, Cn, Z)]
    o_xp, o_px = slab.region(n * 4), slab.region(n * 4)
    L = _lib.lib()

    def go(ptr, s):
        _lib.check(L.aldm_ddim_step(*(ptr(o) for o in offs), ptr(o_xp), ptr(o_px) if with_px0 else None, n, st["a_t"],
                                    st["a_prev"], st["sigma_t"], st["sqrt_one_minus_at"], guidance, s), "ddim_step")

    wins = [Win(o_xp, 1, n, n, 4)] + ([Win(o_px, 1, n, n, 4)] if with_px0 else [])
    ws = slab.run(go, wins)
    x, u_, cn, z = (t.to(DEV, torch.float64) for t in (X, Uu, Cn, Z))
    e = u_ + c["g"] * (cn - u_)
    p0 = (x - c["s1m"] * e) / c["inv_sqrt_at"]
    xp = c["sqrt_aprev"] * p0 + c["dir"] * e + c["sigma"] * z
    de = 3 * U * (u_.abs() + c["g"] * (cn.abs() + u_.abs()))
    dp = (c["s1m"] * de + 3 * U * (x.abs() + c["s1m"] * e.abs())) / c["inv_sqrt_at"] + U * p0.abs()
    dx = c["sqrt_aprev"] * dp + c["dir"] * de + 4 * U * (c["sqrt_aprev"] * p0.abs() + c["dir"] * e.abs() + c["sigma"] * z.abs())
    _within(f"ddim step={step} eta={eta} g={guidance} x_prev", _flat(ws, o_xp, n), xp, dx, 1e-6)
    if with_px0:
        _within(f"ddim step={step} pred_x0", _flat(ws, o_px, n), p0, dp, 1e-6)


@pytest.mark.gpu
def test_masked_blend():
    """masked_blend (in place) for B = 3 with a per-batch mask of 0, 1 and fractional values.  Bound: the fp32
    sa x0 + sb qn, the two mask products and the sum: 4 u (sa |x0| + sb |qn| + |img|)."""
    g = torch.Generator().manual_seed(3)
    B, Cc, T, Fq = 3, 8, 37, 16
    img, x0, qn = (torch.randn(B, Cc, T, Fq, generator=g) for _ in range(3))
    mask = (torch.rand(B, 1, T, Fq, generator=g) > 0.5).float()
    mask[1, :, 5:9] = 0.25
    mask[2] = 1 - mask[0]
    sa, sb = float(np.float32(0.8)), float(np.float32(0.6))
    slab = _Slab()
    oi, ox, om, oq = (slab.put(t) for t in (img, x0, mask, qn))
    L = _lib.lib()
    n = img.numel()

    def go(ptr, s):
        _lib.check(L.aldm_masked_blend(ptr(oi), ptr(ox), ptr(om), ptr(oq), B, Cc, T * Fq, sa, sb, s), "masked_blend")

    ws = slab.run(go, [Win(oi, 1, n, n, 4)])
    d = dict(device=DEV, dtype=torch.float64)
    m = mask.to(**d)
    want = (sa * x0.to(**d) + sb * qn.to(**d)) * m + (1 - m) * img.to(**d)
    bound = 4 * U * (sa * x0.to(**d).abs() + sb * qn.to(**d).abs() + img.to(**d).abs())
    _within("masked_blend", _flat(ws, oi, n), want, bound, 1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("zc", [8, 16])
def test_posterior(zc):
    """posterior_sample: NHWC moments (mean | log-variance), NCHW noise and output, odd HW; log-variances beyond both
    clamps (-30, 20), where the mean is zero so that the clamped exp(lv / 2) decides the output.  Bound: expf (2 ulp),
    the product, the sum and the scale: |scale| (2^-21 exp(lv / 2) |noise| + 2 u (|mean| + exp(lv / 2) |noise|))."""
    g = torch.Generator().manual_seed(zc)
    B, H, W = 2, 5, 7
    mean = torch.randn(B, H, W, zc, generator=g)
    lv = 4 * torch.randn(B, H, W, zc, generator=g)
    lv.view(-1)[::5] = torch.tensor([-50.0, -31.0, 21.0, 25.0])[torch.arange(lv.numel())[::5] % 4]
    mean[(lv < -30) | (lv > 20)] = 0.0
    mom = torch.cat([mean, lv], dim=-1).contiguous()
    noise = torch.randn(B, zc, H, W, generator=g)
    scale = float(np.float32(0.7))
    slab = _Slab()
    o_m, o_n = slab.put(mom), slab.put(noise)
    o_z = slab.region(noise.numel() * 4)
    L = _lib.lib()
    n = noise.numel()

    def go(ptr, s):
        _lib.check(L.aldm_posterior_sample(ptr(o_m), ptr(o_n), ptr(o_z), B, zc, H * W, scale, s), "posterior_sample")

    ws = slab.run(go, [Win(o_z, 1, n, n, 4)])
    d = dict(device=DEV, dtype=torch.float64)
    mean = mom[..., :zc].permute(0, 3, 1, 2).to(**d)
    sd = torch.exp(0.5 * mom[..., zc:].permute(0, 3, 1, 2).to(**d).clamp(-30.0, 20.0))
    nz = noise.to(**d)
    want = scale * (mean + sd * nz)
    bound = scale * (2.0 ** -21 * sd * nz.abs() + 2 * U * (mean.abs() + sd * nz.abs()))
    _within(f"posterior zc={zc}", _flat(ws, o_z, n), want, bound, 1e-6)


def _temb_dims():
    return sorted({arch.model_config("audioldm2-full")["unet"]["model_channels"], arch.tiny_config()["unet"]["model_channels"]})


@pytest.mark.gpu
@pytest.mark.parametrize("dim", _temb_dims())
def test_temb(dim):
    """Timestep embedding of every t in 0..999 in one batch, two planes and one.  Reference: cos / sin in float64 of
    the fp32 argument t * freqs (the host's fp32 table), as util.py forms it.  cosf / sinf are within 2 ulp
    (2^-22 absolute for values <= 1) after an exact argument reduction; then PLANE_ERR."""
    half = dim // 2
    freqs = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32) / half)
    t = torch.arange(1000, dtype=torch.int64)
    B = t.numel()
    P = Planner()
    t_ref, f_ref = _guarded(P, B * 8), P.vec(freqs)
    o2, o1 = _guarded_planes(P, B, dim, 2), _guarded_planes(P, B, dim, 1)
    for o in (o2, o1):
        P.ops.append(dict(kind="temb", t=t_ref, freqs=f_ref, out_hi=o.hi, out_lo=o.lo, B=B, dim=dim))
    pl = P.finish({})
    prog = _run_guarded(pl, [(t_ref.off, t)], _planes_wins(o2, B, dim) + _planes_wins(o1, B, dim))
    arg = (t.float()[:, None] * freqs[None]).to(DEV, torch.float64)
    want = torch.cat([torch.cos(arg), torch.sin(arg)], dim=1)
    for o, planes in ((o2, 2), (o1, 1)):
        hi, lo = _planes_of(prog.ws, o, B, dim)
        got = hi.double() + (lo.double() if lo is not None else 0)
        _within(f"temb dim={dim} planes={planes}", got, want, _plane_err(want, planes) + (1 if planes == 2 else 2) * 2.0 ** -22,
                2e-5 if planes == 2 else 3e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 8])
def test_transpose(C):
    """transpose_chw [B, C, HW] -> [B, HW, C] and back, odd HW: exact."""
    g = torch.Generator().manual_seed(C)
    B, HW = 3, 37
    x = torch.randn(B, C, HW, generator=g)
    slab = _Slab()
    o_x, o_t, o_b = slab.put(x), slab.region(x.numel() * 4), slab.region(x.numel() * 4)
    L = _lib.lib()
    n = x.numel()

    def go(ptr, s):
        _lib.check(L.aldm_transpose_chw(ptr(o_x), ptr(o_t), B, C, HW, 1, s), "transpose")
        _lib.check(L.aldm_transpose_chw(ptr(o_t), ptr(o_b), B, C, HW, 0, s), "transpose")

    ws = slab.run(go, [Win(o_t, 1, n, n, 4), Win(o_b, 1, n, n, 4)])
    assert torch.equal(_flat(ws, o_t, n).cpu().reshape(B, HW, C), x.permute(0, 2, 1))
    assert torch.equal(_flat(ws, o_b, n).cpu().reshape(B, C, HW), x)


# ----------------------------------------------------------------------------------------------
# kernel inventory (CPU)
# ----------------------------------------------------------------------------------------------
KERNEL_TESTS = {
    "gemm_tc3_kernel": "test_gpu_kernel_matrix::test_gemm_matrix",
    "splitk_epilogue_kernel": "test_gpu_kernel_matrix::test_gemm_matrix",
    "splitk_reduce4_kernel": "test_gpu_kernel_matrix::test_gemm_matrix",
    "attention_tc_kernel": "test_gpu_kernel_matrix::test_attention_matrix",
    "attention_short_kernel": "test_gpu_kernel_matrix::test_attention_matrix",
    "gn_stats_kernel": "test_gpu_kernel_matrix::test_groupnorm_offset",
    "gn_apply_kernel": "test_gpu_kernel_matrix::test_groupnorm_offset",
    "gn_stats_col_kernel": "test_gpu_kernel_matrix::test_groupnorm_offset",
    "gn_apply_col_kernel": "test_gpu_kernel_matrix::test_groupnorm_offset",
    "gn_fused_kernel": "test_gpu_kernel_matrix::test_groupnorm_offset",
    "ln_kernel": "test_gpu_kernel_conformance::test_layernorm",
    "ew_kernel": "test_gpu_kernel_conformance::test_prep_elementwise",
    "pack_b_kernel": "test_gpu_kernel_conformance::test_pack_b",
    "softmax_rows_kernel": "test_gpu_kernel_conformance::test_softmax_rows",
    "stft_mel_kernel": "test_gpu_kernel_conformance::test_stft_mel",
    "ddim_step_kernel": "test_gpu_kernel_conformance::test_ddim_step",
    "masked_blend_kernel": "test_gpu_kernel_conformance::test_masked_blend",
    "temb_kernel": "test_gpu_kernel_conformance::test_temb",
    "transpose_kernel": "test_gpu_kernel_conformance::test_transpose",
    "posterior_kernel": "test_gpu_kernel_conformance::test_posterior",
}
KERNEL_EXEMPT = {
    "store_rate_kernel": "store-bandwidth microbenchmark, not on the sampling path",
    "gemm_simt_kernel": "CUDA-core checker of the GEMM, validation only",
    "attention_simt_kernel": "CUDA-core checker of the attention kernel, validation only",
    "fill_i64_kernel": "fills the timestep slot; covered by the engine-ABI tests",
}


def test_every_kernel_has_a_conformance_test():
    import importlib
    names = set()
    csrc = os.path.join(ROOT, "audioldm2_b200", "csrc")
    for f in sorted(os.listdir(csrc)):
        if f.endswith(".cu"):
            with open(os.path.join(csrc, f)) as fh:
                names |= set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s*)?(\w+)", fh.read()))
    assert len(names) > 20, sorted(names)
    missing = names - set(KERNEL_TESTS) - set(KERNEL_EXEMPT)
    assert not missing, f"kernels without a conformance test or an exemption: {sorted(missing)}"
    stale = (set(KERNEL_TESTS) | set(KERNEL_EXEMPT)) - names
    assert not stale, f"inventory entries for kernels that no longer exist: {sorted(stale)}"
    for k, ref in KERNEL_TESTS.items():
        mod, fn = ref.split("::")
        assert callable(getattr(importlib.import_module("tests." + mod), fn, None)), f"{k}: {ref} does not exist"


def test_full_plans_do_not_use_the_generic_groupnorm():
    """Every GroupNorm of the audioldm2-full UNet (batch 8), VAE decoder and encoder has C % 128 == 0, so it runs the
    single-pass or column-owner kernels; the generic statistics kernel (gn_stats_kernel) only runs on the 32- and
    64-channel layers of the small topologies."""
    from audioldm2_b200 import synth
    cfg = arch.model_config("audioldm2-full")
    ds = 2 ** (len(cfg["vae"]["ch_mult"]) - 1)
    _, T, Fq = cfg["latent"]
    vsd = synth.vae_state_dict(cfg["vae"])
    plans = {"unet": plan.build_unet(synth.unet_state_dict(cfg["unet"]), cfg["unet"], cfg["latent"], 8, ctx_max_len=(8, 32)),
             "vae_dec": plan.build_vae_decoder(vsd, cfg["vae"], cfg["latent"], 8),
             "vae_enc": plan.build_vae_encoder(vsd, cfg["vae"], (T * ds, Fq * ds), 8)}
    for name, pl in plans.items():
        gn = [o for o in pl.ops if o["kind"] == "prep" and o["mode"] in (_lib.PREP_GN, _lib.PREP_GN_SILU)]
        assert gn, name
        bad = sorted({(o["c0"], o["c1"]) for o in gn if (o["c0"] + o["c1"]) % 128})
        assert not bad, f"{name}: GroupNorm on the generic path for (c0, c1) in {bad}"


# ----------------------------------------------------------------------------------------------
# PDL bit-identity: every program with programmatic dependent launch equals a serialized run (ALDM_PDL=0)
# ----------------------------------------------------------------------------------------------
PDL_PROGRAMS = ["tiny_unet", "tiny_vae_dec", "tiny_vae_enc", "tiny_vocoder", "full_unet_b2", "vae_attn"]


def _pdl_outputs(which: str, check_graph: bool) -> dict:
    """Run one program on fixed inputs; outputs as CPU tensors.  check_graph: also replay it as a CUDA graph and
    assert the replay equals the eager run."""
    from audioldm2_b200 import model, synth
    from tests.golden import cases
    out = {}
    if which == "vae_attn":
        pl, x, o, xin, _, _ = _plan_vae_attn(2, 4096, 512, seed=7)
        prog = engine.DeviceProgram(pl, torch.device(DEV), dict(all=(0, len(pl.ops))))
        prog.ws[x.ref.off:x.ref.off + xin.numel() * 4].copy_(xin.reshape(-1).view(torch.uint8).to(DEV))
        prog.run("all")
        wo = Win(o.ref.off, x.rows, x.C, x.C, 4)
        out["out"] = wo.view(prog.ws).cpu().clone()
        if check_graph:
            wo.view(prog.ws).fill_(float("nan"))
            prog.replay("all")
            torch.cuda.synchronize()
            assert torch.equal(wo.view(prog.ws).cpu(), out["out"]), "vae_attn: graph replay differs from the eager run"
        return out
    full = which.startswith("full")
    cfg = arch.model_config("audioldm2-full") if full else arch.tiny_config()
    B = 2
    t5 = 32 if full else 5
    eng = model.build_synthetic(cfg=cfg, batch=B, device=DEV, t5_len=t5, with_encoder=which == "tiny_vae_enc")
    if which.endswith("unet") or which == "full_unet_b2":
        cond, unc = synth.conditioning(cfg, B, seed=77, t5_len=t5)
        to = lambda c: dict(context_list=[t.to(DEV) for t in c["context_list"]], mask_list=[t.to(DEV) for t in c["mask_list"]],
                            y=None)
        eng.set_conditioning(to(cond), to(unc))
        x = cases.latent(cfg, B, seed=3).to(DEV).contiguous()
        e_u, e_c = eng.apply_model_pair(x, 417)          # first call: eager run, then capture
        out["eps_u"], out["eps_c"] = e_u.cpu().clone(), e_c.cpu().clone()
        if check_graph:
            e_u2, e_c2 = eng.apply_model_pair(x, 417)    # graph replay
            assert torch.equal(e_u2.cpu(), out["eps_u"]) and torch.equal(e_c2.cpu(), out["eps_c"]), \
                f"{which}: graph replay differs from the eager run"
        return out
    if which == "tiny_vae_dec":
        prog, io_in, io_out = eng.vae_dec, "z", "mel"
        val = cases.latent(cfg, B, seed=5)
    elif which == "tiny_vae_enc":
        prog, io_in, io_out = eng.vae_enc, "mel", "moments"
        val = cases.mel_input(cfg, B)
    else:
        prog, io_in, io_out = eng.vocoder, "mel", "wave"
        g = torch.Generator().manual_seed(9)
        val = torch.randn(prog.view("mel").shape, generator=g)
    prog.view(io_in).copy_(val.reshape(prog.view(io_in).shape).to(DEV))
    prog.run("all")
    torch.cuda.synchronize()
    out[io_out] = prog.view(io_out).cpu().clone()
    if check_graph:
        prog.view(io_out).fill_(float("nan"))
        prog.replay("all")
        torch.cuda.synchronize()
        assert torch.equal(prog.view(io_out).cpu(), out[io_out]), f"{which}: graph replay differs from the eager run"
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("which", PDL_PROGRAMS)
def test_pdl_matches_serialized_run(which, tmp_path):
    """The kernels are deterministic, and with programmatic dependent launch a kernel may start while its
    predecessor drains, so it must not touch memory before griddepcontrol.wait: the outputs of a program run with
    PDL (this process) must equal, bit for bit, those of the same program in a child process with ALDM_PDL=0
    (every launch fully serialized).  The eager run must also equal its graph replay."""
    got = _pdl_outputs(which, check_graph=True)
    path = str(tmp_path / "serial.pt")
    env = dict(os.environ, ALDM_PDL="0")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), which, path]
    r = subprocess.run(cmd, env=env, cwd=ROOT, timeout=900, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    assert r.returncode == 0, f"serialized run failed:\n{r.stdout.decode(errors='replace')[-4000:]}"
    want = torch.load(path)
    assert set(want) == set(got)
    for k in got:
        assert torch.isfinite(got[k]).all(), f"{which}/{k}: non-finite output"
        assert torch.equal(got[k], want[k]), (f"{which}/{k}: PDL run differs from the serialized run in "
                                              f"{int((got[k] != want[k]).sum())} elements")


if __name__ == "__main__":          # child of test_pdl_matches_serialized_run: run one program, save its outputs
    assert os.environ.get("ALDM_PDL") == "0"
    torch.save(_pdl_outputs(sys.argv[1], check_graph=False), sys.argv[2])
