"""Accumulator hand-off of the persistent GEMM: one launch with many tiles per CTA against row-slice launches.

The persistent kernel hands every tile's accumulator from the consumer warpgroups to the epilogue warpgroup through one
shared-memory buffer and two mbarriers, while the consumers already run the next tile's MMAs.  A race in that hand-off
(the consumers overwriting rows the epilogue has not read yet, or the epilogue reading rows not yet written) changes
output bits without necessarily leaving a tolerance, so each case here runs the same GEMM twice in one program:

  * full: one launch over all rows, at least 16 tiles per CTA, so every CTA hands the accumulator over many times;
  * sliced: the same rows as separate launches of at most one wave each (batch elements for convolutions, groups of
    sequences for the Q|K|V projections), so no CTA reuses the buffer,

and requires the two outputs to be bit-identical (each output element's arithmetic does not depend on the tile that
computes it), finite, and every byte outside the output windows unchanged (the 4 KB guard bands of
test_gpu_kernel_matrix.py).  The cases cover every (N tile, epilogue body, A planes, reduction, store mode) that
aldm_gemm_variant can return, split-K included; the full and sliced launches of a case run the same variant (checked on
the CPU).  Each case runs once."""
import math

import pytest
import torch

from audioldm2_b200 import _lib, plan
from audioldm2_b200.packing import round_up
from audioldm2_b200.plan import VT, Planes, Planner
from tests.test_gpu_kernel_matrix import GUARD, Win, _guarded, _guarded_planes, _n_sm, _reachable_variants, _run_guarded

GEGLU, TANH, SILU = _lib.ACT_GEGLU, _lib.ACT_TANH, _lib.ACT_SILU
MIN_TILES_PER_CTA = 16
TPB = 203            # tokens per sequence of the Q|K|V cases (ragged against 128-row tiles; V^T has padding keys)

# kind -> (activation, split-K, output: f32 / planes1 / planes2 / qkv1 / qkv2, residual, row vector)
KINDS = {
    "f32n": (_lib.ACT_NONE, 1, "f32", True, False),          # EPI_F32N, compact
    "pln": (_lib.ACT_NONE, 1, "planes2", True, False),       # EPI_PLN, compact
    "pln_pair": (_lib.ACT_NONE, 1, "planes1", False, False),  # EPI_PLN, full-line stores
    "fast": (_lib.ACT_NONE, 1, "f32", True, True),           # EPI_FAST, row vector + residual
    "qkv2": (_lib.ACT_NONE, 1, "qkv2", False, False),        # EPI_FAST, V^T planes + padding keys
    "qk_pair": (_lib.ACT_NONE, 1, "qkv1", False, False),     # EPI_FAST, Q|K full-line stores
    "geglu": (GEGLU, 1, "f32", False, False),                # EPI_GEGLU, fp32 out
    "geglu_pl": (GEGLU, 1, "planes2", False, False),         # EPI_GEGLU, staged plane stores
    "geglu_pair": (GEGLU, 1, "planes1", False, False),       # EPI_GEGLU, full-line stores
    "gen": (SILU, 1, "f32", False, False),                   # EPI_GENERIC
    "sk4": (_lib.ACT_NONE, 3, "f32", True, False),           # split-K partials, coalesced reduction
    "skg": (TANH, 3, "f32", False, False),                   # split-K partials, row-owner reduction
}


def _cases():
    out = {}
    for ap in (1, 2):
        for bn in (32, 64, 128):
            kinds = ["f32n", "pln", "fast", "qkv2", "gen", "sk4", "skg"]
            if bn >= 64:
                kinds += ["pln_pair", "qk_pair", "geglu", "geglu_pl"]
            if bn == 128:
                kinds.append("geglu_pair")
            for k in kinds:
                out[f"{k}_b{bn}_a{ap}"] = (k, bn, ap)
    return out


CASES = _cases()


def build(name: str, n_sm: int):
    """Plan of one case: the full launch (op 0), then the slice launches.  Returns the plan, the input writes, pairs of
    (full, sliced) output windows, the split-K scratch regions and the tile counts."""
    kind, bn, ap = CASES[name]
    act, splitk, outk, has_res, has_rowvec = KINDS[kind]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    qkv = outk.startswith("qkv")
    conv = ap == 2 and not qkv                     # two-plane operands: the 3x3 convolution gather, sliced by batch element
    N = 3 * bn if qkv else 2 * bn
    Cc = N // 3
    n_out = N // 2 if act == GEGLU else N
    taps = plan.TAPS_3x3 if conv else ((0, 0),)
    Cin = (32 if splitk > 1 else 16) if conv else (256 if splitk > 1 else 64)
    tiles_n = math.ceil(N / bn) * splitk
    mt_slice = n_sm // tiles_n                     # M tiles one slice may have: at most one wave
    if qkv:
        nseq = mt_slice * 128 // TPB
        H, W = nseq * TPB, 1
    elif conv:
        H, W = (mt_slice * 128 - 51) // 8, 8
    else:
        H, W = mt_slice * 128 - 51, 1
    R = H * W                                      # rows of one slice (input rows = output rows: unit stride)
    S = math.ceil(MIN_TILES_PER_CTA * n_sm / (math.ceil(R / 128) * tiles_n)) + 1
    M = S * R

    P = Planner(splitk=False)
    T = len(taps)
    cp = round_up(Cin, 8)
    a = P.planes(M, Cin, ap)
    wm = torch.randn(N, T * cp, generator=g) / math.sqrt(T * Cin)
    bias = 0.1 * torch.randn(N, generator=g)
    w = P.wmat(wm, bias, T, cp, geglu=act == GEGLU, bn=bn)
    res = P.raw(M * n_out * 4) if has_res else None
    rowvec = P.raw(S * n_out * 4) if has_rowvec else None
    npl = 1 if outk in ("planes1", "qkv1") else 2
    ld_t = round_up(TPB, 8)

    def outputs():
        if qkv:
            vhi = _guarded(P, S * nseq * Cc * ld_t * 2)
            return dict(qk=_guarded_planes(P, M, 2 * Cc, npl),
                        vt=VT(vhi, _guarded(P, S * nseq * Cc * ld_t * 2) if npl == 2 else None, ld_t))
        if outk.startswith("planes"):
            return dict(planes=_guarded_planes(P, M, n_out, npl))
        return dict(f32=_guarded(P, M * n_out * 4))

    def add(o, b0, nb):        # slices [b0, b0 + nb)
        r0 = b0 * R
        kw = dict(a_off_rows=r0, act=act)
        if res is not None:
            kw.update(res_ref=res + r0 * n_out * 4, ld_res=n_out)
        if rowvec is not None:
            kw.update(rowvec=rowvec + b0 * n_out * 4, ld_rowvec=n_out)
        if qkv:
            qk, vt = o["qk"], o["vt"]
            qk_s = Planes(qk.hi + r0 * 2 * Cc * 2, qk.lo + r0 * 2 * Cc * 2 if qk.lo is not None else None, nb * R, 2 * Cc)
            vo = b0 * nseq * Cc * ld_t * 2
            vt_s = VT(vt.hi + vo, vt.lo + vo if vt.lo is not None else None, ld_t)
            op = P.gemm(a, w, B=1, H=nb * R, qkv=(qk_s, vt_s, 2 * Cc, TPB), **kw)
        elif "planes" in o:
            p = o["planes"]
            ps = Planes(p.hi + r0 * n_out * 2, p.lo + r0 * n_out * 2 if p.lo is not None else None, nb * R, n_out)
            op = P.gemm(a, w, B=nb, H=H, W=W, taps=taps, out_planes=ps, ldo=n_out, **kw)
        else:
            op = P.gemm(a, w, B=nb, H=H, W=W, taps=taps, out_ref=o["f32"] + r0 * n_out * 4, ldo=n_out, **kw)
        if splitk > 1:            # [splitk][Mpad][Npad] fp32 partial sums, shared by the launches, then GUARD zero bytes
            op["splitk"], op["ws"] = splitk, "SPLITK"
            P.splitk_ws_bytes = max(P.splitk_ws_bytes, splitk * round_up(nb * R, 128) * round_up(N, bn) * 4 + GUARD)

    full, sliced = outputs(), outputs()
    add(full, 0, S)
    for b in range(S):
        add(sliced, b, 1)
    pl = P.finish({})

    def wins(o):
        if qkv:
            vt = o["vt"]
            ws_ = [Win(o["qk"].hi.off, M, 2 * Cc, 2 * Cc, 2), Win(vt.hi.off, S * nseq * Cc, ld_t, ld_t, 2)]
            if npl == 2:
                ws_ += [Win(o["qk"].lo.off, M, 2 * Cc, 2 * Cc, 2), Win(vt.lo.off, S * nseq * Cc, ld_t, ld_t, 2)]
            return ws_
        if "planes" in o:
            p = o["planes"]
            return [Win(p.hi.off, M, n_out, n_out, 2)] + ([Win(p.lo.off, M, n_out, n_out, 2)] if p.lo is not None else [])
        return [Win(o["f32"].off, M, n_out, n_out, 4)]

    writes = []
    x = torch.zeros(M, a.Cp)
    x[:, :Cin] = torch.randn(M, Cin, generator=g)
    hi = x.half()
    writes.append((a.hi.off, hi))
    if a.lo is not None:
        writes.append((a.lo.off, (x - hi.float()).half()))
    if res is not None:
        writes.append((res.off, torch.randn(M, n_out, generator=g)))
    if rowvec is not None:
        writes.append((rowvec.off, torch.randn(S, n_out, generator=g)))
    zero, scratch = [], []
    if splitk > 1:
        ws = pl.ops[0]["ws"]
        part = splitk * round_up(M, 128) * round_up(N, bn) * 4
        zero.append((ws.off, part + GUARD))
        scratch.append((ws.off, part))
    tiles_full = math.ceil(M / 128) * tiles_n
    tiles_slice = math.ceil(R / 128) * tiles_n
    return pl, writes, list(zip(wins(full), wins(sliced))), zero, scratch, tiles_full, tiles_slice


def test_overlap_cases_cover_every_variant():
    """CPU: the full launch of every case has >= 16 tiles per CTA, every slice fits one wave, the full and sliced launches
    run the same kernel variant, and the cases together reach every variant aldm_gemm_variant can return."""
    _lib.build()
    seen = set()
    for name in CASES:
        pl, _, _, _, _, tiles_full, tiles_slice = build(name, plan.H100_SMS)
        assert tiles_full >= MIN_TILES_PER_CTA * plan.H100_SMS and tiles_slice <= plan.H100_SMS, (name, tiles_full, tiles_slice)
        arr = pl.resolve(1 << 32, 1 << 40)
        vs = {_lib.gemm_variant(arr[i].u.gemm) for i in range(len(arr))}
        assert len(vs) == 1, (name, vs)
        seen |= vs
    assert seen == _reachable_variants(), sorted(_reachable_variants() ^ seen)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_gemm_overlap_bit_identical(name):
    pl, writes, pairs, zero, scratch, tiles_full, _ = build(name, _n_sm())
    assert tiles_full >= MIN_TILES_PER_CTA * _n_sm()
    prog = _run_guarded(pl, writes, [w for pair in pairs for w in pair], zero, scratch)
    for wf, wsl in pairs:
        f, s = wf.view(prog.ws), wsl.view(prog.ws)
        assert torch.isfinite(f).all(), f"{name}: output at {wf.off} not (fully) written"
        fb = f.contiguous().view(torch.int16 if wf.esz == 2 else torch.int32)
        sb = s.contiguous().view(torch.int16 if wsl.esz == 2 else torch.int32)
        diff = (fb != sb).nonzero()
        assert diff.numel() == 0, (f"{name}: {diff.shape[0]} elements of the output at {wf.off} differ between the full and the "
                                   f"sliced launches; first at (row, column) {tuple(diff[0].tolist())}")
