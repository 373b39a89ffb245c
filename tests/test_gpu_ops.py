"""GPU parity tests of the individual kernels, called through the C-ABI (ctypes) and compared with
the CPU oracle / op-table emulator on the same seeded inputs.

Tolerances (written per test): elementwise kernels 1e-6; kernels behind fp16 hi/lo operand planes 2e-5 relative L2
(the emulator applies the same operand splitting, so GEMM-vs-emulator comparisons are at accumulate-order noise,
<= 1e-5; planes themselves carry 2^-22); single-plane outputs are compared after the same fp16 rounding (one-ulp flips
of a 2^-12 rounding: 3e-4 bound); the attention kernel rounds its probabilities to fp16 relative to the RUNNING row
maximum while the emulator rounds relative to the final one, so that comparison is bounded by 5e-4."""
import ctypes as C
import math

import numpy as np
import os

import pytest
import torch

from audioldm2_b200 import _lib, engine, packing, plan
from audioldm2_b200.plan import F32, Planes, Planner, Ref
from tests.conftest import rel_l2
from tests.emulator import Emulator

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def run_both(pl: plan.Plan, inputs: dict, fill=None):
    """Run a Plan on the GPU and in the emulator from identical workspace contents."""
    em = Emulator(pl)
    prog = engine.DeviceProgram(pl, torch.device(DEV), dict(all=(0, len(pl.ops))))
    for name, val in inputs.items():
        em.write_io(name, val)
        prog.view(name).copy_(val.to(DEV))
    em.run()
    prog.run("all")
    torch.cuda.synchronize()
    return em, prog


def read_gpu_f32(prog, ref: Ref, n: int):
    return prog.ws[ref.off:ref.off + 4 * n].view(torch.float32).cpu()


def read_gpu_planes(prog, p: Planes):
    n = p.rows * p.Cp
    x = prog.ws[p.hi.off:p.hi.off + 2 * n].view(torch.float16).float().cpu()
    if p.lo is not None:
        x = x + prog.ws[p.lo.off:p.lo.off + 2 * n].view(torch.float16).float().cpu()
    return x.reshape(p.rows, p.Cp)


# ----------------------------------------------------------------------------------------------
def test_device_and_library():
    L = _lib.lib()
    assert L.aldm_device_check(0) == 0, L.aldm_last_error()


def test_ddim_step_matches_oracle():
    from oracle import functional as OF
    g = torch.Generator().manual_seed(0)
    shape = (3, 8, 256, 16)
    x, eu, ec, nz = (torch.randn(shape, generator=g) for _ in range(4))
    st = OF.ddim_schedule(OF.ddpm_tables(), 200, 1.0)[17]
    want, want_p0 = OF.ddim_update(x, eu, ec, nz, st, 3.5)
    out = torch.empty(shape, device=DEV); p0 = torch.empty(shape, device=DEV)
    engine.ddim_step(x.to(DEV), eu.to(DEV), ec.to(DEV), nz.to(DEV), out, st["a_t"], st["a_prev"], st["sigma_t"],
                     st["sqrt_one_minus_at"], 3.5, p0)
    assert rel_l2(out, want) < 1e-6 and rel_l2(p0, want_p0) < 1e-6


def test_masked_blend_matches_oracle():
    from oracle import functional as OF
    g = torch.Generator().manual_seed(1)
    shape = (2, 8, 32, 8)
    img, x0, qn = (torch.randn(shape, generator=g) for _ in range(3))
    mask = torch.ones(2, 1, 32, 8); mask[:, :, 12:19] = 0
    st = OF.ddim_schedule(OF.ddpm_tables(), 50, 1.0)[3]
    want = OF.masked_blend(img, x0, mask, qn, st)
    got = img.to(DEV).clone()
    engine.masked_blend(got, x0.to(DEV), mask.to(DEV), qn.to(DEV), st["sqrt_acp_t"], st["sqrt_1m_acp_t"])
    assert rel_l2(got, want) < 1e-6


def test_groupnorm_fast_path():
    """C multiple of 128 (4 | channels per group) takes the column-owner kernels; concat of two sources."""
    g = torch.Generator().manual_seed(21)
    P = Planner(keep_plain=True)
    B, HW = 3, 70
    a = F32(P.raw(B * HW * 256 * 4), B * HW, 256)
    b = F32(P.raw(B * HW * 128 * 4), B * HW, 128)
    gam = P.vec(1 + 0.1 * torch.randn(384, generator=g)); bet = P.vec(0.1 * torch.randn(384, generator=g))
    o1 = P.prep(_lib.PREP_GN_SILU, a, b, gam, bet, eps=1e-5, B=B, HW=HW)
    o2 = P.prep(_lib.PREP_GN, a, None, gam, bet, eps=1e-6, B=B, HW=HW)
    pl = P.finish(dict(a=("f32", a.ref, (a.rows, a.C)), b=("f32", b.ref, (b.rows, b.C))))
    em, prog = run_both(pl, dict(a=torch.randn(a.rows, a.C, generator=g) * 2 + 0.5, b=torch.randn(b.rows, b.C, generator=g)))
    for o in (o1, o2):
        assert rel_l2(read_gpu_planes(prog, o), em.read_planes(o.hi, o.lo, o.rows, o.Cp)) < 2e-5


@pytest.mark.parametrize("B,HW,C", [(2, 4096, 128), (80, 2048, 128), (16, 64, 640), (3, 1000, 256), (2, 300, 1280), (4, 1024, 640)])
def test_groupnorm_large_and_repeated(B, HW, C):
    """GroupNorm kernels.  Single-pass kernel (all rows of a batch element for a chunk of groups parked in shared memory) where
    HW x chunk fits: (16, 64, 640), (3, 1000, 256), (2, 300, 1280), (4, 1024, 640).  Two-kernel path otherwise: many blocks per
    batch row (statistics published by the last block through the self-resetting ticket: (2, 4096, 128)) and few (the apply kernel
    reduces the partials: (80, 2048, 128)); repeated runs must see the tickets back at zero."""
    g = torch.Generator().manual_seed(5)
    P = Planner(keep_plain=True)
    a = F32(P.raw(B * HW * C * 4), B * HW, C)
    junk = P.raw(1 << 20); P.free(junk)          # a freed hole: the GroupNorm scratch must not land in reusable pool space
    gam = P.vec(1 + 0.1 * torch.randn(C, generator=g)); bet = P.vec(0.1 * torch.randn(C, generator=g))
    o1 = P.prep(_lib.PREP_GN_SILU, a, None, gam, bet, eps=1e-5, B=B, HW=HW)
    o2 = P.prep(_lib.PREP_GN, a, None, gam, bet, eps=1e-6, B=B, HW=HW, n=1)
    pl = P.finish(dict(a=("f32", a.ref, (a.rows, a.C))))
    x = torch.randn(a.rows, a.C, generator=g) * 3 + 1.5
    em, prog = run_both(pl, dict(a=x))
    want = [em.read_planes(o.hi, o.lo, o.rows, o.Cp) for o in (o1, o2)]
    for rep in range(3):
        if rep:
            prog.run("all"); torch.cuda.synchronize()
        for o, w in zip((o1, o2), want):
            assert rel_l2(read_gpu_planes(prog, o), w) < (2e-5 if o.lo is not None else 3e-4), (rep, B, HW, C)


@pytest.mark.parametrize("C", [96, 256, 384, 640, 1024])
def test_layernorm_widths(C):
    """ln_kernel<NQ>: float4 per lane sized to C (2 / 4 / 8)."""
    g = torch.Generator().manual_seed(C)
    P = Planner(keep_plain=True)
    rows = 333
    a = F32(P.raw(rows * C * 4), rows, C)
    gam = P.vec(1 + 0.1 * torch.randn(C, generator=g)); bet = P.vec(0.1 * torch.randn(C, generator=g))
    o = P.prep(_lib.PREP_LN, a, None, gam, bet, eps=1e-5, n=1)
    em, prog = run_both(P.finish(dict(a=("f32", a.ref, (rows, C)))), dict(a=torch.randn(rows, C, generator=g) * 2 + 0.7))
    assert rel_l2(read_gpu_planes(prog, o), em.read_planes(o.hi, o.lo, o.rows, o.Cp)) < 3e-4


@pytest.mark.parametrize("planes", [2, 1])
@pytest.mark.parametrize("mode", ["copy", "silu", "lrelu", "gn", "gn_silu", "ln", "nchw", "cat", "pad"])
def test_prep_modes(mode, planes):
    g = torch.Generator().manual_seed(2)
    P = Planner(keep_plain=True)
    B, HW = 3, 50
    if mode == "pad":
        src = F32(P.raw(B * HW * 1 * 4), B * HW, 1)
    elif mode == "ln":
        src = F32(P.raw(B * HW * 96 * 4), B * HW, 96)
    else:
        src = F32(P.raw(B * HW * 64 * 4), B * HW, 64)
    src2 = F32(P.raw(B * HW * 32 * 4), B * HW, 32)
    gam = P.vec(1 + 0.1 * torch.randn(96, generator=g)); bet = P.vec(0.1 * torch.randn(96, generator=g))
    m = dict(copy=_lib.PREP_COPY, silu=_lib.PREP_SILU, lrelu=_lib.PREP_LRELU, gn=_lib.PREP_GN, gn_silu=_lib.PREP_GN_SILU,
             ln=_lib.PREP_LN, nchw=_lib.PREP_COPY, cat=_lib.PREP_GN_SILU, pad=_lib.PREP_COPY)[mode]
    out = P.prep(m, src, src2 if mode == "cat" else None, gam, bet, eps=1e-5 if mode != "gn" else 1e-6, slope=0.1,
                 B=B, HW=HW, src_nchw=(mode == "nchw"), n=planes)
    assert (out.lo is None) == (planes == 1)
    pl = P.finish(dict(a=("f32", src.ref, (src.rows, src.C)), b=("f32", src2.ref, (src2.rows, src2.C))))
    em, prog = run_both(pl, dict(a=torch.randn(src.rows, src.C, generator=g) * 2 + 0.3,
                                 b=torch.randn(src2.rows, src2.C, generator=g)))
    want = em.read_planes(out.hi, out.lo, out.rows, out.Cp)
    got = read_gpu_planes(prog, out)
    assert torch.isfinite(got).all()
    assert rel_l2(got, want) < (2e-5 if planes == 2 else 3e-4), mode


def _gemm_case(P: Planner, g, *, B, H, W, Cin, N, taps, OH=None, OW=None, sy=1, sx=1, up=0, bmod=0, act=_lib.ACT_NONE,
               res=False, rowvec=False, alpha=1.0, accumulate=False, out_kind="f32", geglu=False, bias=True, dual=False,
               a_planes=2, out_planes_n=2):
    Hs, Ws = H >> up, W >> up
    Bsrc = bmod if bmod else B
    src = F32(P.raw(Bsrc * Hs * Ws * Cin * 4), Bsrc * Hs * Ws, Cin)
    a = P.prep(_lib.PREP_COPY, src, n=a_planes)
    cp = a.Cp
    wm = torch.zeros(N, len(taps), cp)
    wm[:, :, :Cin] = torch.randn(N, len(taps), Cin, generator=g) / math.sqrt(len(taps) * Cin)
    w = P.wmat(wm.reshape(N, -1), 0.1 * torch.randn(N, generator=g) if bias else None, len(taps), cp, geglu=geglu)
    OHv, OWv = (H if OH is None else OH), (W if OW is None else OW)
    M = B * OHv * OWv
    n_out = N // 2 if geglu else N
    kw = dict(B=B, H=H, W=W, taps=taps, OH=OH, OW=OW, sy=sy, sx=sx, up=up, bmod=bmod, act=act, alpha=alpha, accumulate=accumulate)
    ios = dict(src=("f32", src.ref, (src.rows, Cin)))
    ins = dict(src=torch.randn(src.rows, Cin, generator=g))
    if res:
        r = F32(P.raw(M * n_out * 4), M, n_out); kw["res"] = r
        ios["res"] = ("f32", r.ref, (M, n_out)); ins["res"] = torch.randn(M, n_out, generator=g)
    if rowvec:
        rv = P.raw(B * (n_out + 8) * 4); kw["rowvec"] = rv + 4 * 4; kw["ld_rowvec"] = n_out + 8
        ios["rv"] = ("f32", rv, (B, n_out + 8)); ins["rv"] = torch.randn(B, n_out + 8, generator=g)
    if out_kind == "f32":
        o = P.f32(M, n_out); kw["out"] = o
        ios["out"] = ("f32", o.ref, (M, n_out)); ins["out"] = torch.randn(M, n_out, generator=g)   # for accumulate
        if dual:
            dp = P.planes(M, n_out, out_planes_n); kw["also_planes"] = dp
            P.gemm(a, w, **kw)
            return ios, ins, ("dual", (o, dp))
        P.gemm(a, w, **kw)
        return ios, ins, ("f32", o)
    if out_kind == "planes":
        o = P.planes(M, n_out, out_planes_n); kw["out_planes"] = o
        P.gemm(a, w, **kw)
        return ios, ins, ("planes", o)
    o = P.raw(B * N * OHv * OWv * 4)
    P.gemm(a, w, out_ref=o, out_mode=_lib.OUT_NCHW, **kw)
    return ios, ins, ("nchw", (o, B * N * OHv * OWv))


GEMM_CASES = {
    "linear": dict(B=1, H=300, W=1, Cin=200, N=96, taps=((0, 0),)),
    "linear_big": dict(B=1, H=1000, W=1, Cin=640, N=384, taps=((0, 0),), res=True),
    "conv3x3": dict(B=2, H=20, W=6, Cin=24, N=128, taps=plan.TAPS_3x3, rowvec=True, res=True),
    "conv3x3_s2": dict(B=2, H=16, W=8, Cin=32, N=64, taps=plan.TAPS_3x3, OH=8, OW=4, sy=2, sx=2),
    "conv3x3_asym": dict(B=1, H=16, W=8, Cin=16, N=32, taps=plan.TAPS_3x3_ASYM, OH=8, OW=4, sy=2, sx=2),
    "conv3x3_up": dict(B=2, H=16, W=8, Cin=40, N=40, taps=plan.TAPS_3x3, up=1),
    "conv_bmod": dict(B=4, H=12, W=4, Cin=8, N=32, taps=plan.TAPS_3x3, bmod=2),
    "conv1d_dil": dict(B=2, H=333, W=1, Cin=32, N=32, taps=plan.taps_1d(11, 5), res=True, alpha=1 / 3, accumulate=True),
    "conv1d_k7_tanh": dict(B=2, H=500, W=1, Cin=32, N=1, taps=plan.taps_1d(7), act=_lib.ACT_TANH),
    "geglu": dict(B=1, H=200, W=1, Cin=64, N=512, taps=((0, 0),), geglu=True, act=_lib.ACT_GEGLU, out_kind="planes"),
    "silu_planes": dict(B=1, H=16, W=1, Cin=32, N=128, taps=((0, 0),), act=_lib.ACT_SILU, out_kind="planes"),
    "nchw_out": dict(B=2, H=16, W=8, Cin=32, N=8, taps=plan.TAPS_3x3, out_kind="nchw"),
    "deepK_splitk": dict(B=2, H=8, W=2, Cin=640, N=640, taps=plan.TAPS_3x3, res=True, rowvec=True),
    "nobias": dict(B=1, H=130, W=1, Cin=96, N=288, taps=((0, 0),), bias=False),
    "dual_out": dict(B=1, H=300, W=1, Cin=128, N=256, taps=((0, 0),), res=True, dual=True),
    # single-plane activations (two UMMAs per K step, 4-stage ring) and single-plane outputs: the token side of the UNet
    "a1_linear_big": dict(B=1, H=1000, W=1, Cin=640, N=384, taps=((0, 0),), res=True, a_planes=1),
    "a1_geglu_p1": dict(B=1, H=200, W=1, Cin=256, N=512, taps=((0, 0),), geglu=True, act=_lib.ACT_GEGLU, out_kind="planes",
                        a_planes=1, out_planes_n=1),
    "a1_planes_p1": dict(B=1, H=260, W=1, Cin=128, N=256, taps=((0, 0),), out_kind="planes", a_planes=1, out_planes_n=1),
    # full-line pair stores with 64-wide tiles, without bias, with a residual (falls back to the per-warp stores) and two-plane output
    "a1_planes_p1_n192": dict(B=1, H=700, W=1, Cin=128, N=192, taps=((0, 0),), out_kind="planes", a_planes=1, out_planes_n=1),
    "a1_planes_p1_nobias": dict(B=1, H=515, W=1, Cin=64, N=128, taps=((0, 0),), out_kind="planes", a_planes=1, out_planes_n=1, bias=False),
    "a1_planes_p2_res": dict(B=1, H=400, W=1, Cin=256, N=256, taps=((0, 0),), out_kind="planes", a_planes=1, res=True),
    "a1_planes_p1_res": dict(B=1, H=400, W=1, Cin=256, N=256, taps=((0, 0),), out_kind="planes", a_planes=1, out_planes_n=1, res=True),
    "a1_geglu_p1_wide": dict(B=1, H=1000, W=1, Cin=128, N=1024, taps=((0, 0),), geglu=True, act=_lib.ACT_GEGLU, out_kind="planes",
                             a_planes=1, out_planes_n=1),
    "a1_dual_p2": dict(B=1, H=300, W=1, Cin=1024, N=256, taps=((0, 0),), res=True, dual=True, a_planes=1),
    "a1_conv3x3": dict(B=2, H=20, W=6, Cin=24, N=128, taps=plan.TAPS_3x3, rowvec=True, res=True, a_planes=1),
    "a1_deepK_splitk": dict(B=2, H=8, W=2, Cin=640, N=640, taps=plan.TAPS_3x3, res=True, a_planes=1),
    # many tiles per persistent CTA, ragged last tile
    "a1_long_linear_res": dict(B=1, H=30001, W=1, Cin=128, N=128, taps=((0, 0),), res=True, a_planes=1),
    "long_conv3x3_rowvec": dict(B=8, H=64, W=64, Cin=32, N=128, taps=plan.TAPS_3x3, rowvec=True, res=True),
}

@pytest.mark.parametrize("impl", ["simt", "tc"])
@pytest.mark.parametrize("case", sorted(GEMM_CASES))
def test_gemm_vs_emulator(case, impl):
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    P = Planner(impl=impl, keep_plain=True)
    ios, ins, (kind, o) = _gemm_case(P, g, **GEMM_CASES[case])
    pl = P.finish(ios)
    if case.endswith("deepK_splitk") and impl != "simt":
        assert pl.ops[-1]["splitk"] > 1
    if "a1_" in case:
        assert pl.ops[-1]["a_lo"] is None
    em, prog = run_both(pl, ins)
    ptol = 3e-4 if GEMM_CASES[case].get("out_planes_n", 2) == 1 else 2e-5      # single plane: one-ulp flips of an 11-bit rounding
    if kind == "dual":
        o, dp = o
        assert rel_l2(read_gpu_planes(prog, dp), em.read_planes(dp.hi, dp.lo, dp.rows, dp.Cp)) < ptol
        kind = "f32"
    if kind == "f32":
        want, got = em.f32(o.ref, o.rows * o.C).clone(), read_gpu_f32(prog, o.ref, o.rows * o.C)
    elif kind == "planes":
        want, got = em.read_planes(o.hi, o.lo, o.rows, o.Cp), read_gpu_planes(prog, o)
    else:
        want, got = em.f32(o[0], o[1]).clone(), read_gpu_f32(prog, o[0], o[1])
    assert torch.isfinite(got).all(), f"{case}/{impl}: non-finite output"
    err = rel_l2(got, want)
    assert err < (ptol if kind == "planes" else 2e-5), f"{case}/{impl}: rel L2 {err:.3e}"


@pytest.mark.parametrize("impl", ["simt", "tc"])
@pytest.mark.parametrize("case", ["self", "self_long", "cross_mask", "cross_allmasked", "ragged", "bmod",
                                  "cross8_bmod", "cross32", "cross_tc_33"])
def test_attention(case, impl):
    """Q|K planes + transposed V planes -> attention kernel (wgmma / SIMT checker) vs the emulator."""
    g = torch.Generator().manual_seed(5)
    P = Planner(impl=impl)
    B, heads = 3, 4
    Cc = heads * 32
    # Nk <= 32 takes the CUDA-core short-key kernel (8 / 16 / 32 key instantiations), longer sets the wgmma kernel
    Nq, Nk = dict(self=(200, 200), self_long=(1024, 1024), cross_mask=(70, 9), cross_allmasked=(70, 9), ragged=(33, 130),
                  bmod=(64, 40), cross8_bmod=(300, 8), cross32=(130, 32), cross_tc_33=(130, 33))[case]
    Bkv = 1 if case.endswith("bmod") else B
    selfattn = case.startswith("self")
    ldq = 2 * Cc if selfattn else Cc
    qf = F32(P.raw(B * Nq * ldq * 4), B * Nq, ldq)
    qp = P.prep(_lib.PREP_COPY, qf, n=1)
    ios = dict(q=("f32", qf.ref, (B * Nq, ldq)))
    ins = dict(q=torch.randn(B * Nq, ldq, generator=g))
    vt = P.vt(Bkv, Cc, Nk, 1)
    mk = None
    if selfattn:
        kp, kcol = qp, Cc
    else:
        kf = F32(P.raw(Bkv * Nk * Cc * 4), Bkv * Nk, Cc)
        kp, kcol = P.prep(_lib.PREP_COPY, kf, n=1), 0
        ios["k"] = ("f32", kf.ref, (Bkv * Nk, Cc)); ins["k"] = torch.randn(Bkv * Nk, Cc, generator=g)
        if case != "ragged":
            mk = P.raw(Bkv * Nk * 4)
            m = (torch.rand(Bkv, Nk, generator=g) > 0.4).float(); m[:, 0] = 1
            if case == "cross_allmasked":
                m[1] = 0          # fully-masked row -> uniform weights (SURVEY.md 8a' item 5)
            ios["mask"] = ("f32", mk, (Bkv, Nk)); ins["mask"] = m
    ao = P.planes(B * Nq, Cc, 1)
    P.attn(qp, 0, kp, kcol, vt, ao, B=B, heads=heads, Nq=Nq, Nk=Nk, mask=mk, scale=32 ** -0.5,
           kv_bmod=1 if case.endswith("bmod") else 0)
    pl = P.finish(ios)
    # V^T planes are written directly (in the network they come from an ALDM_OUT_QKV GEMM)
    v = torch.randn(Bkv, Cc, vt.ld_t, generator=g)
    v[:, :, Nk:] = 0
    vh = v.to(torch.float16)
    em = Emulator(pl)
    prog = engine.DeviceProgram(pl, torch.device(DEV), dict(all=(0, len(pl.ops))))
    n = Bkv * Cc * vt.ld_t
    em.f16(vt.hi, n)[:] = vh.reshape(-1)
    prog.ws[vt.hi.off:vt.hi.off + 2 * n].view(torch.float16).copy_(vh.reshape(-1))
    for name, val in ins.items():
        em.write_io(name, val); prog.view(name).copy_(val.to(DEV))
    em.run(); prog.run("all"); torch.cuda.synchronize()
    got, want = read_gpu_planes(prog, ao), em.read_planes(ao.hi, ao.lo, ao.rows, ao.Cp)
    assert torch.isfinite(got).all()
    err = rel_l2(got, want)
    assert err < 5e-4, f"{case}/{impl}: {err:.3e}"


@pytest.mark.parametrize("planes", [2, 1])
@pytest.mark.parametrize("impl", ["simt", "tc"])
@pytest.mark.parametrize("Cc", [64, 128])
def test_gemm_qkv_output(impl, planes, Cc):
    """ALDM_OUT_QKV: Q|K columns as planes (full-line pair stores when single-plane), V columns as transposed planes (keys contiguous,
    pad zeroed); 64- and 128-wide tiles."""
    g = torch.Generator().manual_seed(11)
    P = Planner(impl=impl, keep_plain=True)
    Bt, HW = 3, 37
    rows = Bt * HW
    src = F32(P.raw(rows * Cc * 4), rows, Cc)
    a = P.prep(_lib.PREP_COPY, src, n=planes)
    wm = torch.randn(3 * Cc, Cc, generator=g) / 8
    w = P.wmat(wm, None, 1, Cc, bn=P.bn_for_split(3 * Cc, 2 * Cc))
    qk = P.planes(rows, 2 * Cc, planes)
    vt = P.vt(Bt, Cc, HW, planes)
    P.gemm(a, w, B=1, H=rows, qkv=(qk, vt, 2 * Cc, HW))
    em, prog = run_both(P.finish(dict(src=("f32", src.ref, (rows, Cc)))), dict(src=torch.randn(rows, Cc, generator=g)))
    tol = 2e-5 if planes == 2 else 3e-4
    assert rel_l2(read_gpu_planes(prog, qk), em.read_planes(qk.hi, qk.lo, rows, qk.Cp)) < tol
    n = Bt * Cc * vt.ld_t
    gv = prog.ws[vt.hi.off:vt.hi.off + 2 * n].view(torch.float16).float().cpu()
    ev = em.f16(vt.hi, n).float()
    if planes == 2:
        gv = gv + prog.ws[vt.lo.off:vt.lo.off + 2 * n].view(torch.float16).float().cpu()
        ev = ev + em.f16(vt.lo, n).float()
    assert torch.isfinite(gv).all() and rel_l2(gv, ev) < tol
    assert float(gv.reshape(Bt, Cc, vt.ld_t)[:, :, HW:].abs().max()) == 0.0


def test_softmax_temb_packb():
    g = torch.Generator().manual_seed(6)
    P = Planner(keep_plain=True)
    x = F32(P.raw(40 * 256 * 4), 40, 256)
    sm = P.planes(40, 256)
    P.ops.append(dict(kind="softmax", x=x.ref, out_hi=sm.hi, out_lo=sm.lo, rows=40, n=256, scale=1.0))
    t = P.raw(4 * 8)
    fr = P.vec(torch.exp(-math.log(10000.0) * torch.arange(64, dtype=torch.float32) / 64))
    te = P.planes(4, 128)
    P.ops.append(dict(kind="temb", t=t, freqs=fr, out_hi=te.hi, out_lo=te.lo, B=4, dim=128))
    src = F32(P.raw(100 * 72 * 4), 100, 72)
    dp, dpl = P.raw(128 * 128 * 4), P.raw(128 * 128 * 4)
    P.ops.append(dict(kind="packb", src=src.ref, dst_packed=dp, dst_plain=dpl, lds=72, transpose=0, N=100, K=72, bn=32))
    dp2 = P.raw(128 * 128 * 4)
    P.ops.append(dict(kind="packb", src=src.ref, dst_packed=dp2, dst_plain=None, lds=72, transpose=1, N=72, K=100, bn=64))
    pl = P.finish(dict(x=("f32", x.ref, (40, 256)), t=("i64", t, (4,)), src=("f32", src.ref, (100, 72))))
    em, prog = run_both(pl, dict(x=torch.randn(40, 256, generator=g) * 3, t=torch.tensor([1, 501, 996, 37]),
                                 src=torch.randn(100, 72, generator=g)))
    assert rel_l2(read_gpu_planes(prog, sm), em.read_planes(sm.hi, sm.lo, 40, 256)) < 2e-5
    assert rel_l2(read_gpu_planes(prog, te), em.read_planes(te.hi, te.lo, 4, 128)) < 1e-5
    n1 = packing.round_up(100, 32) * 128 * 4
    assert torch.equal(prog.ws[dp.off:dp.off + n1].cpu(), em.mem["ws"][dp.off:dp.off + n1])       # bit-exact tile images
    n2 = packing.round_up(72, 64) * 128 * 4
    assert torch.equal(prog.ws[dp2.off:dp2.off + n2].cpu(), em.mem["ws"][dp2.off:dp2.off + n2])


@pytest.mark.parametrize("args,n", [((256, 40, 16, 4000, 0, 2000), 4000), ((1024, 160, 64, 16000, 0, 8000), 163840),
                                     ((2048, 480, 256, 48000, 20, 24000), 48000)])
def test_stft_mel_vs_oracle(args, n):
    from oracle import mel as OM
    from tests.golden import cases
    n_fft, hop, n_mels, sr, fmin, fmax = args
    wav = cases.wav_input(n)
    want, _ = OM.stft_mel(wav.numpy(), *args)                       # [1, n_mels, frames]
    basis = torch.from_numpy(OM.mel_filterbank(sr, n_fft, n_mels, fmin, fmax)).to(DEV)
    got = engine.stft_mel(wav.to(DEV).contiguous(), n_fft, hop, basis)            # [1, frames, n_mels]
    assert got.shape[1] == want.shape[2]
    # fp32 FFT vs float64 oracle; log() of small mel energies amplifies relative error a little
    assert rel_l2(got[0].t(), torch.from_numpy(want[0])) < 1e-4
    if n == 163840:
        g = cases.load("stft_16k")                                  # reference TacotronSTFT output
        assert rel_l2(got[0].t(), g["logmel"][0]) < 1e-4


def test_posterior_sample():
    from oracle import functional as OF
    g = torch.Generator().manual_seed(8)
    mom = torch.randn(2, 6, 5, 16, generator=g)                     # NHWC, 2*zc = 16
    noise = torch.randn(2, 8, 6, 5, generator=g)
    want = OF.posterior_sample(mom.permute(0, 3, 1, 2), noise, 0.7)
    got = engine.posterior_sample(mom.to(DEV).contiguous(), noise.to(DEV), 0.7)
    assert rel_l2(got, want) < 1e-6
