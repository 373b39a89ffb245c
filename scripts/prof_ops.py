#!/usr/bin/env python
"""Micro-benchmark / ncu target: the dominant UNet op shapes (audioldm2-full, 2*B_l = 16), each op
launched back-to-back many times between two CUDA events (steady state, no launch-gap artefacts).

    python scripts/prof_ops.py [--reps 40] [--only NAME] [--impl tc]
    ncu --set full -k regex:gemm_tc2 ... python scripts/prof_ops.py --reps 2 --only lin_k256_n256
"""
import argparse
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from audioldm2_b200 import _lib, engine, plan  # noqa: E402
from audioldm2_b200.plan import F32, Planner  # noqa: E402

CASES = {
    # name: (kind, params)
    "lin_k256_n256": ("gemm", dict(B=1, H=16384, W=1, Cin=256, N=256, taps=((0, 0),), res=True)),
    "lin_k256_n256_pln": ("gemm", dict(B=1, H=16384, W=1, Cin=256, N=256, taps=((0, 0),), pln=True)),
    "lin_k256_n2048_geglu": ("gemm", dict(B=1, H=16384, W=1, Cin=256, N=2048, taps=((0, 0),), geglu=True)),
    "lin_k256_n768_qkv": ("gemm", dict(B=1, H=16384, W=1, Cin=256, N=768, taps=((0, 0),), qkv=1024)),
    "lin_k1024_n256": ("gemm", dict(B=1, H=16384, W=1, Cin=1024, N=256, taps=((0, 0),), res=True)),
    "lin_k384_n384": ("gemm", dict(B=1, H=4096, W=1, Cin=384, N=384, taps=((0, 0),), res=True)),
    "lin_k640_n640": ("gemm", dict(B=1, H=1024, W=1, Cin=640, N=640, taps=((0, 0),), res=True)),
    "lin_k640_n5120_geglu": ("gemm", dict(B=1, H=1024, W=1, Cin=640, N=5120, taps=((0, 0),), geglu=True)),
    "conv_l1_128": ("gemm", dict(B=16, H=256, W=16, Cin=128, N=128, taps=plan.TAPS_3x3, res=True)),
    "conv_l2_256": ("gemm", dict(B=16, H=128, W=8, Cin=256, N=256, taps=plan.TAPS_3x3, res=True)),
    "conv_l1_128_k2304": ("gemm", dict(B=16, H=256, W=16, Cin=256, N=128, taps=plan.TAPS_3x3, res=True)),
    "conv_l1_128_k3456": ("gemm", dict(B=16, H=256, W=16, Cin=384, N=128, taps=plan.TAPS_3x3, res=True)),
    "conv_l2_256_k5760": ("gemm", dict(B=16, H=128, W=8, Cin=640, N=256, taps=plan.TAPS_3x3, res=True)),
    "conv_l2_256_k4608": ("gemm", dict(B=16, H=128, W=8, Cin=512, N=256, taps=plan.TAPS_3x3, res=True)),
    "conv_up_l1_256": ("gemm", dict(B=16, H=256, W=16, Cin=256, N=256, taps=plan.TAPS_3x3, up=1)),
    "conv_l4_640": ("gemm", dict(B=16, H=32, W=2, Cin=640, N=640, taps=plan.TAPS_3x3, res=True)),
    "attn_1024": ("attn", dict(B=16, heads=8, N=1024)),
    "attn_256": ("attn", dict(B=16, heads=12, N=256)),
    "attn_64": ("attn", dict(B=16, heads=20, N=64)),
    "ln_16384x256": ("prep", dict(rows=16384, C=256, mode=_lib.PREP_LN)),
    "gn_silu_l1": ("prep", dict(rows=65536, C=128, mode=_lib.PREP_GN_SILU, B=16)),
    "gn_silu_l4": ("prep", dict(rows=1024, C=640, mode=_lib.PREP_GN_SILU, B=16)),
}


TOK = 1      # planes of the token-side operands (--planes)


def build(name, impl):
    kind, p = CASES[name]
    tok = TOK if name.startswith(("lin_", "ln_")) else 2
    g = torch.Generator().manual_seed(0)
    P = Planner(impl=impl)
    ios, ins = {}, {}
    flops = 0.0
    if kind == "gemm":
        B, H, W, Cin, N, taps = p["B"], p["H"], p["W"], p["Cin"], p["N"], p["taps"]
        src = F32(P.raw(B * H * W * Cin * 4), B * H * W, Cin)
        a = P.prep(_lib.PREP_COPY, src, n=tok)
        first = len(P.ops)
        wm = torch.randn(N, len(taps) * Cin, generator=g) / math.sqrt(len(taps) * Cin)
        M = B * H * W
        kw = dict(B=B, H=H, W=W, taps=taps, up=p.get("up", 0))
        if p.get("geglu"):
            w = P.wmat(wm, torch.zeros(N), len(taps), Cin, geglu=True)
            P.gemm(a, w, out_planes=P.planes(M, N // 2, tok), act=_lib.ACT_GEGLU, **kw)
        elif p.get("pln"):
            w = P.wmat(wm, torch.zeros(N), len(taps), Cin)
            P.gemm(a, w, out_planes=P.planes(M, N, tok), **kw)
        elif p.get("qkv"):
            Cc = N // 3
            w = P.wmat(wm, None, len(taps), Cin, bn=P.bn_for_split(N, 2 * Cc))
            P.gemm(a, w, qkv=(P.planes(M, 2 * Cc, tok), P.vt(M // p["qkv"], Cc, p["qkv"], tok), 2 * Cc, p["qkv"]), **kw)
        else:
            w = P.wmat(wm, torch.zeros(N), len(taps), Cin)
            r = P.f32(M, N) if p.get("res") else None
            P.gemm(a, w, out=P.f32(M, N), res=r, **kw)
            if r is not None:
                ios["res"] = ("f32", r.ref, (M, N)); ins["res"] = torch.zeros(M, N)
        ios["src"] = ("f32", src.ref, (src.rows, Cin)); ins["src"] = torch.randn(src.rows, Cin, generator=g)
        flops = 2.0 * M * N * len(taps) * Cin
    elif kind == "attn":
        B, h, N = p["B"], p["heads"], p["N"]
        Cc = h * 32
        src = F32(P.raw(B * N * 2 * Cc * 4), B * N, 2 * Cc)
        qk = P.prep(_lib.PREP_COPY, src, n=1)
        vt = P.vt(B, Cc, N, 1)
        first = len(P.ops)
        P.attn(qk, 0, qk, Cc, vt, P.planes(B * N, Cc, 1), B=B, heads=h, Nq=N, Nk=N, mask=None, scale=32 ** -0.5)
        ios["src"] = ("f32", src.ref, (B * N, 2 * Cc)); ins["src"] = torch.randn(B * N, 2 * Cc, generator=g)
        flops = 4.0 * B * h * N * N * 32
    else:
        rows, Cc = p["rows"], p["C"]
        src = F32(P.raw(rows * Cc * 4), rows, Cc)
        first = len(P.ops)
        gam, bet = P.vec(torch.ones(Cc)), P.vec(torch.zeros(Cc))
        P.prep(p["mode"], src, None, gam, bet, eps=1e-5, B=p.get("B", 0), HW=rows // max(1, p.get("B", 1)), n=tok)
        ios["src"] = ("f32", src.ref, (rows, Cc)); ins["src"] = torch.randn(rows, Cc, generator=g)
        flops = 0.0
    pl = P.finish(ios)
    arr = pl.resolve(1 << 32, 1 << 40)        # placeholder addresses: enough for the A-mode query
    nbytes = sum(operand_bytes(o, _lib.gemm_a_mode(arr[i].u.gemm)) for i, o in enumerate(pl.ops) if i >= first and o["kind"] == "gemm")
    return pl, ins, first, flops, nbytes


def operand_bytes(o, amode=_lib.AMODE_GATHER) -> int:
    """Bytes one GEMM launch moves from L2 into shared memory: every 128-row tile gathers its A rows (K fp16 values per
    plane) and receives its own copy of the [hi | lo] weight image of its N tile (Kpad x bn x 2 planes).  In halo mode a
    tile (64 columns wide) loads its 180-pixel halo once per 64-channel block instead of 9 x 128 pixel rows."""
    M = o["B"] * o["OH"] * o["OW"]
    bn = 64 if amode == _lib.AMODE_HALO else o["bn"]       # the halo kernel runs 64-wide N tiles
    tiles_m, tiles_n = math.ceil(M / 128), math.ceil(o["N"] / bn)
    ap = 2 if o["a_lo"] is not None else 1
    a_rows = 180 * o["K"] // len(o["taps"]) if amode == _lib.AMODE_HALO else 128 * o["K"]
    return tiles_m * tiles_n * (a_rows * 2 * ap + bn * o["Kpad"] * 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=40)
    ap.add_argument("--only", default=None)
    ap.add_argument("--impl", default="tc")
    ap.add_argument("--planes", type=int, default=1, help="planes of the token-side operands (lin_* / ln_* cases)")
    ap.add_argument("--dbg", type=int, default=0, help="GEMM profiling aid bits: 1 skip A loads, 2 skip B loads, 4 skip MMA, 8 skip epilogue")
    a = ap.parse_args()
    global TOK
    TOK = a.planes
    dev = torch.device("cuda:0")
    print(f"{'case':28s} {'us/launch':>10s} {'TFLOP/s':>9s} {'A+B MB':>8s} {'A+B TB/s':>9s}")
    for name in CASES:
        if a.only and name not in a.only.split(","):
            continue
        pl, ins, first, flops, nbytes = build(name, a.impl)
        if a.dbg:
            for o in pl.ops:
                if o["kind"] == "gemm":
                    o["impl"] = o["impl"] | (a.dbg << 8)
        if first == 0:      # no setup op: insert a harmless copy so the range is not empty
            pl.ops.insert(0, dict(kind="copy", src=plan.Ref("ws", 0), dst=plan.Ref("ws", 0), bytes=0)); first = 1
        prog = engine.DeviceProgram(pl, dev, dict(setup=(0, first), op=(first, len(pl.ops))))
        for k, v in ins.items():
            prog.view(k).copy_(v.to(dev))
        prog.run("setup"); prog.run("op"); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps):
            prog.run("op")
        e1.record(); torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / a.reps
        print(f"{name:28s} {us:10.1f} {flops / (us * 1e-6) / 1e12 if flops else 0:9.1f} {nbytes / 1e6:8.1f} "
              f"{nbytes / (us * 1e-6) / 1e12:9.2f}", flush=True)
        if a.dbg & 128:
            import ctypes as C
            buf = (C.c_longlong * (4 * 256 * 2))()
            _lib.check(_lib.lib().aldm_debug_timeline(buf, 4 * 256 * 2), "timeline")
            t = torch.tensor(list(buf), dtype=torch.int64).reshape(4, 256, 2)
            t0 = int(t[t > 0].min())
            print("  iter | prod: wait_done issued | B: wait_done | MMA: full_seen committed | (cycles since first event)")
            for i in range(0, 40):
                r = lambda x: (int(x) - t0) if int(x) > 0 else -1
                print(f"  {i:4d} | {r(t[0, i, 0]):7d} {r(t[0, i, 1]):7d} | {r(t[1, i, 0]):7d} | {r(t[2, i, 0]):7d} {r(t[2, i, 1]):7d}")
            print("  tile | epi: prologue_done tfull_seen | ch0: ld_done staged res_issued emitted | ch1: ld_done staged res_issued emitted | done"
                  "   (GEGLU: ld_done gelu_done staged emitted)")
            for i in range(0, 4):
                f = [r(t[3, 64 + i * 8 + k, ph]) for k in range(1, 5) for ph in (0, 1)]
                print(f"  {i:4d} | {r(t[3, 64 + i * 8, 0]):7d} {r(t[3, i, 0]):7d} | " + " ".join(f"{x:7d}" for x in f[:4]) + " | " +
                      " ".join(f"{x:7d}" for x in f[4:]) + f" | {r(t[3, i, 1]):7d}")


if __name__ == "__main__":
    main()
