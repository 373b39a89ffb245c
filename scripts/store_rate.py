#!/usr/bin/env python
"""SM -> L2 store throughput of the epilogue's access pattern (csrc/microbench.cu: store_rate_kernel).
mode 0 = STG.128 full-line stores from 8 warps, mode 1 = one 8 KB TMA bulk store per warp from shared memory."""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from audioldm2_b200 import _lib  # noqa: E402

torch.zeros(1, device="cuda")
L = _lib.lib()
iters = 256
print(f"{'mode':>5s} {'CTAs':>5s} {'region':>8s} {'B/clk/SM':>9s} {'TB/s chip @1.98GHz':>20s}")
for mode in (0, 1):
    for n in (132, 66, 16, 1):
        for region in (65536 * 4, 65536 * 64):       # 256 KB per CTA (L2-resident), 4 MB per CTA (592 MB total: streams to HBM)
            buf = (C.c_longlong * n)()
            _lib.check(L.aldm_debug_store_rate(n, iters, mode, region, buf), "store_rate")
            cyc = sorted(buf)[len(buf) // 2]
            bpc = iters * 65536 / cyc
            print(f"{mode:5d} {n:5d} {region >> 10:6d}KB {bpc:9.1f} {bpc * n * 1.98e9 / 1e12:20.2f}", flush=True)
