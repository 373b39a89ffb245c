"""PLMS against DDIM on the native engine, in one process (GPU only; there is no CPU fallback).

At audioldm2-full, batch 8 (the benchmark's latent batch), seeded synthetic weights and conditioning: ms per PLMS step
against ms per DDIM step over the same number of steps, and whole-sampler time of S-step PLMS generations (S = 25, 50:
S + 1 UNet pairs each) against the default 200-step DDIM run.  Each figure is the median of --reps runs timed with CUDA
events after a warm-up (graph capture) run; DDIM and PLMS runs alternate.  Prints the card and its power limit and writes
JSON (default ./plms_time.json).

    python scripts/plms_time.py [--batch 8] [--steps 40] [--reps 3] [--out PATH]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch                                            # noqa: E402

from audioldm2_b200 import arch, model, synth           # noqa: E402
from seqgen_time import card                            # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=40, help="steps of the per-step comparison")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--model", default="audioldm2-full")
    ap.add_argument("--out", default="plms_time.json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("plms_time.py needs a CUDA device")
    info = card()
    print(f"card: {info['name']}, power limit {info['power_limit_w']} W")
    dev = torch.device("cuda:0")
    cfg = arch.model_config(a.model)
    eng = model.build_synthetic(a.model, batch=a.batch, device=dev, t5_len=32)
    cond, unc = synth.conditioning(cfg, a.batch, seed=77, t5_len=32, device=dev)
    run = lambda S, plms: eng.generate_latent(cond, unc, ddim_steps=S, guidance=3.5, use_plms=plms)
    run(8, False)                                       # warm-up: module load, graph capture
    run(8, True)
    torch.cuda.synchronize()

    def timed(S, plms):
        ts = []
        for rep in range(a.reps):
            torch.manual_seed(rep)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); run(S, plms); e1.record()
            e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        return sorted(ts)[len(ts) // 2]

    # per step: S DDIM steps are S UNet pairs, S PLMS steps are S + 1
    ddim_ms, plms_ms = timed(a.steps, False), timed(a.steps, True)
    res = dict(card=info, model=a.model, batch=a.batch, steps=a.steps,
               ms_per_ddim_step=round(ddim_ms / a.steps, 3), ms_per_plms_step=round(plms_ms / a.steps, 3),
               ms_per_plms_unet_pair=round(plms_ms / (a.steps + 1), 3))
    print(f"batch {a.batch}, {a.steps} steps: DDIM {res['ms_per_ddim_step']:.3f} ms/step, PLMS {res['ms_per_plms_step']:.3f} "
          f"ms/step ({res['ms_per_plms_unet_pair']:.3f} ms per UNet pair, {a.steps + 1} pairs)")
    ddim200 = timed(200, False)
    res["ddim_200_ms"] = round(ddim200, 1)
    print(f"{'sampler':<12} {'UNet pairs':>10} {'ms':>9} {'vs DDIM 200':>12}")
    print(f"{'DDIM 200':<12} {200:>10} {ddim200:>9.1f} {1.0:>11.2f}x")
    for S in (25, 50):
        t = timed(S, True)
        res[f"plms_{S}_ms"] = round(t, 1)
        print(f"{'PLMS ' + str(S):<12} {S + 1:>10} {t:>9.1f} {ddim200 / t:>11.2f}x")
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    json.dump(res, open(a.out, "w"), indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
