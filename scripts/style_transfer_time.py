"""Style transfer against a full generation on the native engine, in one process (GPU only; there is no CPU fallback).

At audioldm2-full, batch 8, S = 200, seeded synthetic weights and conditioning: the whole audio-to-audio path (VAE
encoder, posterior sample, the device-side latent guard, stochastic_encode, t_enc = strength * S DDIM steps, decoder
and vocoder) at strengths 0.25 / 0.5 / 0.75, against the same engine's 200-step generation with decoder and vocoder
(text_to_audio's sampling path).  Each figure is the median of --reps runs timed with CUDA events after a warm-up run of
every shape; the calls alternate.  Prints the card and its power limit and writes JSON (default ./style_transfer_time.json).

    python scripts/style_transfer_time.py [--batch 8] [--steps 200] [--reps 3] [--out PATH]
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

from audioldm2_b200 import arch, model, parallel, synth   # noqa: E402
from audioldm2_b200.sampler import transfer_steps       # noqa: E402
from seqgen_time import card                            # noqa: E402

STRENGTHS = (0.25, 0.5, 0.75)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--model", default="audioldm2-full")
    ap.add_argument("--out", default="style_transfer_time.json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("style_transfer_time.py needs a CUDA device")
    info = card()
    print(f"card: {info['name']}, power limit {info['power_limit_w']} W")
    dev = torch.device("cuda:0")
    cfg = arch.model_config(a.model)
    B, S = a.batch, a.steps
    eng = model.build_synthetic(a.model, batch=B, device=dev, t5_len=32, with_encoder=True)
    cond, unc = synth.conditioning(cfg, B, seed=77, t5_len=32, device=dev)
    C_, T, F_ = cfg["latent"]
    ds = 2 ** (len(cfg["vae"]["ch_mult"]) - 1)
    mel = torch.randn(B, 1, T * ds, F_ * ds, generator=torch.Generator().manual_seed(9)).to(dev) - 5.0

    def style(strength):
        post = torch.randn(B, C_, T, F_)                 # the CPU posterior draw, as the pipeline makes it
        x0 = eng.get_first_stage_encoding(eng.encode_first_stage_moments(mel), post)
        return eng.style_transfer_waveform(x0, cond, unc, transfer_steps(strength, S), ddim_steps=S, guidance=2.5,
                                           clip_flag=parallel.latent_guard_flag(x0))

    def generate():
        return eng.generate_waveform(cond, unc, ddim_steps=S, guidance=3.5)

    runs = {f"style_{s}": (lambda s=s: style(s)) for s in STRENGTHS}
    runs["generate"] = generate
    for fn in runs.values():                             # warm-up: module load, graph capture, every shape
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in runs}
    for rep in range(a.reps):
        for k, fn in runs.items():
            torch.manual_seed(rep)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record()
            e1.synchronize()
            times[k].append(e0.elapsed_time(e1))
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    gen = med["generate"]
    res = dict(card=info, model=a.model, batch=B, steps=S, reps=a.reps, generate_ms=round(gen, 1))
    print(f"{'call':<22} {'DDIM steps':>10} {'ms':>9} {'vs generation':>14}")
    print(f"{'generation S=' + str(S):<22} {S:>10} {gen:>9.1f} {1.0:>13.2f}x")
    for s in STRENGTHS:
        t = med[f"style_{s}"]
        res[f"style_{s}_ms"] = round(t, 1)
        print(f"{'style strength ' + str(s):<22} {transfer_steps(s, S):>10} {t:>9.1f} {t / gen:>13.3f}x")
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    json.dump(res, open(a.out, "w"), indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
