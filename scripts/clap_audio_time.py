"""Time the native CLAP audio encoder (GPU only; there is no CPU fallback).

For n in {3, 12, 24} clips of 10.24 s at 16 kHz (the re-ranker's input at batchsize 1, 4 and 8 with 3 candidates): the
native encoder as one CUDA-graph replay of the (n, L, 16 kHz) plan (median over many replays, CUDA events, after
warm-up), against the reference computation on the same GPU (oracle/clap_audio.py in torch-CUDA: torchaudio's resample as
a conv1d, the STFT as a matmul with the DFT basis as torchlibrosa does, HTSAT-base, audio_projection) in fp32 and with
TF32 matmuls.  Prints the card and its power limit and writes JSON (default ./clap_audio_time.json).

    python scripts/clap_audio_time.py [--reps 50] [--out PATH]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch                                            # noqa: E402

from audioldm2_b200 import synth                        # noqa: E402
from audioldm2_b200.clap import NativeCLAPAudioEncoder  # noqa: E402
from oracle import clap_audio as OA                     # noqa: E402
from tests.golden.clap_audio_cases import waveform      # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "scripts"))
from seqgen_time import _time, card                     # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default="clap_audio_time.json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("clap_audio_time.py needs a CUDA device")
    info = card()
    print(f"card: {info['name']}, power limit {info['power_limit_w']} W")
    sd = synth.clap_audio_state_dict()
    enc = NativeCLAPAudioEncoder(sd, "cuda:0", sampling_rate=16000)
    sd_dev = {k: v.cuda() for k, v in sd.items()}
    L = 163840
    rows = []
    for n in (3, 12, 24):
        wav = waveform(n, L, seed=n).cuda()
        e = enc.embed(wav)
        prog = enc.program(n, L)
        t_nat = _time(lambda: prog.replay("all"), a.reps)
        r = dict(n=n, seconds=L / 16000, native_ms=t_nat, launches=int(prog.num_launches("all")))
        with torch.no_grad():
            for name, tf32 in (("fp32", False), ("tf32", True)):
                torch.backends.cuda.matmul.allow_tf32 = tf32
                torch.backends.cudnn.allow_tf32 = tf32
                r[f"reference_{name}_ms"] = _time(lambda: OA.clap_audio_embed(sd_dev, wav, 16000, dtype=torch.float32,
                                                                              device="cuda"), a.reps)
            torch.backends.cuda.matmul.allow_tf32 = False
            torch.backends.cudnn.allow_tf32 = False
            ref = OA.clap_audio_embed(sd_dev, wav, 16000, dtype=torch.float32, device="cuda")
        r["rel_l2_vs_fp32_reference"] = float((e - ref).norm() / ref.norm())
        rows.append(r)
        print(f"n={n} x 10.24 s: native {t_nat:.3f} ms ({r['launches']} launches); reference fp32 "
              f"{r['reference_fp32_ms']:.3f} ms ({r['reference_fp32_ms'] / t_nat:.2f}x), TF32 {r['reference_tf32_ms']:.3f} ms "
              f"({r['reference_tf32_ms'] / t_nat:.2f}x); rel L2 vs fp32 {r['rel_l2_vs_fp32_reference']:.2e}")
        while enc._progs:                                # free the plan's graph and workspace before the next n
            enc._progs.popitem()[1].close()
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    json.dump(dict(card=info, rows=rows), open(a.out, "w"), indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
