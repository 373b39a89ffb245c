"""Time the native AudioMAE token generator (GPU only; there is no CPU fallback).

For B in {1, 8} and L in {32, 128}: the native stage as one CUDA-graph replay, and its prefill and decode ranges as
separate graphs; the reference algorithm on the same GPU (oracle/seqgen.py in fp32 torch-CUDA: 8 full GPT-2 forward
passes without a cache, as Sequence2AudioMAE.generate runs them); and the decode passes' achieved weight bandwidth
(packed weight bytes streamed per decode pass / decode time per pass).  Prints the card and its power limit and
writes JSON (default ./seqgen_time.json).

    python scripts/seqgen_time.py [--reps 20] [--out PATH]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch                                            # noqa: E402

from audioldm2_b200 import synth                        # noqa: E402
from audioldm2_b200.seqgen import NativeAudioMAEGenerator  # noqa: E402
from oracle import seqgen as OS                         # noqa: E402


def _time(fn, reps: int) -> float:
    fn(); fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def card() -> dict:
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, timeout=30).stdout.decode().strip().split(",")
        return dict(name=name, power_limit_w=float(q[0]), max_sm_clock_mhz=float(q[1]))
    except Exception:
        return dict(name=name, power_limit_w=None, max_sm_clock_mhz=None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="seqgen_time.json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("seqgen_time.py needs a CUDA device")
    info = card()
    print(f"card: {info['name']}, power limit {info['power_limit_w']} W")
    sd = synth.seqgen_state_dict()
    gen = NativeAudioMAEGenerator(sd, "cuda:0")
    sd_dev = {k: v.cuda() for k, v in sd.items() if k != "model.wte.weight"}
    # packed weights streamed per decode pass: the 48 GPT-2 matrices (two fp16 planes); embeddings and norms are negligible
    refs = gen.weights.refs
    w_bytes = sum(r.N * r.Kpad * 4 for k, r in refs.items() if "." in k and hasattr(r, "Kpad") and k.split(".")[0].isdigit())
    rows = []
    for B in (1, 8):
        for L in (32, 128):
            clap, t5, mask = (t.cuda() for t in synth.encoder_outputs(B, [L] * B, seed=3))
            gen.generate(clap, t5, mask)
            prog = gen.program(B, L)
            t_all = _time(lambda: prog.replay("all"), a.reps)
            t_pre = _time(lambda: prog.replay("prefill"), a.reps)
            t_dec = _time(lambda: prog.replay("decode"), a.reps)
            with torch.no_grad():
                t_ref = _time(lambda: OS.audiomae_generate(sd_dev, clap, t5, mask, 12), max(3, a.reps // 4))
            per_pass = t_dec / 7
            r = dict(B=B, L=L, native_ms=t_all, prefill_ms=t_pre, decode_ms=t_dec, decode_pass_ms=per_pass,
                     reference_no_cache_fp32_ms=t_ref, speedup=t_ref / t_all, decode_weight_gbps=w_bytes / (per_pass * 1e-3) / 1e9,
                     launches=int(prog.num_launches("all")))
            rows.append(r)
            print(f"B={B} L={L}: native {t_all:.3f} ms (prefill {t_pre:.3f}, 7 decode passes {t_dec:.3f}; {r['launches']} launches), "
                  f"reference algorithm fp32 {t_ref:.2f} ms -> {r['speedup']:.1f}x; decode weight stream "
                  f"{r['decode_weight_gbps']:.0f} GB/s ({w_bytes / 1e6:.0f} MB per pass)")
            gen._progs.clear()
            torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    json.dump(dict(card=info, weight_bytes_per_pass=w_bytes, rows=rows), open(a.out, "w"), indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
