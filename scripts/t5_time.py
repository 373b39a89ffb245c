"""Time the native Flan-T5 encoder (GPU only; there is no CPU fallback).

For B in {1, 8} and L in {32, 128}, 24 blocks: the native encoder as one CUDA-graph replay (median over many replays,
CUDA events, after warm-up), against the reference computation on the same GPU (oracle/t5.py in torch-CUDA, the
operations HF T5EncoderModel runs) in fp32 and with TF32 matmuls.  Prints the card and its power limit and writes JSON
(default ./t5_time.json).

    python scripts/t5_time.py [--reps 50] [--out PATH]
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
from audioldm2_b200.t5 import NativeFlanT5Encoder       # noqa: E402
from oracle import t5 as OT                             # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "scripts"))
from seqgen_time import _time, card                     # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default="t5_time.json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("t5_time.py needs a CUDA device")
    info = card()
    print(f"card: {info['name']}, power limit {info['power_limit_w']} W")
    sd = synth.t5_state_dict()
    enc = NativeFlanT5Encoder(sd, "cuda:0")
    sd_dev = {k: v.cuda() for k, v in sd.items() if k != "encoder.embed_tokens.weight"}
    rows = []
    for B in (1, 8):
        for L in (32, 128):
            ids, mask = (t.cuda() for t in synth.token_ids([L] * B, seed=3))
            h = enc.encode(ids, mask)
            prog = enc.program(B, L)
            t_nat = _time(lambda: prog.replay("all"), a.reps)
            r = dict(B=B, L=L, native_ms=t_nat, launches=int(prog.num_launches("all")))
            with torch.no_grad():
                for name, tf32 in (("fp32", False), ("tf32", True)):
                    torch.backends.cuda.matmul.allow_tf32 = tf32
                    r[f"reference_{name}_ms"] = _time(lambda: OT.t5_encode(sd_dev, ids, mask, 24, dtype=torch.float32,
                                                                           device="cuda"), max(5, a.reps // 5))
                torch.backends.cuda.matmul.allow_tf32 = False
                ref = OT.t5_encode(sd_dev, ids, mask, 24, dtype=torch.float32, device="cuda")
            r["rel_l2_vs_fp32_reference"] = float((h - ref).norm() / ref.norm())
            rows.append(r)
            print(f"B={B} L={L}: native {t_nat:.3f} ms ({r['launches']} launches); reference fp32 {r['reference_fp32_ms']:.3f} ms "
                  f"({r['reference_fp32_ms'] / t_nat:.2f}x), TF32 {r['reference_tf32_ms']:.3f} ms "
                  f"({r['reference_tf32_ms'] / t_nat:.2f}x); rel L2 vs fp32 {r['rel_l2_vs_fp32_reference']:.2e}")
            enc._progs.clear()
            torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    json.dump(dict(card=info, rows=rows), open(a.out, "w"), indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
