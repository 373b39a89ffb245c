"""Time the native CLAP text encoder (GPU only; there is no CPU fallback).

For B in {1, 8} and L_eff in {16, 77, 512} (every row holds L_eff tokens, padded to the tokenizer's 512), 12 blocks: the
native encoder as one CUDA-graph replay of the (B, L_eff) plan (median over many replays, CUDA events, after warm-up),
against the reference computation on the same GPU at the reference's padded 512 positions (oracle/clap.py in
torch-CUDA, the operations HF RobertaModel, the pooler, text_projection and F.normalize run) in fp32 and with TF32
matmuls.  Prints the card and its power limit and writes JSON (default ./clap_time.json).

    python scripts/clap_time.py [--reps 50] [--out PATH]
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
from audioldm2_b200.clap import NativeCLAPTextEncoder   # noqa: E402
from oracle import clap as OC                           # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "scripts"))
from seqgen_time import _time, card                     # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default="clap_time.json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("clap_time.py needs a CUDA device")
    info = card()
    print(f"card: {info['name']}, power limit {info['power_limit_w']} W")
    sd = synth.clap_text_state_dict()
    enc = NativeCLAPTextEncoder(sd, "cuda:0")
    sd_dev = {k: v.cuda() for k, v in sd.items()}
    rows = []
    for B in (1, 8):
        for L in (16, 77, 512):
            ids, mask = (t.cuda() for t in synth.clap_token_ids([L] * B, seed=3))
            e = enc.embed(ids, mask)
            prog = enc.program(B, L)
            t_nat = _time(lambda: prog.replay("all"), a.reps)
            r = dict(B=B, L_eff=L, native_ms=t_nat, launches=int(prog.num_launches("all")))
            with torch.no_grad():
                for name, tf32 in (("fp32", False), ("tf32", True)):
                    torch.backends.cuda.matmul.allow_tf32 = tf32
                    r[f"reference_{name}_ms"] = _time(lambda: OC.clap_text_embed(sd_dev, ids, mask, 12, dtype=torch.float32,
                                                                                 device="cuda"), max(5, a.reps // 5))
                torch.backends.cuda.matmul.allow_tf32 = False
                ref = OC.clap_text_embed(sd_dev, ids, mask, 12, dtype=torch.float32, device="cuda")
            r["rel_l2_vs_fp32_reference"] = float((e - ref).norm() / ref.norm())
            rows.append(r)
            print(f"B={B} L_eff={L}: native {t_nat:.3f} ms ({r['launches']} launches); reference (512 positions) fp32 "
                  f"{r['reference_fp32_ms']:.3f} ms ({r['reference_fp32_ms'] / t_nat:.2f}x), TF32 {r['reference_tf32_ms']:.3f} ms "
                  f"({r['reference_tf32_ms'] / t_nat:.2f}x); rel L2 vs fp32 {r['rel_l2_vs_fp32_reference']:.2e}")
            enc._progs.clear()
            torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    json.dump(dict(card=info, rows=rows), open(a.out, "w"), indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
