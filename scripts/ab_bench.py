#!/usr/bin/env python
"""A/B timing of two source trees of this project on one GPU, alternating runs, with a byte comparison of their waveforms.

    python scripts/ab_bench.py --a PARENT_TREE --b NEW_TREE [--runs 3] [--out DIR]

Each tree must already be built (its __graft_entry__.build()).  The script runs, from each tree in turn (a, b, a, b, ...),

    bench.py --steps 2 --warmup 1 --no-cpu-baseline --no-torch-cuda-baseline --dump-outputs DIR

and prints, per run, the benchmark's ms per timed generation and ms per DDIM step, with the card's name, power limit and SM
clock read by `nvidia-smi --query-gpu` right after the run.  Then it compares the dumped waveforms byte for byte: every run
of a tree must reproduce that tree's first waveform, and the two trees must agree, or, when they differ, lie within
--max-rel-l2 of each other (their relative L2 is reported either way).  The last stdout line is a JSON summary.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile


def gpu_info() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        f = [c.strip() for c in r.stdout.splitlines()[0].split(",")]
        return dict(name=f[0], power_limit=f[1], sm_clock=f[2], sm_clock_max=f[3])
    except Exception as e:        # the timing itself does not depend on it
        return dict(error=repr(e))


def run_bench(tree: str, dump: str) -> dict:
    cmd = [sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", "2", "--warmup", "1", "--no-cpu-baseline",
           "--no-torch-cuda-baseline", "--dump-outputs", dump]
    r = subprocess.run(cmd, cwd=tree, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"bench.py failed in {tree} (exit {r.returncode}):\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}")
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")][-1]
    return json.loads(line)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--a", required=True, help="tree root of side A (e.g. the parent commit)")
    ap.add_argument("--b", required=True, help="tree root of side B")
    ap.add_argument("--runs", type=int, default=3, help="runs per tree (at least 3)")
    ap.add_argument("--out", default=None, help="directory for the dumped waveforms (default: a temporary directory)")
    ap.add_argument("--max-rel-l2", type=float, default=0.0,
                    help="accept two trees whose waveforms differ by less than this relative L2 (default: byte-identical only)")
    a = ap.parse_args()
    if a.runs < 3:
        ap.error("--runs must be at least 3")
    out = os.path.abspath(a.out or tempfile.mkdtemp(prefix="ab_bench_"))      # bench.py runs from each tree's root
    trees = dict(a=os.path.abspath(a.a), b=os.path.abspath(a.b))
    res = {k: [] for k in trees}
    for i in range(a.runs):
        for side, tree in trees.items():
            dump = os.path.join(out, f"{side}{i}")
            os.makedirs(dump, exist_ok=True)
            line = run_bench(tree, dump)
            gi = gpu_info()
            step = line["breakdown"]["ms_per_ddim_step"]
            res[side].append(dict(ms_per_generation=line["ms_per_step"], ms_per_ddim_step=step, gpu=gi, dump=dump))
            print(f"run {i} {side}: {line['ms_per_step']:9.1f} ms/generation  {step:7.3f} ms/DDIM step  | {gi}", flush=True)

    def wave(side, i):
        with open(os.path.join(res[side][i]["dump"], "waveform.npy"), "rb") as f:
            return f.read()

    same = {side: all(wave(side, i) == wave(side, 0) for i in range(a.runs)) for side in trees}
    identical = wave("a", 0) == wave("b", 0)
    summary = dict(trees=trees, repeatable=same, waveforms_byte_identical=identical)
    if not identical:     # e.g. a change that reorders fp32 sums: how far apart the two trees' waveforms are
        import numpy as np
        wa, wb = (np.load(os.path.join(res[s][0]["dump"], "waveform.npy")).astype(np.float64) for s in ("a", "b"))
        summary["waveform_rel_l2_b_vs_a"] = float(np.linalg.norm(wb - wa) / np.linalg.norm(wa))
    for side in trees:
        gen = [r["ms_per_generation"] for r in res[side]]
        step = [r["ms_per_ddim_step"] for r in res[side]]
        summary[side] = dict(ms_per_generation=gen, ms_per_ddim_step=step, median_ms_per_generation=statistics.median(gen),
                             median_ms_per_ddim_step=statistics.median(step),
                             spread_ms_per_generation=max(gen) - min(gen))
    summary["b_over_a_ms_per_generation"] = summary["b"]["median_ms_per_generation"] / summary["a"]["median_ms_per_generation"]
    summary["b_over_a_ms_per_ddim_step"] = summary["b"]["median_ms_per_ddim_step"] / summary["a"]["median_ms_per_ddim_step"]
    summary["gpu"] = gpu_info()
    print(json.dumps(summary))
    if not all(same.values()) or not (identical or summary["waveform_rel_l2_b_vs_a"] < a.max_rel_l2):
        sys.exit(1)


if __name__ == "__main__":
    main()
