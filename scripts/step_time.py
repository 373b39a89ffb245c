"""ms per DDIM step of the native engine for one configuration (env switches are read at plan / first-launch time, so
every configuration runs in its own process).  Prints one JSON line.

    [ALDM_GN_FUSED=1] [ALDM_BN256=1] python scripts/step_time.py --lanes 2 [--batch 8] [--steps 40] [--model audioldm2-full]
"""
import argparse, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from audioldm2_b200 import arch, model, synth

ap = argparse.ArgumentParser()
ap.add_argument("--lanes", type=int, default=None)
ap.add_argument("--batch", type=int, default=8)
ap.add_argument("--steps", type=int, default=40)
ap.add_argument("--model", default="audioldm2-full")
ap.add_argument("--t5-len", type=int, default=32)
ap.add_argument("--tag", default="")
ap.add_argument("--warm", type=int, default=8, help="DDIM steps of the warm-up / graph-capture call")
ap.add_argument("--reps", type=int, default=3)
a = ap.parse_args()
dev = torch.device("cuda:0")
cfg = arch.model_config(a.model)
eng = model.build_synthetic(a.model, batch=a.batch, device=dev, t5_len=a.t5_len, lanes=a.lanes)
cond, unc = synth.conditioning(cfg, a.batch, seed=77, t5_len=a.t5_len, device=dev)
eng.generate_latent(cond, unc, ddim_steps=a.warm)        # warm-up + graph capture
torch.cuda.synchronize()
best = None
for rep in range(a.reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.manual_seed(rep)
    e0.record(); eng.generate_latent(cond, unc, ddim_steps=a.steps); e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.steps
    best = ms if best is None else min(best, ms)
sw = {k: v for k, v in os.environ.items() if k.startswith("ALDM_")}
print(json.dumps(dict(tag=a.tag, model=a.model, batch=a.batch, lanes=eng.lanes, ms_per_ddim_step=round(best, 3),
                      launches_per_step=eng.launches_per_step(), switches=sw)))
