"""Generate the PLMS fixtures by running the UNMODIFIED reference PLMSSampler (latent_diffusion/models/plms.py).

Run where the reference package is importable (oracle/ref_loader.py):

    python tests/golden/make_plms_golden.py [--only NAME]

The sampler runs on CPU in fp32 over the reference UNet (strict-loaded with the seeded synthetic weights, as
make_golden.py does) through a stub model.  The reference's schedule, coefficients, first-step improved-Euler pass and
RNG draws are all its own code.  Two details of the stub:

* the sampler instance's ``register_buffer`` keeps tensors on the CPU (the reference moves every buffer to cuda);
* at guidance != 1 the stub's ``apply_model`` returns ``unet(x, t, uc) + s (unet(x, t, c) - unet(x, t, uc))``, the
  reference UNet called twice as ddim.py:293-300 does, and the sampler runs at scale 1.0 around it: the reference's own
  guided PLMS path concatenates AudioLDM2's dict conditioning with torch.cat and raises (plms.py:290).

After each loop ``rng_after = torch.randn(4)`` is stored, so that tests can check how many draws the loop made.
"""
from __future__ import annotations

import argparse
import importlib
import os
import sys
import time

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from audioldm2_b200 import arch                                       # noqa: E402
from oracle import functional as OF                                   # noqa: E402
from oracle import ref_loader                                         # noqa: E402
from tests.golden import cases                                        # noqa: E402
from tests.golden.make_golden import _StubModel, _save, ref_unet, ref_vae, ref_vocoder   # noqa: E402


class _GuidedStub(_StubModel):
    """apply_model with the DDIM combine of ddim.py:293-300 folded in (guidance 1: the conditional branch alone)."""

    def __init__(self, unet, tables, uncond, scale):
        super().__init__(unet, tables)
        self.uncond, self.scale = uncond, scale

    def apply_model(self, x, t, c):
        e_c = super().apply_model(x, t, c)
        if self.uncond is None:
            return e_c
        e_u = super().apply_model(x, t, self.uncond)
        return e_u + self.scale * (e_c - e_u)


@torch.no_grad()
def gen_plms(R, name, cfg, B, S, guidance=3.5, masked=False, with_audio=False, t5_len=32):
    m = ref_unet(R, cfg["unet"])
    tables = OF.ddpm_tables(cfg["linear_start"], cfg["linear_end"], cfg["timesteps"])
    _, _, cond, unc = cases.unet_inputs(cfg, B, t5_len=t5_len)
    stub = _GuidedStub(m, tables, unc if guidance != 1.0 else None, guidance)
    sampler = R.PLMSSampler(stub)
    sampler.register_buffer = lambda n, attr: setattr(sampler, n, attr)
    C, T, Fq = cfg["latent"]
    mask = x0 = None
    if masked:
        mask, x0 = cases.inpaint_mask(cfg, B)
    torch.manual_seed(cases.SAMPLER_SEED)
    t0 = time.time()
    # sample()'s two calls (plms.py:130-153; its batch-size printout reads .shape of the first conditioning entry, a
    # list here).  generate_batch passes eta 1.0, which make_schedule replaces by 0; at guidance 1.0 the unconditional
    # dict is passed and ignored, the reference path exactly as it runs
    sampler.make_schedule(ddim_num_steps=S, ddim_eta=1.0, verbose=False)
    img, _ = sampler.plms_sampling(cond, (B, C, T, Fq), mask=mask, x0=x0, unconditional_guidance_scale=1.0,
                                   unconditional_conditioning=unc if guidance == 1.0 else None)
    out = dict(latent=img, rng_after=torch.randn(4))
    print(f"  {name}: S={S} in {time.time() - t0:.1f}s")
    if with_audio:
        dec, _, sd = ref_vae(R, cfg["vae"])
        h = torch.nn.functional.conv2d(img, sd["post_quant_conv.weight"], sd["post_quant_conv.bias"])
        mel = dec(h)
        wave = ref_vocoder(R, cfg["vocoder"])(mel.squeeze(1).permute(0, 2, 1))        # ddpm.py:932-935
        out["mel"], out["wave"] = mel, wave
    _save(name, out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default=None)
    a = ap.parse_args()
    torch.set_num_threads(os.cpu_count())
    R = ref_loader.load()
    R.PLMSSampler = importlib.import_module("audioldm2.latent_diffusion.models.plms").PLMSSampler
    tiny, full = arch.tiny_config(), arch.model_config("audioldm2-full")
    jobs = {
        "plms_tiny": lambda: gen_plms(R, "plms_tiny", tiny, 2, 5, t5_len=5),
        "plms_tiny_g1": lambda: gen_plms(R, "plms_tiny_g1", tiny, 2, 5, guidance=1.0, t5_len=5),
        "plms_tiny_masked": lambda: gen_plms(R, "plms_tiny_masked", tiny, 2, 5, masked=True, t5_len=5),
        # S = 6: range(0, 1000, 166) has 7 steps (S = 3 would give 4, but its last timestep, 1000, is out of the table and
        # the reference's make_schedule raises IndexError there)
        "plms_tiny_s6": lambda: gen_plms(R, "plms_tiny_s6", tiny, 2, 6, t5_len=5),
        "plms_full_10": lambda: gen_plms(R, "plms_full_10", full, 1, 10, with_audio=True),
        "plms_full_50": lambda: gen_plms(R, "plms_full_50", full, 1, 50, with_audio=True),
    }
    for k, fn in jobs.items():
        if a.only and k != a.only:
            continue
        print(k)
        fn()


if __name__ == "__main__":
    main()
