"""Generate the style-transfer fixtures by running the UNMODIFIED reference DDIMSampler's make_schedule,
stochastic_encode and decode (latent_diffusion/models/ddim.py:33-91,434-491).

Run where the reference package is importable (oracle/ref_loader.py):

    python tests/golden/make_style_golden.py [--only NAME]

Everything runs on the CPU in fp32: the reference Encoder and quant_conv (autoencoder.py:104-109), the reference
DiagonalGaussianDistribution's sample (one CPU draw), the sampler over the reference UNet through make_golden.py's stub
model, the reference Decoder and the HiFi-GAN.  Only two pieces are restated: get_first_stage_encoding's
``scale_factor * z`` (ddpm.py:793-802) and AudioLDM 1's two-line latent guard, whose source is not part of the
reference tree.  After each call ``rng_after = torch.randn(4)`` is stored, so that tests can check how many draws it made.
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

from oracle import functional as OF                                   # noqa: E402
from oracle import ref_loader                                         # noqa: E402
from tests.golden import cases, style_cases                           # noqa: E402
from tests.golden.make_golden import _StubModel, _save, ref_unet, ref_vae, ref_vocoder   # noqa: E402


@torch.no_grad()
def gen_style(R, name):
    key, B, S, t_enc, guidance, scale_factor, t5_len, with_audio = style_cases.CASES[name]
    cfg = style_cases.config(key)
    m = ref_unet(R, cfg["unet"])
    dec, enc, sd = ref_vae(R, cfg["vae"])
    tables = OF.ddpm_tables(cfg["linear_start"], cfg["linear_end"], cfg["timesteps"])
    _, _, cond, unc = cases.unet_inputs(cfg, B, t5_len=t5_len)
    sampler = R.DDIMSampler(_StubModel(m, tables), device=torch.device("cpu"))
    mel = style_cases.mel(cfg, B)
    torch.manual_seed(cases.SAMPLER_SEED)
    t0 = time.time()
    moments = torch.nn.functional.conv2d(enc(mel), sd["quant_conv.weight"], sd["quant_conv.bias"])   # autoencoder.py:106
    z = R.DiagonalGaussianDistribution(moments).sample()
    init_latent = scale_factor * z                                     # get_first_stage_encoding (ddpm.py:793-802)
    if torch.max(torch.abs(init_latent)) > 1e2:                        # AudioLDM 1's latent guard
        init_latent = torch.clip(init_latent, -10, 10)
    sampler.make_schedule(ddim_num_steps=S, ddim_eta=1.0, verbose=False)
    z_enc = sampler.stochastic_encode(init_latent, torch.tensor([t_enc] * B))
    latent = sampler.decode(z_enc, cond, t_enc, unconditional_guidance_scale=guidance, unconditional_conditioning=unc)
    out = dict(init_latent=init_latent, z_enc=z_enc, latent=latent, rng_after=torch.randn(4))
    if with_audio:
        h = torch.nn.functional.conv2d(latent, sd["post_quant_conv.weight"], sd["post_quant_conv.bias"])
        mel_out = dec(h)
        out["mel"] = mel_out
        out["wave"] = ref_vocoder(R, cfg["vocoder"])(mel_out.squeeze(1).permute(0, 2, 1))      # ddpm.py:932-935
    print(f"  {name}: S={S} t_enc={t_enc} in {time.time() - t0:.1f}s")
    _save(name, out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default=None)
    a = ap.parse_args()
    torch.set_num_threads(os.cpu_count())
    R = ref_loader.load()
    R.DiagonalGaussianDistribution = importlib.import_module(
        "audioldm2.latent_diffusion.modules.distributions.distributions").DiagonalGaussianDistribution
    for name in style_cases.CASES:
        if a.only and name != a.only:
            continue
        print(name)
        gen_style(R, name)


if __name__ == "__main__":
    main()
