"""TEST INFRASTRUCTURE -- CPU (torch fp32) restatement of audio-to-audio style transfer (AudioLDM 1's
``style_transfer`` on AudioLDM2's primitives): AudioLDM 1's latent guard, DDIMSampler.stochastic_encode and
DDIMSampler.decode (latent_diffusion/models/ddim.py:434-491), next to oracle.functional.ddim_sample.  Pinned against the
unmodified reference sampler by tests/golden/make_style_golden.py and tests/test_style_transfer_cpu.py.  The product
path never imports it."""
from __future__ import annotations

from typing import List, Optional

import torch

from oracle import functional as OF


def latent_guard(x0):
    """AudioLDM 1's guard on the initial latent: one decision for the whole batch, strict comparison; a NaN makes the
    max NaN, so nothing is clipped then."""
    if torch.max(torch.abs(x0)) > 1e2:
        return torch.clip(x0, -10, 10)
    return x0


def encode_coefficients(steps: List[dict], t_enc: int):
    """(sqrt(ddim_alphas)[t_enc], ddim_sqrt_one_minus_alphas[t_enc]) as fp32 scalars (ddim.py:441-442); ``steps`` is
    oracle.functional.ddim_schedule, whose entry with ``index`` t_enc carries both tables' fp32 values."""
    st = next(s for s in steps if s["index"] == t_enc)
    c0 = torch.sqrt(torch.tensor([st["a_t"]], dtype=torch.float32))
    c1 = torch.tensor([st["sqrt_one_minus_at"]], dtype=torch.float32)
    return c0, c1


def stochastic_encode(x0, steps: List[dict], t_enc: int, noise):
    """ddim.py:434-449: c0 * x0 + c1 * noise, the two products then the sum, in fp32."""
    c0, c1 = encode_coefficients(steps, t_enc)
    return c0.reshape(1, 1, 1, 1) * x0 + c1.reshape(1, 1, 1, 1) * noise


def decode_steps(steps: List[dict], t_enc: int) -> List[dict]:
    """The steps DDIMSampler.decode runs (ddim.py:462-491): indices t_enc - 1, ..., 0, the last t_enc entries of the
    schedule -- one entry below the noise level stochastic_encode used."""
    return steps[len(steps) - t_enc:] if t_enc > 0 else []


def style_transfer_latent(unet_sd, ucfg: dict, x0, cond: dict, uncond: Optional[dict], S: int, t_enc: int,
                          guidance: float, enc_noise, step_noises: List[torch.Tensor], tables: Optional[dict] = None):
    """Guard -> stochastic_encode -> decode, with recorded noise (one draw for the encode, one per decode step)."""
    steps = OF.ddim_schedule(tables or OF.ddpm_tables(), S, 1.0)
    z = stochastic_encode(latent_guard(x0), steps, t_enc, enc_noise)
    for i, st in enumerate(decode_steps(steps, t_enc)):
        ts = torch.full((z.shape[0],), st["t"], dtype=torch.long)
        e_c = OF.unet_forward(unet_sd, ucfg, z, ts, cond["context_list"], cond["mask_list"], cond["y"])
        if uncond is None or guidance == 1.0:
            e_u = e_c
        else:
            e_u = OF.unet_forward(unet_sd, ucfg, z, ts, uncond["context_list"], uncond["mask_list"], uncond["y"])
        z, _ = OF.ddim_update(z, e_u, e_c, step_noises[i], st, guidance)
    return z
