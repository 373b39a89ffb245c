"""Seeded inputs of the style-transfer fixtures (tests/golden/make_style_golden.py): the cases, and the reference's CPU
RNG draw order replayed, so that tests feed the native path and the oracle the noise the reference consumed."""
from __future__ import annotations

import torch

from audioldm2_b200 import arch
from tests.golden.cases import SAMPLER_SEED, mel_input

# name -> (config, B, S, t_enc, guidance, scale_factor, t5_len, with_audio)
CASES = {
    "style_tiny_t0": ("tiny", 2, 10, 0, 3.5, 1.0, 5, False),
    "style_tiny_t1": ("tiny", 2, 10, 1, 3.5, 1.0, 5, False),
    "style_tiny_t5": ("tiny", 2, 10, 5, 3.5, 1.0, 5, False),
    "style_tiny_t9": ("tiny", 2, 10, 9, 3.5, 1.0, 5, False),
    "style_tiny_g1": ("tiny", 2, 10, 5, 1.0, 1.0, 5, False),
    "style_tiny_48k": ("tiny-48k", 2, 10, 5, 3.5, 1.0, 32, False),
    # scale_factor large enough that max |init_latent| > 100: AudioLDM 1's guard clips the latent to [-10, 10]
    "style_tiny_guard": ("tiny", 2, 10, 5, 3.5, 1000.0, 5, False),
    "style_full": ("audioldm2-full", 1, 20, 10, 3.5, 1.0, 32, True),
    "style_48k_full": ("audioldm_48k", 1, 10, 5, 3.5, 1.0, 32, True),
}


def config(key: str) -> dict:
    if key == "tiny":
        return arch.tiny_config()
    if key == "tiny-48k":
        return arch.tiny_config(variant="48k")
    return arch.model_config(key)


def mel(cfg: dict, B: int) -> torch.Tensor:
    """The mel the VAE encodes: seeded, one row repeated B times as style_transfer repeats it."""
    return mel_input(cfg, 1).expand(B, -1, -1, -1).contiguous()


def style_noise(cfg: dict, B: int, t_enc: int, seed: int = SAMPLER_SEED):
    """posterior.sample() (distributions.py:38), randn_like in stochastic_encode (ddim.py:445), one noise_like per
    decode step (ddim.py:351) -> (posterior draw, encode draw, step draws, torch.randn(4) drawn after the loop)."""
    C, T, F = cfg["latent"]
    torch.manual_seed(seed)
    post = torch.randn(B, C, T, F)
    enc = torch.randn(B, C, T, F)
    steps = [torch.randn(B, C, T, F) for _ in range(t_enc)]
    return post, enc, steps, torch.randn(4)
