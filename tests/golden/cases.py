"""Seeded inputs shared by the fixture generator and the tests (inputs are regenerated from
seeds; only reference OUTPUTS are stored in the .pt fixtures)."""
from __future__ import annotations

import os

import torch

from audioldm2_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
SAMPLER_SEED = 42          # pipeline.py:185 default seed


class Sampled:
    """A fixture tensor kept as an evenly spaced sample of its flattened elements (the full-size outputs would make the
    fixture files too large to keep in the repository).  ``rel_l2`` (tests/conftest.py) compares the same elements of
    the computed tensor; ``s[b]`` restricts the sample to one index of the leading dimension."""

    def __init__(self, values: torch.Tensor, shape, idx: torch.Tensor = None):
        self.shape = tuple(int(v) for v in shape)
        numel = 1
        for v in self.shape:
            numel *= v
        self.idx = sample_index(numel, values.numel()) if idx is None else idx
        self.values = values

    def take(self, x: torch.Tensor) -> torch.Tensor:
        assert x.numel() == self.numel(), (tuple(x.shape), self.shape)
        return x.reshape(-1)[self.idx.to(x.device)]

    def numel(self) -> int:
        n = 1
        for v in self.shape:
            n *= v
        return n

    def __getitem__(self, b: int) -> "Sampled":
        row = self.numel() // self.shape[0]
        sel = (self.idx // row) == b
        return Sampled(self.values[sel], self.shape[1:], self.idx[sel] - b * row)


def sample_index(numel: int, n: int) -> torch.Tensor:
    """n evenly spaced flat indices out of numel (arithmetic only: the same on every torch version)."""
    return torch.arange(n, dtype=torch.int64) * numel // n


def load(name: str) -> dict:
    d = torch.load(os.path.join(HERE, name + ".pt"), map_location="cpu", weights_only=True)
    for k in [k for k in d if k.endswith(".shape")]:
        key = k[:-len(".shape")]
        d[key] = Sampled(d.pop(key + ".sample"), d.pop(k).tolist())
    return d


def latent(cfg: dict, B: int, seed: int = 3) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    C, T, F = cfg["latent"]
    return torch.randn(B, C, T, F, generator=g)


def unet_inputs(cfg: dict, B: int, t5_len: int = 32, t_value: int = 501):
    x = latent(cfg, B, seed=3)
    t = torch.full((B,), t_value, dtype=torch.long)
    cond, unc = synth.conditioning(cfg, B, seed=77, t5_len=t5_len)
    return x, t, cond, unc


def mel_input(cfg: dict, B: int, seed: int = 9) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    C, T, F = cfg["latent"]
    ds = 2 ** (len(cfg["vae"]["ch_mult"]) - 1)
    return torch.randn(B, 1, T * ds, F * ds, generator=g)


def vocoder_input(cfg: dict, B: int, frames: int, seed: int = 11) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, cfg["vocoder"]["num_mels"], frames, generator=g)


def wav_input(n: int, seed: int = 13) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(1, n, generator=g) - 0.5)


def inpaint_mask(cfg: dict, B: int, seed: int = 15):
    """generate_batch_masked mask (ddpm.py:1611-1617): ones, zero over time rows [0.4,0.6)."""
    C, T, F = cfg["latent"]
    mask = torch.ones(B, 1, T, F)
    mask[:, :, int(T * 0.4):int(T * 0.6), :] = 0
    g = torch.Generator().manual_seed(seed)
    x0 = torch.randn(B, C, T, F, generator=g)
    return mask, x0


def sampler_noise(cfg: dict, B: int, S: int, masked: bool = False, seed: int = SAMPLER_SEED):
    """Replays the reference's CPU RNG draw order (SURVEY.md 7 H3): x_T (ddim.py:191), then per
    step [randn_like(x0) in q_sample when masked (ddpm.py:431)] and randn(shape) (ddim.py:351)."""
    C, T, F = cfg["latent"]
    torch.manual_seed(seed)
    x_T = torch.randn(B, C, T, F)
    noises, qn = [], []
    for _ in range(S):
        if masked:
            qn.append(torch.randn(B, C, T, F))
        noises.append(torch.randn(B, C, T, F))
    return x_T, noises, qn
