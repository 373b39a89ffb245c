"""Seeded cases of the CLAP audio-embedding fixtures (tests/golden/clap_audio.pt): the audio branch's weights come from
synth.clap_audio_state_dict, the text branch of the ranking case from synth.clap_text_state_dict, its texts through
synth.clap_tokenize, and the waveforms from seeds below, so only the reference outputs are stored."""
from __future__ import annotations

import os

import torch

from audioldm2_b200 import synth
from tests.golden import cases

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "clap_audio.pt")
WEIGHT_SEED = 1240
TEXT_SEED = 1239
TEXT_LAYERS = 2
SMALL, BASE = (2, 2, 2, 2), (2, 2, 12, 2)

# name -> (depths, sampling rate, samples, clips, waveform seed)
CASES = {
    "small_16k_10s": (SMALL, 16000, 163840, 1, 11),      # 491 520 samples at 48 kHz: truncated to 480 000, T = 1001
    "small_16k_2s5": (SMALL, 16000, 40000, 6, 12),
    "small_16k_short": (SMALL, 16000, 5120, 1, 13),      # the shortest latent (8 frames): T = 33
    "small_48k_10s": (SMALL, 48000, 491520, 1, 14),
    "base_16k_10s": (BASE, 16000, 163840, 1, 21),
    "base_16k_2s5": (BASE, 16000, 40000, 6, 22),
    "base_16k_short": (BASE, 16000, 5120, 1, 23),
    "base_48k_10s": (BASE, 48000, 491520, 1, 24),
}
# the seeded cos_similarity call: B prompts x N_GEN candidates of RANK_SAMPLES at 16 kHz, SMALL depths
RANK_B, RANK_N_GEN, RANK_SAMPLES, RANK_SEED = 2, 3, 40000, 31
RANK_TEXTS = ("a dog barks in the rain", "piano and a soft choir")


def weights(depths):
    return synth.clap_audio_state_dict(seed=WEIGHT_SEED, depths=depths)


def text_weights():
    return synth.clap_text_state_dict(seed=TEXT_SEED, n_layer=TEXT_LAYERS)


def waveform(n: int, L: int, seed: int) -> torch.Tensor:
    """Vocoder-like audio: a few decaying partials plus noise at |x| ~ 0.1, [n, L] float32."""
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(L, dtype=torch.float64) / 16000.0
    out = []
    for _ in range(n):
        f = 80.0 + 3000.0 * torch.rand(4, generator=g, dtype=torch.float64)
        a = 0.05 * torch.rand(4, generator=g, dtype=torch.float64)
        x = (a[:, None] * torch.sin(2 * torch.pi * f[:, None] * t[None]) * torch.exp(-t[None] * (1 + 3 * a[:, None]))).sum(0)
        x = x + 0.03 * torch.randn(L, generator=g, dtype=torch.float64)
        out.append(x)
    return torch.stack(out).float()


def inputs(name: str) -> torch.Tensor:
    _, _, L, n, seed = CASES[name]
    return waveform(n, L, seed)


def rank_inputs():
    """-> (waveform [B n_gen, L], texts (the reference's text * n_gen), B)"""
    return waveform(RANK_B * RANK_N_GEN, RANK_SAMPLES, 41), list(RANK_TEXTS) * RANK_N_GEN, RANK_B


def load() -> dict:
    """name -> embedding [n, 512]; "rank_similarity" [B n_gen], "rank_best", "rank_audio_replaced",
    "rank_text_replaced", "rank_seed", "rank_rng_state"; "relative_position_index" [64, 64]; "attn_mask_bits.<R>"
    (np.packbits of attn_mask != 0, attn_mask values being 0 / -100) of the shifted blocks; "param_shapes"."""
    return cases.load("clap_audio")
