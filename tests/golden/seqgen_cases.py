"""Seeded cases of the AudioMAE token generator fixtures (tests/golden/seqgen.pt): the generator's weights come from
synth.seqgen_state_dict and its inputs from synth.encoder_outputs, so only the reference outputs are stored."""
from __future__ import annotations

import os

import torch

from audioldm2_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "seqgen.pt")
WEIGHT_SEED = 1237

# name -> (n_layer, per-row T5 lengths (L = max), input seed).  B = 3 rows are ragged: the shorter rows are padded.
CASES = {
    "tiny_b1_l1": (2, (1,), 11),
    "tiny_b3_l32": (2, (32, 17, 5), 12),
    "tiny_b3_l128": (2, (128, 64, 9), 13),
    "full_b1_l1": (12, (1,), 21),
    "full_b3_l32": (12, (32, 17, 5), 22),
    "full_b3_l128": (12, (128, 64, 9), 23),
}


def weights(n_layer: int):
    return synth.seqgen_state_dict(seed=WEIGHT_SEED, n_layer=n_layer)


def inputs(name: str):
    """-> (clap [B, 1, 512], t5 [B, L, 1024], t5_mask [B, L])"""
    _, lens, seed = CASES[name]
    return synth.encoder_outputs(len(lens), lens, seed=seed)


def load() -> dict:
    return torch.load(PATH, map_location="cpu", weights_only=True)
