"""Seeded cases of the Flan-T5 encoder fixtures (tests/golden/t5.pt): the encoder's weights come from
synth.t5_state_dict and its token ids from synth.token_ids, so only the reference outputs are stored (the larger ones as
evenly spaced samples of their elements, cases.Sampled)."""
from __future__ import annotations

import os

from audioldm2_b200 import synth
from tests.golden import cases

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "t5.pt")
WEIGHT_SEED = 1238

# name -> (n_layer, per-row token counts (L = max), id seed).  B = 3 rows are ragged: the shorter rows are padded.
CASES = {
    "tiny_b1_l1": (2, (1,), 31),
    "tiny_b3_l32": (2, (32, 17, 5), 32),
    "tiny_b3_l128": (2, (128, 64, 9), 33),
    "full_b1_l1": (24, (1,), 41),
    "full_b3_l32": (24, (32, 17, 5), 42),
    "full_b3_l128": (24, (128, 64, 9), 43),
}
# name -> n_layer: the unconditional state T5("") (get_unconditional_condition), stored as [1, 1, 1024]
UNCOND = {"tiny_uncond": 2, "full_uncond": 24}


def weights(n_layer: int):
    return synth.t5_state_dict(seed=WEIGHT_SEED, n_layer=n_layer)


def inputs(name: str):
    """-> (ids [B, L] int64, mask [B, L] float)"""
    _, lens, seed = CASES[name]
    return synth.token_ids(lens, seed=seed)


def load() -> dict:
    """name -> hidden states (a tensor, or a cases.Sampled that tests.conftest.rel_l2 compares), plus "param_shapes"."""
    return cases.load("t5")
