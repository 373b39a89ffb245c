"""Seeded cases of the CLAP text-embedding fixtures (tests/golden/clap.pt): the text branch's weights come from
synth.clap_text_state_dict and its token ids from synth.clap_token_ids (padded to the tokenizer's 512), so only the
reference outputs are stored."""
from __future__ import annotations

import os

from audioldm2_b200 import synth
from tests.golden import cases

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "clap.pt")
WEIGHT_SEED = 1239

RAGGED8 = (512, 77, 31, 16, 9, 5, 3, 2)     # one row of the full 512 tokens (the truncation limit), one two-token row
# name -> (n_layer, per-row token counts including BOS / EOS, id seed)
CASES = {
    "tiny_b1": (2, (7,), 51),
    "tiny_b3": (2, (40, 13, 2), 52),
    "tiny_b8": (2, RAGGED8, 53),
    "tiny_b8_short": (2, (33, 20, 14, 9, 7, 5, 4, 3), 54),
    "full_b1": (12, (12,), 61),
    "full_b3": (12, (40, 13, 2), 62),
    "full_b8": (12, RAGGED8, 63),
}
# name -> n_layer: CLAP("") (get_unconditional_condition), stored as [1, 512]
UNCOND = {"tiny_uncond": 2, "full_uncond": 12}
# the seeded forward() of the reference conditioner, with its random replacement by CLAP(""): (n_layer, case)
# (its prompts are all longer than "", so a row equal to CLAP("") is a replaced row)
FORWARD = (2, "tiny_b8_short")


def weights(n_layer: int):
    return synth.clap_text_state_dict(seed=WEIGHT_SEED, n_layer=n_layer)


def inputs(name: str):
    """-> (ids [B, 512] int64, mask [B, 512] float)"""
    _, lens, seed = CASES[name]
    return synth.clap_token_ids(lens, seed=seed)


def load() -> dict:
    """name -> embedding [B, 512]; "forward" -> the seeded forward's output [8, 1, 512], "forward_seed",
    "forward_replaced" (rows replaced by CLAP("")), "forward_rng_state" (torch.get_rng_state() after the call); plus
    "param_shapes"."""
    return cases.load("clap")
