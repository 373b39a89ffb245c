"""Seeded inputs of the PLMS fixtures (tests/golden/make_plms_golden.py): the reference PLMSSampler's CPU RNG draw
order replayed, so that tests feed the native sampler and the oracle the same noise the reference consumed."""
from __future__ import annotations

import torch

from tests.golden.cases import SAMPLER_SEED


def plms_num_steps(S: int, num_timesteps: int = 1000) -> int:
    """len(make_ddim_timesteps("uniform", S, T)) (util.py:55-75): range(0, T, T // S), so S = 6 gives 7 steps."""
    return len(range(0, num_timesteps, num_timesteps // S))


def plms_noise(cfg: dict, B: int, S: int, masked: bool = False, seed: int = SAMPLER_SEED):
    """x_T (plms.py:180), then per step [randn_like(x0) in q_sample when masked (plms.py:224, ddpm.py:431)] and one
    noise_like per get_x_prev_and_pred_x0 (plms.py:334): two at the first step, one at every later step.  The step draws
    are multiplied by sigma = 0 and change nothing but the generator state.  -> (x_T, q draws per step, step draws per
    step, torch.randn(4) drawn after the loop)."""
    C, T, F = cfg["latent"]
    torch.manual_seed(seed)
    x_T = torch.randn(B, C, T, F)
    qn, steps = [], []
    for i in range(plms_num_steps(S, cfg["timesteps"])):
        if masked:
            qn.append(torch.randn(B, C, T, F))
        steps.append([torch.randn(B, C, T, F) for _ in range(2 if i == 0 else 1)])
    return x_T, qn, steps, torch.randn(4)


def noise_fn(qn, steps, device=None, log=None):
    """``noise_fn(i, kind)`` for PLMSSampler.sample over the replayed draws; checks that the sampler asks for them in the
    reference's order (``log`` collects the (i, kind) calls)."""
    used = {}

    def fn(i: int, kind: str) -> torch.Tensor:
        if log is not None:
            log.append((i, kind))
        if kind == "q":
            t = qn[i]
        else:
            k = used.get(i, 0)
            used[i] = k + 1
            t = steps[i][k]
        return t.to(device) if device is not None else t
    return fn
