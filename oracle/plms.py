"""TEST INFRASTRUCTURE -- CPU (torch fp32) restatement of the reference PLMS sampler
(latent_diffusion/models/plms.py), next to oracle.functional.ddim_sample.  Pinned against the unmodified reference
PLMSSampler by tests/golden/make_plms_golden.py and tests/test_plms_cpu.py.  The product path never imports it."""
from __future__ import annotations

from typing import Callable, List, Optional

import torch

from oracle import functional as OF


def plms_eps_prime(e_t, old: List[torch.Tensor]):
    """plms.py:346-356: the Adams-Bashforth combination of e_t and the held values (``old[-1]`` the most recent), in
    the reference's operation order.  The first step's average is made by the caller."""
    if len(old) == 1:
        return (3 * e_t - old[-1]) / 2
    if len(old) == 2:
        return (23 * e_t - 16 * old[-1] + 5 * old[-2]) / 12
    return (55 * e_t - 59 * old[-1] + 37 * old[-2] - 9 * old[-3]) / 24


def plms_update(x, e, st: dict):
    """get_x_prev_and_pred_x0 (plms.py:319-338) with sigma = 0 (make_schedule forces eta = 0, plms.py:30): the noise
    term is an exact zero and is left out."""
    f = lambda v: torch.full((x.shape[0], 1, 1, 1), v, dtype=torch.float32, device=x.device)
    a_t, a_prev, sigma_t, s1m = f(st["a_t"]), f(st["a_prev"]), f(st["sigma_t"]), f(st["sqrt_one_minus_at"])
    pred_x0 = (x - s1m * e) / a_t.sqrt()
    dir_xt = (1.0 - a_prev - sigma_t ** 2).sqrt() * e
    return a_prev.sqrt() * pred_x0 + dir_xt, pred_x0


def plms_sample(unet_sd, ucfg: dict, x_T, cond: dict, uncond: Optional[dict], S: int, guidance: float = 3.5,
                tables: Optional[dict] = None, mask=None, x0=None, q_noises=None):
    """PLMSSampler.plms_sampling (plms.py:157-258) with recorded q_sample noise.  With an unconditional dict and
    guidance != 1 the two branches are combined as DDIM does (e_u + s (e_c - e_u), ddim.py:293-300), the value
    plms.py:288-292 means to compute; the reference's own code raises there on dict conditioning."""
    def eps(x, t):
        ts = torch.full((x.shape[0],), t, dtype=torch.long)
        e_c = OF.unet_forward(unet_sd, ucfg, x, ts, cond["context_list"], cond["mask_list"], cond["y"])
        if uncond is None or guidance == 1.0:
            return e_c
        e_u = OF.unet_forward(unet_sd, ucfg, x, ts, uncond["context_list"], uncond["mask_list"], uncond["y"])
        return e_u + guidance * (e_c - e_u)

    return plms_loop(eps, OF.ddim_schedule(tables or OF.ddpm_tables(), S, 0.0), x_T, mask, x0, q_noises)


def plms_loop(eps: Callable, steps: List[dict], x_T, mask=None, x0=None, q_noises=None):
    """The loop of plms_sampling (plms.py:212-258) over ``eps(x, t)`` (get_model_output) and the schedule ``steps``
    (oracle.functional.ddim_schedule at eta 0)."""
    img = x_T
    old: List[torch.Tensor] = []
    for i, st in enumerate(steps):
        t_next = steps[min(i + 1, len(steps) - 1)]["t"]
        if mask is not None:
            img = OF.masked_blend(img, x0, mask, q_noises[i], st)
        e_t = eps(img, st["t"])
        if not old:                                            # plms.py:341-345, pseudo improved Euler
            x_mid, _ = plms_update(img, e_t, st)
            e_p = (e_t + eps(x_mid, t_next)) / 2
        else:
            e_p = plms_eps_prime(e_t, old)
        img, _ = plms_update(img, e_p, st)
        old.append(e_t)
        if len(old) >= 4:
            old.pop(0)
    return img
