"""Host-side DDIM and PLMS schedulers: mirror ``DDIMSampler`` (latent_diffusion/models/ddim.py) and ``PLMSSampler``
(latent_diffusion/models/plms.py) -- the Python loop, the schedule tables and the RNG draw order stay on the host exactly
as in the reference; each UNet evaluation with its update (two UNet branches + CFG combine + x_{t-1} update) is one
native call.  ``DDIMSampler.stochastic_encode`` / ``decode`` serve style transfer.
"""
from __future__ import annotations

from typing import Callable, List, Optional

import numpy as np
import torch

from . import _lib


def ddpm_tables(linear_start: float = 0.0015, linear_end: float = 0.0195, timesteps: int = 1000) -> dict:
    """DDPM.register_schedule (ddpm.py:201-262), 'linear' beta schedule (util.py:23-29)."""
    betas = (torch.linspace(linear_start ** 0.5, linear_end ** 0.5, timesteps, dtype=torch.float64) ** 2).numpy()
    ac = np.cumprod(1.0 - betas, axis=0)
    f32 = lambda a: torch.tensor(a, dtype=torch.float32)
    return dict(betas=f32(betas), alphas_cumprod=f32(ac), alphas_cumprod_prev=f32(np.append(1.0, ac[:-1])),
                sqrt_alphas_cumprod=f32(np.sqrt(ac)), sqrt_one_minus_alphas_cumprod=f32(np.sqrt(1.0 - ac)))


def ddim_schedule_length(S: int, num_timesteps: int = 1000) -> int:
    """len(make_ddim_timesteps("uniform", S, T)) (util.py:55-75): range(0, T, T // S), so S = 6 gives 7 entries."""
    if int(S) < 1 or num_timesteps // int(S) < 1:
        raise ValueError(f"ddim_steps={S} must be in [1, {num_timesteps}]")
    return len(range(0, num_timesteps, num_timesteps // int(S)))


def transfer_steps(transfer_strength: float, ddim_steps: int, num_timesteps: int = 1000) -> int:
    """Style transfer's t_enc = int(transfer_strength * ddim_steps) (Python float arithmetic: int(0.29 * 100) == 28),
    checked against the schedule: stochastic_encode gathers index t_enc of it, so 0 <= t_enc < its length, which for
    S = 6 (7 entries) admits strength 1.0.  ValueError otherwise -- the reference fails later with an index error."""
    n = ddim_schedule_length(ddim_steps, num_timesteps)
    t_enc = int(transfer_strength * ddim_steps)
    if not 0 <= t_enc < n:
        raise ValueError(f"transfer_strength={transfer_strength} with ddim_steps={ddim_steps} gives t_enc={t_enc}; "
                         f"it must lie in [0, {n - 1}], the indices of the {n}-entry DDIM schedule")
    return t_enc


def _single_index(t) -> int:
    """The one timestep index of ``t`` (an int, or a tensor of equal entries as AudioLDM passes)."""
    if torch.is_tensor(t):
        v = t.reshape(-1)
        if v.numel() == 0 or not bool((v == v[0]).all()):
            raise NotImplementedError("stochastic_encode: one t for the whole batch (AudioLDM passes [t_enc] * B)")
        return int(v[0])
    return int(t)


class DDIMSampler:
    """Same constructor / ``make_schedule`` / ``sample`` surface as the reference class
    (ddim.py:14-163); ``model`` is a ``NativeLatentDiffusion``."""

    def __init__(self, model, schedule: str = "linear", device=None, **kwargs):
        self.model = model
        self.ddpm_num_timesteps = model.num_timesteps
        self.schedule = schedule
        self.device = device or model.device

    def make_schedule(self, ddim_num_steps: int, ddim_discretize: str = "uniform", ddim_eta: float = 0.0, verbose: bool = False):
        assert ddim_discretize == "uniform"
        n = self.ddpm_num_timesteps
        c = n // ddim_num_steps
        self.ddim_timesteps = np.asarray(list(range(0, n, c))) + 1                 # util.py:55-75
        ac = self.model.alphas_cumprod.clone().detach().to(torch.float32).cpu()      # ddim.py:47
        alphas = ac[self.ddim_timesteps]
        alphas_prev = np.asarray([ac[0]] + ac[self.ddim_timesteps[:-1]].tolist())   # util.py:78-81 (float64 ndarray)
        with np.errstate(all="ignore"):
            import warnings
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                sigmas = ddim_eta * np.sqrt((1 - alphas_prev) / (1 - alphas) * (1 - alphas / alphas_prev))
                sqrt_1m = np.sqrt(1.0 - alphas)
        self.ddim_sigmas, self.ddim_alphas, self.ddim_alphas_prev = sigmas, alphas, alphas_prev
        self.ddim_sqrt_one_minus_alphas = sqrt_1m
        # per-step fp32 scalars exactly as torch.full(...) casts them (ddim.py:330-335)
        f = lambda v: torch.full((1,), v).item()
        self.steps = []
        for i, step in enumerate(np.flip(self.ddim_timesteps)):
            idx = len(self.ddim_timesteps) - i - 1
            self.steps.append(dict(t=int(step), index=idx, a_t=f(alphas[idx]), a_prev=f(alphas_prev[idx]),
                                   sigma_t=f(sigmas[idx]), sqrt_one_minus_at=f(sqrt_1m[idx]),
                                   sqrt_acp_t=float(self.model.sqrt_alphas_cumprod[int(step)]),
                                   sqrt_1m_acp_t=float(self.model.sqrt_one_minus_alphas_cumprod[int(step)])))

    @torch.no_grad()
    def sample(self, S: int, batch_size: int, shape, conditioning=None, eta: float = 0.0, mask=None, x0=None,
               unconditional_guidance_scale: float = 1.0, unconditional_conditioning=None, x_T=None,
               noise_fn: Optional[Callable[[int, str], torch.Tensor]] = None, verbose: bool = False, **kwargs):
        """ddim.py:94-163.  ``noise_fn(i, kind)`` (kind in {"step", "q"}) lets tests inject recorded noise;
        by default noise is drawn with torch.randn on the device in the reference's order (SURVEY 7 H3)."""
        self.make_schedule(ddim_num_steps=S, ddim_eta=eta, verbose=verbose)
        C_, T, F_ = shape
        size = (batch_size, C_, T, F_)
        samples = self.ddim_sampling(conditioning, size, x_T=x_T, mask=mask, x0=x0,
                                     unconditional_guidance_scale=unconditional_guidance_scale,
                                     unconditional_conditioning=unconditional_conditioning, noise_fn=noise_fn)
        return samples, None

    @torch.no_grad()
    def ddim_sampling(self, cond, shape, x_T=None, mask=None, x0=None, unconditional_guidance_scale: float = 1.0,
                      unconditional_conditioning=None, noise_fn=None):
        """ddim.py:166-262 -- the hot loop."""
        m = self.model
        dev = m.device
        img = torch.randn(shape, device=dev) if x_T is None else x_T.to(dev).contiguous().clone()   # ddim.py:191
        # ddim.py:293-296: without an unconditional branch (or with scale 1.0) the model output is apply_model(x, t, c)
        # alone.  The engine always evaluates two halves, so the conditional branch is loaded into both: e_u == e_c
        # bit for bit (same kernels, same data) and e_u + s (e_c - e_u) == e_c exactly.
        single = unconditional_conditioning is None or unconditional_guidance_scale == 1.0
        m.set_conditioning(cond, None if single else unconditional_conditioning)
        nxt = torch.empty_like(img)
        for i, st in enumerate(self.steps):
            if mask is not None:                                                   # ddim.py:226-231
                qn = noise_fn(i, "q") if noise_fn else torch.randn_like(x0)        # q_sample noise (ddpm.py:431)
                m.masked_blend(img, x0, mask, qn, st)
            noise = noise_fn(i, "step") if noise_fn else torch.randn(shape, device=dev)   # ddim.py:351
            m.p_sample_ddim(img, st, noise, unconditional_guidance_scale, out=nxt)
            img, nxt = nxt, img
        return img

    @torch.no_grad()
    def stochastic_encode(self, x0, t, use_original_steps: bool = False, noise=None, *, clip_flag=None):
        """ddim.py:434-449: sqrt(ddim_alphas)[t] * x0 + ddim_sqrt_one_minus_alphas[t] * noise, both coefficients fp32 as
        the reference gathers them; ``noise`` is drawn with randn_like(x0) on the device when not given (one CUDA draw).
        ``clip_flag`` (keyword only): a device int32 guard word; when non-zero x0 is clipped to [-10, 10] first (AudioLDM
        1's latent guard, see parallel.latent_guard_flag).  One native pass."""
        if use_original_steps:
            raise NotImplementedError("stochastic_encode: use_original_steps is not part of AudioLDM's style transfer")
        ti = _single_index(t)
        n = len(self.ddim_timesteps)
        if not 0 <= ti < n:
            raise ValueError(f"stochastic_encode: t={ti} outside the {n}-entry DDIM schedule")
        m = self.model
        x0 = x0.to(m.device, torch.float32).contiguous()
        noise = torch.randn_like(x0) if noise is None else noise.to(m.device, torch.float32).contiguous()
        c0 = float(torch.sqrt(torch.as_tensor(self.ddim_alphas, dtype=torch.float32))[ti])
        c1 = float(torch.as_tensor(self.ddim_sqrt_one_minus_alphas, dtype=torch.float32)[ti])
        return m.stochastic_encode(x0, noise, c0, c1, clip_flag)

    @torch.no_grad()
    def decode(self, x_latent, cond, t_start: int, unconditional_guidance_scale: float = 1.0,
               unconditional_conditioning=None, use_original_steps: bool = False, callback=None,
               noise_fn: Optional[Callable[[int, str], torch.Tensor]] = None):
        """ddim.py:451-491: p_sample_ddim at indices t_start - 1, ..., 0 -- the last t_start entries of ``steps`` -- with
        one noise draw per step (``noise_fn(i, "step")`` or torch.randn on the device), as ddim_sampling's loop does.
        t_start = 0 runs no step."""
        if use_original_steps:
            raise NotImplementedError("decode: use_original_steps is not part of AudioLDM's style transfer")
        t_start = int(t_start)
        if not 0 <= t_start <= len(self.steps):
            raise ValueError(f"decode: t_start={t_start} outside [0, {len(self.steps)}]")
        m = self.model
        dev = m.device
        img = x_latent.to(dev, torch.float32).contiguous().clone()
        if t_start == 0:
            return img
        shape = tuple(img.shape)
        single = unconditional_conditioning is None or unconditional_guidance_scale == 1.0     # ddim.py:284-285
        m.set_conditioning(cond, None if single else unconditional_conditioning)
        nxt = torch.empty_like(img)
        for i, st in enumerate(self.steps[len(self.steps) - t_start:]):
            noise = noise_fn(i, "step") if noise_fn else torch.randn(shape, device=dev)   # ddim.py:351
            m.p_sample_ddim(img, st, noise, unconditional_guidance_scale, out=nxt)
            img, nxt = nxt, img
            if callback:
                callback(i)
        return img


class PLMSSampler(DDIMSampler):
    """The reference ``PLMSSampler`` surface (plms.py:14-154) on the DDIM tables: ``make_schedule`` is DDIM's with eta
    forced to 0 (plms.py:30), so every sigma is 0.  The loop keeps the reference's order of UNet evaluations, e_t
    history and RNG draws; each evaluation is one native call (``model.p_sample_plms``).

    With an unconditional dict and guidance != 1 the two branches are combined as DDIM does (e_u + s (e_c - e_u),
    ddim.py:293-300).  The reference's own PLMS raises there on AudioLDM2's dict conditioning (torch.cat of dicts,
    plms.py:290); this is the value it means to compute.  At guidance 1.0 the path is the reference's."""

    def make_schedule(self, ddim_num_steps: int, ddim_discretize: str = "uniform", ddim_eta: float = 0.0, verbose: bool = False):
        super().make_schedule(ddim_num_steps, ddim_discretize, 0.0, verbose)

    @torch.no_grad()
    def sample(self, S: int, batch_size: int, shape, conditioning=None, eta: float = 0.0, mask=None, x0=None,
               unconditional_guidance_scale: float = 1.0, unconditional_conditioning=None, x_T=None,
               noise_fn: Optional[Callable[[int, str], torch.Tensor]] = None, verbose: bool = False,
               quantize_x0: bool = False, temperature: float = 1.0, noise_dropout: float = 0.0, score_corrector=None,
               **kwargs):
        """plms.py:92-154.  ``eta`` is accepted and ignored, as the reference ignores it.  ``noise_fn(i, kind)`` as in
        DDIMSampler.sample: "q" once per masked step, then one "step" draw per update (two at the first step).  The
        options AudioLDM2 never sets raise unless left at their defaults."""
        if quantize_x0 or temperature != 1.0 or noise_dropout != 0.0 or score_corrector is not None or \
                kwargs.get("ddim_use_original_steps") or kwargs.get("timesteps") is not None:
            raise NotImplementedError("PLMS: quantize_x0, temperature, noise_dropout, score_corrector, timesteps and "
                                      "ddim_use_original_steps are not part of the AudioLDM2 sampling path")
        self.make_schedule(ddim_num_steps=S, ddim_eta=eta, verbose=verbose)
        C_, T, F_ = shape
        samples = self.plms_sampling(conditioning, (batch_size, C_, T, F_), x_T=x_T, mask=mask, x0=x0,
                                     unconditional_guidance_scale=unconditional_guidance_scale,
                                     unconditional_conditioning=unconditional_conditioning, noise_fn=noise_fn)
        return samples, None

    @torch.no_grad()
    def plms_sampling(self, cond, shape, x_T=None, mask=None, x0=None, unconditional_guidance_scale: float = 1.0,
                      unconditional_conditioning=None, noise_fn=None):
        """plms.py:157-258 -- the hot loop.  e_t values live in four device buffers that rotate by reference: the
        three the reference holds in old_eps (most recent first) and the one being written."""
        m = self.model
        dev = m.device
        img = torch.randn(shape, device=dev) if x_T is None else x_T.to(dev).contiguous().clone()   # plms.py:180
        single = unconditional_conditioning is None or unconditional_guidance_scale == 1.0     # plms.py:282-286
        m.set_conditioning(cond, None if single else unconditional_conditioning)
        g = unconditional_guidance_scale
        step_noise = lambda i: noise_fn(i, "step") if noise_fn else torch.randn(shape, device=dev)   # plms.py:334
        ring = [torch.empty(shape, dtype=torch.float32, device=dev) for _ in range(4)]
        held: List[torch.Tensor] = []                   # old_eps, most recent first
        nxt = torch.empty_like(img)
        n = len(self.steps)
        for i, st in enumerate(self.steps):
            t_next = self.steps[min(i + 1, n - 1)]["t"]                                    # plms.py:215-220
            if mask is not None:                                                           # plms.py:222-227
                qn = noise_fn(i, "q") if noise_fn else torch.randn_like(x0)
                m.masked_blend(img, x0, mask, qn, st)
            e_t = next(r for r in ring if all(r is not h for h in held))
            if not held:                                # plms.py:341-345: improved Euler through x' at t_next
                step_noise(i)
                m.p_sample_plms(img, st["t"], img, [], 1, st, g, e_t_out=e_t, out=nxt)
                step_noise(i)
                m.p_sample_plms(nxt, t_next, img, [e_t], _lib.PLMS_AVERAGE, st, g, out=nxt)
            else:
                step_noise(i)
                m.p_sample_plms(img, st["t"], img, held, len(held) + 1, st, g, e_t_out=e_t, out=nxt)
            held = [e_t] + held[:2]                                                        # plms.py:246-248
            img, nxt = nxt, img
        return img
