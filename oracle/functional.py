"""TEST INFRASTRUCTURE -- CPU (torch fp32) restatement of the AudioLDM2 sampling hot path.

This is the oracle of SURVEY.md 8(c): a plain functional restatement of what the reference
modules compute, driven by a ``state_dict`` with the reference key names.  It is pinned
against the *unmodified imported reference modules* by ``tests/golden/make_golden.py``
(run where a checkout of the reference is available); the committed fixtures under
``tests/golden/`` carry the reference outputs so the pin is re-checked on every test run
(tests/test_oracle.py) without the reference.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / --impl
reference legs may import this module.  The product path (audioldm2_b200/*) never does.

Every function cites the reference lines it restates.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn.functional as F

from audioldm2_b200 import arch

SD = Dict[str, torch.Tensor]


# ------------------------------------------------------------------------------------------
# small helpers
# ------------------------------------------------------------------------------------------

def _conv2d(sd: SD, n: str, x, stride=1, padding=0):
    return F.conv2d(x, sd[n + ".weight"], sd.get(n + ".bias"), stride=stride, padding=padding)


def _lin(sd: SD, n: str, x):
    return F.linear(x, sd[n + ".weight"], sd.get(n + ".bias"))


def _gn(sd: SD, n: str, x, eps):
    return F.group_norm(x, 32, sd[n + ".weight"], sd[n + ".bias"], eps)


def _ln(sd: SD, n: str, x):
    return F.layer_norm(x, (x.shape[-1],), sd[n + ".weight"], sd[n + ".bias"], 1e-5)


def timestep_embedding(t: torch.Tensor, dim: int, max_period: float = 10000.0):
    """util.py:172-196 -- cat([cos, sin]) with freqs = exp(-ln(max_period) * i / half)."""
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(half, dtype=torch.float32) / half).to(t.device)
    args = t[:, None].float() * freqs[None]
    return torch.cat([torch.cos(args), torch.sin(args)], dim=-1)


# ------------------------------------------------------------------------------------------
# UNet (openaimodel.py:837-885)
# ------------------------------------------------------------------------------------------

def _resblock(sd: SD, n: str, x, emb):
    """ResBlock._forward (openaimodel.py:280-300), GroupNorm32 eps 1e-5 (util.py:224-241)."""
    h = _conv2d(sd, n + ".in_layers.2", F.silu(_gn(sd, n + ".in_layers.0", x, 1e-5)), padding=1)
    e = _lin(sd, n + ".emb_layers.1", F.silu(emb))
    h = h + e[:, :, None, None]
    h = _conv2d(sd, n + ".out_layers.3", F.silu(_gn(sd, n + ".out_layers.0", h, 1e-5)), padding=1)
    if (n + ".skip_connection.weight") in sd:
        x = _conv2d(sd, n + ".skip_connection", x)
    return x + h


def _cross_attention(sd: SD, n: str, x, heads: int, context=None, mask=None):
    """CrossAttention.forward (attention.py:343-367)."""
    ctx = x if context is None else context
    q = F.linear(x, sd[n + ".to_q.weight"])
    k = F.linear(ctx, sd[n + ".to_k.weight"])
    v = F.linear(ctx, sd[n + ".to_v.weight"])
    b, nq, c = q.shape
    d = c // heads

    def split(t):
        return t.reshape(b, t.shape[1], heads, d).permute(0, 2, 1, 3).reshape(b * heads, t.shape[1], d)

    q, k, v = split(q), split(k), split(v)
    sim = torch.einsum("bid,bjd->bij", q, k) * (d ** -0.5)
    if mask is not None:
        m = mask.reshape(b, -1)
        m = m[:, None, None, :].expand(b, heads, 1, m.shape[-1]).reshape(b * heads, 1, -1)
        sim = sim.masked_fill(~(m == 1), -torch.finfo(sim.dtype).max)
    attn = sim.softmax(dim=-1)
    out = torch.einsum("bij,bjd->bid", attn, v)
    out = out.reshape(b, heads, nq, d).permute(0, 2, 1, 3).reshape(b, nq, c)
    return _lin(sd, n + ".to_out.0", out)


def _transformer_block(sd: SD, n: str, x, heads, context, mask):
    """BasicTransformerBlock._forward (attention.py:406-410) + GEGLU FF (attention.py:37-63)."""
    x = _cross_attention(sd, n + ".attn1", _ln(sd, n + ".norm1", x), heads) + x
    x = _cross_attention(sd, n + ".attn2", _ln(sd, n + ".norm2", x), heads, context, mask) + x
    h = _lin(sd, n + ".ff.net.0.proj", _ln(sd, n + ".norm3", x))
    a, gate = h.chunk(2, dim=-1)
    x = _lin(sd, n + ".ff.net.2", a * F.gelu(gate)) + x
    return x


def _spatial_transformer(sd: SD, l: arch.Layer, x, context, mask):
    """SpatialTransformer.forward (attention.py:456-467), Normalize eps 1e-6 (attention.py:75-78)."""
    n = l.name
    b, c, h, w = x.shape
    x_in = x
    x = _conv2d(sd, n + ".proj_in", _gn(sd, n + ".norm", x, 1e-6))
    x = x.permute(0, 2, 3, 1).reshape(b, h * w, c)
    for d in range(l.depth):
        x = _transformer_block(sd, f"{n}.transformer_blocks.{d}", x, l.heads, context, mask)
    x = x.reshape(b, h, w, c).permute(0, 3, 1, 2)
    return _conv2d(sd, n + ".proj_out", x) + x_in


def _run_block(sd: SD, layers: List[arch.Layer], h, emb, context_list, mask_list):
    """TimestepEmbedSequential.forward (openaimodel.py:81-103)."""
    for l in layers:
        if l.kind == "conv":
            h = _conv2d(sd, l.name, h, padding=1)
        elif l.kind == "res":
            h = _resblock(sd, l.name, h, emb)
        elif l.kind == "st":
            ctx = context_list[l.ctx_slot] if l.ctx_slot >= 0 else None
            msk = mask_list[l.ctx_slot] if l.ctx_slot >= 0 else None
            h = _spatial_transformer(sd, l, h, ctx, msk)
        elif l.kind == "down":                       # Downsample (openaimodel.py:172-179)
            h = _conv2d(sd, l.name + ".op", h, stride=2, padding=1)
        elif l.kind == "up":                         # Upsample (openaimodel.py:126-136)
            h = F.interpolate(h, scale_factor=2, mode="nearest")
            h = _conv2d(sd, l.name + ".conv", h, padding=1)
    return h


def unet_forward(sd: SD, cfg: dict, x, timesteps, context_list=None, mask_list=None, y=None):
    """UNetModel.forward (openaimodel.py:837-885)."""
    spec = arch.unet_spec(cfg)
    context_list = context_list or []
    mask_list = mask_list or []
    t_emb = timestep_embedding(timesteps, cfg["model_channels"])
    emb = _lin(sd, "time_embed.2", F.silu(_lin(sd, "time_embed.0", t_emb)))
    if cfg.get("extra_film_condition_dim") is not None:
        emb = torch.cat([emb, _lin(sd, "film_emb", y)], dim=-1)      # openaimodel.py:869-870
    hs = []
    h = x
    for blk in spec.input_blocks:
        h = _run_block(sd, blk, h, emb, context_list, mask_list)
        hs.append(h)
    h = _run_block(sd, spec.middle, h, emb, context_list, mask_list)
    for blk in spec.output_blocks:
        h = torch.cat([h, hs.pop()], dim=1)
        h = _run_block(sd, blk, h, emb, context_list, mask_list)
    h = F.silu(_gn(sd, "out.0", h, 1e-5))
    return _conv2d(sd, "out.2", h, padding=1)


# ------------------------------------------------------------------------------------------
# VAE (model.py:419-686, autoencoder.py:103-117), all norms eps 1e-6
# ------------------------------------------------------------------------------------------

def _vae_res(sd: SD, n: str, x):
    """ResnetBlock.forward with temb=None (model.py:155-175)."""
    h = _conv2d(sd, n + ".conv1", F.silu(_gn(sd, n + ".norm1", x, 1e-6)), padding=1)
    h = _conv2d(sd, n + ".conv2", F.silu(_gn(sd, n + ".norm2", h, 1e-6)), padding=1)
    if (n + ".nin_shortcut.weight") in sd:
        x = _conv2d(sd, n + ".nin_shortcut", x)
    return x + h


def _vae_attn(sd: SD, n: str, x):
    """AttnBlock.forward (model.py:204-230): single head over all channels, scale c^-0.5."""
    h = _gn(sd, n + ".norm", x, 1e-6)
    q, k, v = _conv2d(sd, n + ".q", h), _conv2d(sd, n + ".k", h), _conv2d(sd, n + ".v", h)
    b, c, hh, ww = q.shape
    q = q.reshape(b, c, hh * ww).permute(0, 2, 1)
    k = k.reshape(b, c, hh * ww)
    w_ = torch.bmm(q, k) * (int(c) ** -0.5)
    w_ = F.softmax(w_, dim=2)
    v = v.reshape(b, c, hh * ww)
    h = torch.bmm(v, w_.permute(0, 2, 1)).reshape(b, c, hh, ww)
    return x + _conv2d(sd, n + ".proj_out", h)


def vae_decode(sd: SD, cfg: dict, z, scale_factor: float = 1.0):
    """decode_first_stage (ddpm.py:922-926) -> AutoencoderKL.decode (autoencoder.py:111-117)
    -> Decoder.forward (model.py:653-686).  z is NCHW [B, zc, T, F]."""
    z = (1.0 / scale_factor) * z
    h = _conv2d(sd, "post_quant_conv", z)
    h = _conv2d(sd, "decoder.conv_in", h, padding=1)
    h = _vae_res(sd, "decoder.mid.block_1", h)
    h = _vae_attn(sd, "decoder.mid.attn_1", h)
    h = _vae_res(sd, "decoder.mid.block_2", h)
    for lvl in reversed(range(len(cfg["ch_mult"]))):
        for ib in range(cfg["num_res_blocks"] + 1):
            h = _vae_res(sd, f"decoder.up.{lvl}.block.{ib}", h)
        if lvl != 0:
            h = F.interpolate(h, scale_factor=2.0, mode="nearest")       # model.py:53-57
            h = _conv2d(sd, f"decoder.up.{lvl}.upsample.conv", h, padding=1)
    h = F.silu(_gn(sd, "decoder.norm_out", h, 1e-6))
    return _conv2d(sd, "decoder.conv_out", h, padding=1)


def vae_encode_moments(sd: SD, cfg: dict, x):
    """AutoencoderKL.encode up to the moments (autoencoder.py:103-109) -> Encoder.forward
    (model.py:519-543).  x is the mel [B, 1, T, F]; returns [B, 2*embed_dim, T/4.., F/4..]."""
    h = _conv2d(sd, "encoder.conv_in", x, padding=1)
    n_lvl = len(cfg["ch_mult"])
    for lvl in range(n_lvl):
        for ib in range(cfg["num_res_blocks"]):
            h = _vae_res(sd, f"encoder.down.{lvl}.block.{ib}", h)
        if lvl != n_lvl - 1:                                               # model.py:88-91
            h = F.pad(h, (0, 1, 0, 1), mode="constant", value=0)
            h = _conv2d(sd, f"encoder.down.{lvl}.downsample.conv", h, stride=2)
    h = _vae_res(sd, "encoder.mid.block_1", h)
    h = _vae_attn(sd, "encoder.mid.attn_1", h)
    h = _vae_res(sd, "encoder.mid.block_2", h)
    h = F.silu(_gn(sd, "encoder.norm_out", h, 1e-6))
    h = _conv2d(sd, "encoder.conv_out", h, padding=1)
    return _conv2d(sd, "quant_conv", h)


def posterior_sample(moments, noise, scale_factor: float = 1.0):
    """DiagonalGaussianDistribution.sample (distributions.py:24-41) with caller-supplied noise,
    then get_first_stage_encoding's scale (ddpm.py:802)."""
    mean, logvar = torch.chunk(moments, 2, dim=1)
    logvar = torch.clamp(logvar, -30.0, 20.0)
    std = torch.exp(0.5 * logvar)
    return scale_factor * (mean + std * noise)


# ------------------------------------------------------------------------------------------
# HiFi-GAN (hifigan/models.py:96-103,149-165)
# ------------------------------------------------------------------------------------------

def vocoder_forward(sd: SD, cfg: dict, mel_bft):
    """Generator.forward; ``mel_bft`` is [B, num_mels, frames] (ddpm.py:932-935 permutes the
    decoder output [B,1,T,F] to this)."""
    nk = len(cfg["resblock_kernel_sizes"])
    x = F.conv1d(mel_bft, sd["conv_pre.weight"], sd["conv_pre.bias"], padding=3)
    for i, (u, k) in enumerate(zip(cfg["upsample_rates"], cfg["upsample_kernel_sizes"])):
        x = F.leaky_relu(x, 0.1)
        x = F.conv_transpose1d(x, sd[f"ups.{i}.weight"], sd[f"ups.{i}.bias"], stride=u, padding=(k - u) // 2)
        xs = None
        for j, (ks, dil) in enumerate(zip(cfg["resblock_kernel_sizes"], cfg["resblock_dilation_sizes"])):
            r = f"resblocks.{i * nk + j}"
            y = x
            for m in range(3):
                xt = F.leaky_relu(y, 0.1)
                xt = F.conv1d(xt, sd[f"{r}.convs1.{m}.weight"], sd[f"{r}.convs1.{m}.bias"],
                              dilation=dil[m], padding=(ks * dil[m] - dil[m]) // 2)
                xt = F.leaky_relu(xt, 0.1)
                xt = F.conv1d(xt, sd[f"{r}.convs2.{m}.weight"], sd[f"{r}.convs2.{m}.bias"], padding=(ks - 1) // 2)
                y = xt + y
            xs = y if xs is None else xs + y
        x = xs / nk
    x = F.leaky_relu(x)                       # default slope 0.01 (hifigan/models.py:161)
    x = F.conv1d(x, sd["conv_post.weight"], sd["conv_post.bias"], padding=3)
    return torch.tanh(x)


# ------------------------------------------------------------------------------------------
# DDIM (ddim.py:33-91,166-355; util.py:20-95; ddpm.py:201-262)
# ------------------------------------------------------------------------------------------

def ddpm_tables(linear_start=0.0015, linear_end=0.0195, timesteps=1000):
    """register_schedule (ddpm.py:201-262) with the 'linear' schedule (util.py:23-29)."""
    betas = (torch.linspace(linear_start ** 0.5, linear_end ** 0.5, timesteps, dtype=torch.float64) ** 2).numpy()
    ac = np.cumprod(1.0 - betas, axis=0)
    f32 = lambda a: torch.tensor(a, dtype=torch.float32)
    return dict(betas=f32(betas), alphas_cumprod=f32(ac),
                alphas_cumprod_prev=f32(np.append(1.0, ac[:-1])),
                sqrt_alphas_cumprod=f32(np.sqrt(ac)),
                sqrt_one_minus_alphas_cumprod=f32(np.sqrt(1.0 - ac)))


def ddim_schedule(tables: dict, S: int, eta: float):
    """DDIMSampler.make_schedule (ddim.py:33-91) -> per-index fp32 scalars in the order the
    loop visits them (index = S-1-i, ddim.py:222-224).  Mixed numpy/torch dtypes of the
    reference are reproduced: alphas come from the fp32 ``alphas_cumprod``; sigma math is done
    by numpy on fp32 inputs (util.py:78-95); torch.full casts every scalar to fp32
    (ddim.py:330-335)."""
    n = tables["alphas_cumprod"].shape[0]
    c = n // S
    ddim_t = np.asarray(list(range(0, n, c))) + 1                 # util.py:55-75
    ac = tables["alphas_cumprod"].clone().detach().to(torch.float32)   # "to_torch", ddim.py:47
    alphas = ac[ddim_t]                                           # torch fp32
    alphas_prev = np.asarray([ac[0]] + ac[ddim_t[:-1]].tolist())  # float64 ndarray
    sigmas = eta * np.sqrt((1 - alphas_prev) / (1 - alphas) * (1 - alphas / alphas_prev))
    sqrt_1m = np.sqrt(1.0 - alphas)
    steps = []
    for i, step in enumerate(np.flip(ddim_t)):
        idx = len(ddim_t) - i - 1
        a_t = torch.full((1,), alphas[idx]).item()
        a_prev = torch.full((1,), alphas_prev[idx]).item()
        sig = torch.full((1,), sigmas[idx]).item()
        s1m = torch.full((1,), sqrt_1m[idx]).item()
        steps.append(dict(t=int(step), index=idx, a_t=a_t, a_prev=a_prev, sigma_t=sig, sqrt_one_minus_at=s1m,
                          sqrt_acp_t=float(tables["sqrt_alphas_cumprod"][int(step)]),
                          sqrt_1m_acp_t=float(tables["sqrt_one_minus_alphas_cumprod"][int(step)])))
    return steps


def ddim_update(x, e_u, e_c, noise, st: dict, guidance: float):
    """CFG combine + x_{t-1} update of p_sample_ddim (ddim.py:298-300,339-354), fp32."""
    f = lambda v: torch.full((x.shape[0], 1, 1, 1), v, dtype=torch.float32, device=x.device)
    e = e_u + guidance * (e_c - e_u)
    a_t, a_prev, sigma_t, s1m = f(st["a_t"]), f(st["a_prev"]), f(st["sigma_t"]), f(st["sqrt_one_minus_at"])
    pred_x0 = (x - s1m * e) / a_t.sqrt()
    dir_xt = (1.0 - a_prev - sigma_t ** 2).sqrt() * e
    x_prev = a_prev.sqrt() * pred_x0 + dir_xt + sigma_t * noise
    return x_prev, pred_x0


def masked_blend(img, x0, mask, q_noise, st: dict):
    """ddim.py:226-231 with q_sample (ddpm.py:430-436)."""
    img_orig = st["sqrt_acp_t"] * x0 + st["sqrt_1m_acp_t"] * q_noise
    return img_orig * mask + (1.0 - mask) * img


def ddim_sample(unet_sd: SD, ucfg: dict, x_T, noises: List[torch.Tensor], cond: dict, uncond: dict,
                S: int, eta: float = 1.0, guidance: float = 3.5, tables: Optional[dict] = None,
                mask=None, x0=None, q_noises=None):
    """DDIMSampler.ddim_sampling loop (ddim.py:222-262) with recorded noise tensors."""
    tables = tables or ddpm_tables()
    img = x_T
    for i, st in enumerate(ddim_schedule(tables, S, eta)):
        ts = torch.full((img.shape[0],), st["t"], dtype=torch.long)
        if mask is not None:
            img = masked_blend(img, x0, mask, q_noises[i], st)
        e_u = unet_forward(unet_sd, ucfg, img, ts, uncond["context_list"], uncond["mask_list"], uncond["y"])
        e_c = unet_forward(unet_sd, ucfg, img, ts, cond["context_list"], cond["mask_list"], cond["y"])
        img, _ = ddim_update(img, e_u, e_c, noises[i], st, guidance)
    return img
