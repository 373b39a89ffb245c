"""NativeLatentDiffusion: the reference ``LatentDiffusion`` hot-path surface on the native engine.

Method names and argument meaning follow latent_diffusion/models/ddpm.py so the sampler and the
pipeline read like the reference:

    apply_model(x, t, cond)                  ddpm.py:1034-1042  (DiffusionWrapper.forward :1821-1879)
    decode_first_stage(z)                    ddpm.py:922-926
    mel_spectrogram_to_waveform(mel)         ddpm.py:928-939
    encode_first_stage(x) (+ posterior)      ddpm.py:941-943, 793-802
    q_sample / masked blend                  ddpm.py:430-436, ddim.py:226-231
    stochastic_encode (style transfer)       ddim.py:434-449

plus ``p_sample_ddim`` (ddim.py:265-355) fused into one native step, and each UNet evaluation of ``p_sample_plms``
(plms.py:260-360) with its update as one native step.  Conditioning is either the
reference's keyed cond-dict (``{"film_clap_...": y, "crossattn_...": [ctx, mask], ...}``, unpacked by
``unpack_cond_dict`` exactly as DiffusionWrapper.forward does) or the already-unpacked
``{"context_list": [...], "mask_list": [...], "y": ...}``.

All device work goes through the engine-level C-ABI (``aldm_engine_*``, include/aldm_b200.h): one C call
per reference seam.  The UNet runs as ``lanes`` independent sub-batches replayed as parallel branches of one
CUDA graph (csrc/engine_abi.cu).
"""
from __future__ import annotations

import ctypes as C
import math
import os
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib, arch, engine, parallel, plan
from .sampler import DDIMSampler, PLMSSampler, ddpm_tables


def split_state_dict(state_dict: Dict[str, torch.Tensor]):
    """Reference checkpoint keys (SURVEY.md 8b) -> (unet, vae, vocoder, scale_factor)."""
    un = {k[len("model.diffusion_model."):]: v for k, v in state_dict.items() if k.startswith("model.diffusion_model.")}
    voc = {k[len("first_stage_model.vocoder."):]: v for k, v in state_dict.items()
           if k.startswith("first_stage_model.vocoder.")}
    vae = {k[len("first_stage_model."):]: v for k, v in state_dict.items()
           if k.startswith("first_stage_model.") and not k.startswith("first_stage_model.vocoder.")
           and not k.startswith("first_stage_model.loss.")}
    sf = float(state_dict["scale_factor"]) if "scale_factor" in state_dict else 1.0
    return un, vae, voc, sf


def split_seqgen_state_dict(state_dict: Dict[str, torch.Tensor], index: int = 0) -> Dict[str, torch.Tensor]:
    """The AudioMAE token generator's weights from a reference checkpoint: keys under ``cond_stage_models.<index>.``
    (``index`` = position of ``crossattn_audiomae_generated`` in ``cond_stage_config``, 0 for audioldm2-full and -large),
    restricted to arch.seqgen_param_shapes (the module's own CLAP / T5 / AudioMAE sub-models and the
    ``attn.bias`` / ``attn.masked_bias`` buffers some transformers versions store are left out).  Raises if a key the
    generator needs is missing.  ``split_state_dict`` is unchanged and does not return these."""
    pre = f"cond_stage_models.{index}."
    h = [k for k in state_dict if k.startswith(pre + "model.h.") and k.endswith(".ln_1.weight")]
    n_layer = len(h)
    want = arch.seqgen_param_shapes(n_layer, with_wte=False)
    out = {}
    for k, shp in want.items():
        v = state_dict.get(pre + k)
        if v is None:
            raise KeyError(f"checkpoint has no {pre + k} (needed by the AudioMAE token generator)")
        if tuple(v.shape) != tuple(shp):
            raise ValueError(f"{pre + k}: shape {tuple(v.shape)}, expected {shp}")
        out[k] = v
    return out


def split_t5_state_dict(state_dict: Dict[str, torch.Tensor], prefix: str) -> Dict[str, torch.Tensor]:
    """The Flan-T5 encoder's weights from a reference checkpoint: the keys under ``prefix`` (a ``T5EncoderModel``, e.g.
    ``cond_stage_models.1.model.``), named and shaped as arch.t5_param_shapes.  ``encoder.embed_tokens.weight`` (tied to
    ``shared.weight``) is optional and not returned.  Raises KeyError for a missing key, ValueError for a wrong shape."""
    n_layer = len([k for k in state_dict if k.startswith(prefix + "encoder.block.") and k.endswith(".layer.0.layer_norm.weight")])
    if n_layer == 0:
        raise KeyError(f"checkpoint has no T5 encoder blocks under {prefix}encoder.block.")
    out = {}
    for k, shp in arch.t5_param_shapes(n_layer, with_embed_tokens=False).items():
        v = state_dict.get(prefix + k)
        if v is None:
            raise KeyError(f"checkpoint has no {prefix + k} (needed by the Flan-T5 encoder)")
        if tuple(v.shape) != tuple(shp):
            raise ValueError(f"{prefix + k}: shape {tuple(v.shape)}, expected {shp}")
        out[k] = v
    return out


def split_clap_text_state_dict(state_dict: Dict[str, torch.Tensor], prefix: str) -> Dict[str, torch.Tensor]:
    """The CLAP text branch's weights from a reference checkpoint: the keys under ``prefix`` (the CLAP model, e.g.
    ``cond_stage_models.0.model.``), named and shaped as arch.clap_text_param_shapes.  The ``embeddings.position_ids`` /
    ``token_type_ids`` buffers that older transformers saved and everything of the audio branch are ignored.  Raises
    KeyError for a missing key, ValueError for a wrong shape."""
    tail = ".attention.output.LayerNorm.weight"
    n_layer = len([k for k in state_dict if k.startswith(prefix + "text_branch.encoder.layer.") and k.endswith(tail)])
    if n_layer == 0:
        raise KeyError(f"checkpoint has no RoBERTa layers under {prefix}text_branch.encoder.layer.")
    out = {}
    for k, shp in arch.clap_text_param_shapes(n_layer).items():
        v = state_dict.get(prefix + k)
        if v is None:
            raise KeyError(f"checkpoint has no {prefix + k} (needed by the CLAP text encoder)")
        if tuple(v.shape) != tuple(shp):
            raise ValueError(f"{prefix + k}: shape {tuple(v.shape)}, expected {shp}")
        out[k] = v
    return out


def htsat_dft_basis(n_fft: int = 1024) -> Tuple[torch.Tensor, torch.Tensor]:
    """torchlibrosa's STFT conv weights (DFTBase.dft_matrix times the periodic Hann window): real[k, 0, n] =
    cos(2 pi k n / N) w[n], imag[k, 0, n] = -sin(2 pi k n / N) w[n], k = 0 .. N / 2, in float64."""
    nn_ = torch.arange(n_fft, dtype=torch.float64)
    k = torch.arange(n_fft // 2 + 1, dtype=torch.float64)
    win = 0.5 - 0.5 * torch.cos(2 * math.pi * nn_ / n_fft)
    ph = 2 * math.pi * ((k[:, None] * nn_[None, :]) % n_fft) / n_fft
    return (torch.cos(ph) * win)[:, None, :], (-torch.sin(ph) * win)[:, None, :]


def split_clap_audio_state_dict(state_dict: Dict[str, torch.Tensor], prefix: str) -> Dict[str, torch.Tensor]:
    """The CLAP audio branch's weights from a reference checkpoint: the keys under ``prefix`` (the CLAP model, e.g.
    ``clap.model.``), named and shaped as arch.clap_audio_param_shapes, with as many Swin blocks per stage as the
    checkpoint holds.  tscam_conv, head, the relative_position_index / attn_mask buffers, bn0.num_batches_tracked and the
    text branch are ignored.  The log-mel filterbank is the checkpoint's melW; the STFT weights must be torchlibrosa's
    periodic-Hann DFT basis (the native front end computes an FFT instead of reading them).  Raises KeyError for a missing
    key, ValueError for a wrong shape or a different STFT basis."""
    depths = plan.htsat_depths(state_dict, prefix)
    out = {}
    for k, shp in arch.clap_audio_param_shapes(tuple(depths)).items():
        v = state_dict.get(prefix + k)
        if v is None:
            raise KeyError(f"checkpoint has no {prefix + k} (needed by the CLAP audio encoder)")
        if tuple(v.shape) != tuple(shp):
            raise ValueError(f"{prefix + k}: shape {tuple(v.shape)}, expected {shp}")
        out[k] = v
    real, imag = htsat_dft_basis(arch.CLAP_AUDIO["n_fft"])
    for name, ref in (("conv_real", real), ("conv_imag", imag)):
        k = f"audio_branch.spectrogram_extractor.stft.{name}.weight"
        err = float((out[k].double() - ref).abs().max())
        if not err <= 1e-6:
            raise ValueError(f"{prefix + k} differs from the periodic-Hann DFT basis by {err:.3g}: the native front end "
                             "computes that transform as an FFT and cannot use other STFT weights")
    return out


def reorder_cond_dict(cond_dict: dict, conditioning_key: Sequence[str]) -> dict:
    """LatentDiffusion.reorder_cond_dict (ddpm.py:1028-1032): the UNet consumes the conditions in the order of
    ``conditioning_key`` (the config's list), not in the dict's insertion order."""
    return {k: cond_dict[k] for k in conditioning_key}


def unpack_cond_dict(cond_dict: dict) -> dict:
    """DiffusionWrapper.forward's key-ordered unpacking (ddpm.py:1821-1879) -> {"context_list", "mask_list", "y"}.

    * ``film*``      -> y: ``squeeze(1)``, several entries concatenated on the last dim (:1836-1840);
    * ``crossattn*`` -> one (context, mask) pair appended per key; a dict-valued entry (the unconditional
      branch of the sequence-generation model) contributes its LAST inner ``crossattn*`` pair (:1843-1848);
    * ``noncond*``   -> skipped (:1860-1863); ``concat*`` is not on this path (no AudioLDM2 config uses it);
    * anything else raises NotImplementedError, as the reference does."""
    if "context_list" in cond_dict and "mask_list" in cond_dict:        # already unpacked
        return dict(context_list=list(cond_dict["context_list"]), mask_list=list(cond_dict["mask_list"]), y=cond_dict.get("y"))
    y = None
    context_list, mask_list = [], []
    for key in cond_dict.keys():
        v = cond_dict[key]
        if "concat" in key:
            raise NotImplementedError("concat conditioning is not part of the AudioLDM2 sampling path")
        elif "film" in key:
            y = v.squeeze(1) if y is None else torch.cat([y, v.squeeze(1)], dim=-1)
        elif "crossattn" in key:
            if isinstance(v, dict):
                pair = None
                for k in v.keys():
                    if "crossattn" in k:
                        pair = v[k]
                if pair is None:
                    raise ValueError(f"dict-valued condition {key!r} holds no crossattn entry")
                context, attn_mask = pair
            else:
                assert len(v) == 2, f"The context condition for {key} should have two elements, one context one mask"
                context, attn_mask = v
            context_list.append(context)
            mask_list.append(attn_mask)
        elif "noncond" in key:
            continue
        else:
            raise NotImplementedError(key)
    return dict(context_list=context_list, mask_list=mask_list, y=y)


def default_lanes(batch: int) -> int:
    """UNet lanes: 1 unless ALDM_LANES says otherwise.  Parallel lanes overlap the UNet's branches, but what they hide
    at the deep levels is paid back in split-K reductions, second weight streams and wave quantisation at the wide ones."""
    env = os.environ.get("ALDM_LANES")
    if env:
        n = max(1, min(int(env), _lib.MAX_LANES))
        while batch % n:
            n -= 1
        return n
    return 1


class NativeLatentDiffusion:
    def __init__(self, cfg: dict, unet_sd, vae_sd, vocoder_sd, batch: int, device="cuda:0", scale_factor: float = 1.0,
                 ctx_max_len=(8, 128), impl: str = "tc", keep_plain: bool = False, use_graph: bool = True,
                 with_encoder: bool = False, arena_bcast=None, lanes: Optional[int] = None,
                 conditioning_key: Optional[Sequence[str]] = None):
        """``batch`` is the latent batch B_l = batchsize * n_candidate_gen_per_text the programs are
        planned for.  ``arena_bcast(name, cpu_or_none, nbytes) -> device tensor`` lets parallel.py
        replace the H2D upload by an NCCL broadcast from rank 0."""
        self.cfg = cfg
        self.device = torch.device(device)
        self.batch = batch
        self.scale_factor = scale_factor
        self.use_graph = use_graph
        self.num_timesteps = cfg["timesteps"]
        self.parameterization = "eps"
        self.conditioning_key = list(conditioning_key) if conditioning_key is not None else None
        for k, v in ddpm_tables(cfg["linear_start"], cfg["linear_end"], cfg["timesteps"]).items():
            setattr(self, k, v)
        self.latent = tuple(cfg["latent"])
        C_, T, Fq = self.latent
        pk = dict(impl=impl, keep_plain=keep_plain)
        self._pk = pk
        ds = 2 ** (len(cfg["vae"]["ch_mult"]) - 1)
        self.mel_hw = (T * ds, Fq * ds)
        self.lanes = lanes if lanes is not None else default_lanes(batch)
        assert 1 <= self.lanes <= _lib.MAX_LANES and batch % self.lanes == 0, (batch, self.lanes)
        self._arena_bcast = arena_bcast
        self._sd = dict(vae=vae_sd)

        def up(name, p: plan.Plan, ranges, dev_arena=None):
            if dev_arena is None and arena_bcast:
                dev_arena = arena_bcast(name, p.arena, p.arena.numel())
            return engine.DeviceProgram(p, self.device, ranges, dev_arena)

        pu = plan.build_unet(unet_sd, cfg["unet"], self.latent, batch // self.lanes, cfg_batched=True, ctx_max_len=ctx_max_len, **pk)
        ur = dict(cond=(pu.marks["cond_begin"], pu.marks["cond_end"]), step=(pu.marks["step_begin"], pu.marks["step_end"]))
        self.unet_lanes: List[engine.DeviceProgram] = [up("unet", pu, ur)]
        for _ in range(1, self.lanes):           # same plan, own workspace, shared weight arena
            self.unet_lanes.append(up("unet", pu, ur, dev_arena=self.unet_lanes[0].arena))
        self.unet = self.unet_lanes[0]
        pd = plan.build_vae_decoder(vae_sd, cfg["vae"], self.latent, batch, scale_factor=scale_factor, **pk)
        self.vae_dec = up("vae_dec", pd, dict(all=(pd.marks["begin"], pd.marks["end"])))
        pv = plan.build_vocoder(vocoder_sd, cfg["vocoder"], self.mel_hw[0], batch, **pk)
        self.vocoder = up("vocoder", pv, dict(all=(pv.marks["begin"], pv.marks["end"])))
        self.vae_enc = None
        if with_encoder:
            self._build_encoder()
        self.n_ctx = len([c for c in (cfg["unet"].get("context_dim") or []) if c is not None])
        self.film = cfg["unet"].get("extra_film_condition_dim") is not None
        self._eps = torch.empty(2, batch, C_, T, Fq, dtype=torch.float32, device=self.device)
        self._engine = self._create_engine()

    def _build_encoder(self):
        pe = plan.build_vae_encoder(self._sd["vae"], self.cfg["vae"], self.mel_hw, self.batch, **self._pk)
        dev_arena = self._arena_bcast("vae_enc", pe.arena, pe.arena.numel()) if self._arena_bcast else None
        self.vae_enc = engine.DeviceProgram(pe, self.device, dict(all=(pe.marks["begin"], pe.marks["end"])), dev_arena)

    def _create_engine(self):
        L = _lib.lib()
        d = _lib.EngineDesc()
        d.n_lanes = self.lanes
        for i, u in enumerate(self.unet_lanes):
            ln = d.lane[i]
            ln.cond, ln.step = u.handles["cond"].value, u.handles["step"].value
            ln.x_slot, ln.t_slot, ln.eps_slot = u.view("x").data_ptr(), u.view("t").data_ptr(), u.view("eps").data_ptr()
            for s in range(self.n_ctx):
                ln.ctx_slot[s], ln.mask_slot[s] = u.view(f"ctx{s}").data_ptr(), u.view(f"mask{s}").data_ptr()
            if self.film:
                ln.film_slot = u.view("y").data_ptr()
        u = self.unet
        d.n_ctx = self.n_ctx
        for s in range(self.n_ctx):
            ctx = u.view(f"ctx{s}")
            d.ctx_len[s], d.ctx_dim[s] = ctx.shape[1], ctx.shape[2]
        if self.film:
            d.film_dim = u.view("y").shape[1]
        d.vae_dec, d.vocoder = self.vae_dec.handles["all"].value, self.vocoder.handles["all"].value
        d.vae_enc = self.vae_enc.handles["all"].value if self.vae_enc is not None else None
        d.z_slot, d.mel_slot = self.vae_dec.view("z").data_ptr(), self.vae_dec.view("mel").data_ptr()
        d.voc_mel_slot, d.wave_slot = self.vocoder.view("mel").data_ptr(), self.vocoder.view("wave").data_ptr()
        if self.vae_enc is not None:
            d.enc_mel_slot, d.moments_slot = self.vae_enc.view("mel").data_ptr(), self.vae_enc.view("moments").data_ptr()
        d.B = self.batch
        d.latent_elems = int(np.prod(self.latent))
        d.mel_elems = self.mel_hw[0] * self.mel_hw[1]
        d.wave_len = self.vocoder.view("wave").shape[-1]
        d.use_graph = int(self.use_graph)
        h = C.c_void_p()
        _lib.check(L.aldm_engine_create(C.byref(d), C.byref(h)), "engine_create")
        self._engine_desc = d
        return h

    def __del__(self):
        try:
            if getattr(self, "_engine", None):
                _lib.lib().aldm_engine_destroy(self._engine)
                self._engine = None
        except Exception:
            pass

    @staticmethod
    def _st() -> int:
        return torch.cuda.current_stream().cuda_stream

    # ------------------------------------------------------------------------------------------
    # conditioning (DiffusionWrapper.forward's dict unpacking, ddpm.py:1821-1879)
    # ------------------------------------------------------------------------------------------
    def _unpack(self, c: dict) -> dict:
        if "context_list" not in c and self.conditioning_key is not None:
            c = reorder_cond_dict(c, self.conditioning_key)              # apply_model (ddpm.py:1034-1035)
        return unpack_cond_dict(c)

    def set_conditioning(self, cond: dict, uncond: Optional[dict] = None):
        """Half 0 of every conditioning buffer holds the unconditional, half 1 the conditional branch (``uncond`` None:
        the conditional one in both).  Cross-attention K/V of every layer are computed here once per call (step-invariant)."""
        L, st, B = _lib.lib(), self._st(), self.batch
        cond = self._unpack(cond)
        uncond = cond if uncond is None else self._unpack(uncond)
        keep = []
        for half, c in ((0, uncond), (1, cond)):
            a = [None, None, 0, None, None, 0]
            assert len(c["context_list"]) == self.n_ctx == len(c["mask_list"]), \
                f"the UNet takes {self.n_ctx} cross-attention contexts, got {len(c['context_list'])}"
            for s_ in range(self.n_ctx):
                cl = c["context_list"][s_].to(self.device, torch.float32).contiguous()
                ml = c["mask_list"][s_].to(self.device, torch.float32).contiguous()
                assert cl.dim() == 3 and cl.shape[0] == B and tuple(ml.shape) == tuple(cl.shape[:2]), (cl.shape, ml.shape, B)
                assert cl.shape[2] == self._engine_desc.ctx_dim[s_], (cl.shape, self._engine_desc.ctx_dim[s_])
                keep += [cl, ml]
                a[3 * s_], a[3 * s_ + 1], a[3 * s_ + 2] = cl.data_ptr(), ml.data_ptr(), cl.shape[1]
            y = None
            if self.film:
                y = c["y"].to(self.device, torch.float32).contiguous()
                assert tuple(y.shape) == (B, self._engine_desc.film_dim), y.shape
            keep.append(y)
            _lib.check(L.aldm_engine_set_conditioning(self._engine, half, *a, y.data_ptr() if y is not None else None, st),
                       "engine_set_conditioning")
        _lib.check(L.aldm_engine_precompute(self._engine, st), "engine_precompute")
        self._cond_keep = keep           # the copies above are asynchronous

    def apply_model_pair(self, x: torch.Tensor, t: int):
        """Both apply_model calls of ddim.py:293-296 in one batched evaluation -> (eps_uncond, eps_cond)."""
        assert x.shape[0] == self.batch and x.is_contiguous() and x.dtype == torch.float32
        _lib.check(_lib.lib().aldm_engine_unet_eps(self._engine, x.data_ptr(), int(t), self._eps[0].data_ptr(),
                                                   self._eps[1].data_ptr(), self._st()), "engine_unet_eps")
        return self._eps[0], self._eps[1]

    def apply_model(self, x, t, cond: dict):
        """ddpm.py:1034-1042 for a single conditioning (runs the batched program with cond in both halves)."""
        self.set_conditioning(cond, None)
        tv = int(t[0]) if torch.is_tensor(t) else int(t)
        return self.apply_model_pair(x.to(self.device, torch.float32).contiguous(), tv)[1].clone()

    def p_sample_ddim(self, x, st: dict, noise, guidance: float, out=None, pred_x0=None):
        """ddim.py:265-355: eps_u/eps_c, e = e_u + s (e_c - e_u), x_{t-1} update -- one graph replay + K6."""
        out = torch.empty_like(x) if out is None else out
        assert x.is_contiguous() and noise.is_contiguous() and out.is_contiguous() and x.shape[0] == self.batch
        _lib.check(_lib.lib().aldm_engine_ddim_step(
            self._engine, x.data_ptr(), int(st["t"]), noise.data_ptr(), st["a_t"], st["a_prev"], st["sigma_t"],
            st["sqrt_one_minus_at"], float(guidance), out.data_ptr(), pred_x0.data_ptr() if pred_x0 is not None else None,
            self._st()), "engine_ddim_step")
        return out

    def p_sample_plms(self, x_in, t: int, x_base, held: Sequence[torch.Tensor], order: int, st: dict, guidance: float,
                      e_t_out=None, out=None, pred_x0=None):
        """One get_model_output + get_x_prev_and_pred_x0 of plms.py:281-358: eps_u/eps_c at (x_in, t), e_t = e_u + s (e_c -
        e_u), e' of ``order`` (1-4, or _lib.PLMS_AVERAGE with held = [the first evaluation's e_t]) over ``held`` (most
        recent first), x_prev from ``x_base`` with the step's coefficients ``st`` -- one graph replay + the PLMS kernel.
        ``e_t_out`` receives e_t.  ``out`` may be ``x_in`` but not ``x_base``."""
        out = torch.empty_like(x_base) if out is None else out
        bufs = [x_in, x_base, out] + list(held) + [b for b in (e_t_out, pred_x0) if b is not None]
        assert all(b.is_contiguous() and b.dtype == torch.float32 and b.shape == x_base.shape for b in bufs)
        assert x_base.shape[0] == self.batch and len(held) <= 3
        h = [b.data_ptr() for b in held] + [None] * (3 - len(held))
        _lib.check(_lib.lib().aldm_engine_plms_step(
            self._engine, x_in.data_ptr(), int(t), x_base.data_ptr(), *h, int(order),
            e_t_out.data_ptr() if e_t_out is not None else None, st["a_t"], st["a_prev"], st["sqrt_one_minus_at"],
            float(guidance), out.data_ptr(), pred_x0.data_ptr() if pred_x0 is not None else None, self._st()),
            "engine_plms_step")
        return out

    def stochastic_encode(self, x0, noise, c0: float, c1: float, clip_flag=None):
        """The arithmetic of DDIMSampler.stochastic_encode (ddim.py:434-449) with AudioLDM 1's guard word -- one native
        pass, no host synchronisation."""
        return engine.stochastic_encode(x0, noise, c0, c1, clip_flag)

    def masked_blend(self, img, x0, mask, q_noise, st: dict):
        return engine.masked_blend(img, x0, mask, q_noise, st["sqrt_acp_t"], st["sqrt_1m_acp_t"])

    # ------------------------------------------------------------------------------------------
    # first stage
    # ------------------------------------------------------------------------------------------
    def decode_first_stage(self, z: torch.Tensor) -> torch.Tensor:
        """ddpm.py:922-926 -> mel [B, 1, T', F'] (a view into the decoder workspace)."""
        z = z.to(self.device, torch.float32).contiguous()
        assert z.shape[0] == self.batch
        _lib.check(_lib.lib().aldm_engine_vae_decode(self._engine, z.data_ptr(), None, self._st()), "engine_vae_decode")
        return self.vae_dec.view("mel")

    def mel_spectrogram_to_waveform(self, mel: torch.Tensor) -> torch.Tensor:
        """ddpm.py:928-939 (without the .cpu().numpy()): mel [B,1,T,F] -> waveform [B,1,L] on the device."""
        B = mel.shape[0]
        assert B == self.batch
        m = mel.reshape(B, mel.shape[-2], mel.shape[-1]).to(self.device, torch.float32).contiguous()
        _lib.check(_lib.lib().aldm_engine_vocoder(self._engine, m.data_ptr(), None, self._st()), "engine_vocoder")
        return self.vocoder.view("wave")

    def encode_first_stage_moments(self, mel: torch.Tensor) -> torch.Tensor:
        """encode_first_stage up to the moments (ddpm.py:941-943), channels-last [B, T, F, 2C]."""
        if self.vae_enc is None:
            self._build_encoder()
            _lib.lib().aldm_engine_destroy(self._engine)
            self._engine = self._create_engine()
        mel = mel.to(self.device, torch.float32).contiguous()
        assert mel.shape[0] == self.batch
        _lib.check(_lib.lib().aldm_engine_vae_encode(self._engine, mel.data_ptr(), None, self._st()), "engine_vae_encode")
        return self.vae_enc.view("moments")

    def get_first_stage_encoding(self, moments: torch.Tensor, noise: torch.Tensor) -> torch.Tensor:
        """DiagonalGaussianDistribution.sample + scale (distributions.py:24-41, ddpm.py:793-802)."""
        return engine.posterior_sample(moments, noise.to(self.device).contiguous(), self.scale_factor)

    # ------------------------------------------------------------------------------------------
    # generate_batch (ddpm.py:1477-1570) minus the conditioning encoders and the CLAP re-ranker
    # ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def generate_latent(self, cond: dict, uncond: Optional[dict], ddim_steps: int = 200, guidance: float = 3.5, eta: float = 1.0,
                        x_T=None, noise_fn=None, mask=None, x0=None, use_plms: bool = False):
        """sample_log (ddpm.py:1449-1461): DDIM, or PLMS with ``use_plms`` (``eta`` then ignored, as the reference does)."""
        sampler = PLMSSampler(self) if use_plms else DDIMSampler(self)
        z, _ = sampler.sample(S=ddim_steps, batch_size=self.batch, shape=self.latent, conditioning=cond, eta=eta,
                              unconditional_guidance_scale=guidance, unconditional_conditioning=uncond, x_T=x_T,
                              noise_fn=noise_fn, mask=mask, x0=x0)
        return z

    @torch.no_grad()
    def generate_waveform(self, cond: dict, uncond: Optional[dict], ddim_steps: int = 200, guidance: float = 3.5, eta: float = 1.0,
                          x_T=None, noise_fn=None, mask=None, x0=None, use_plms: bool = False):
        z = self.generate_latent(cond, uncond, ddim_steps, guidance, eta, x_T, noise_fn, mask, x0, use_plms)
        mel = self.decode_first_stage(z)
        return self.mel_spectrogram_to_waveform(mel)

    @torch.no_grad()
    def style_transfer_latent(self, x0, cond: dict, uncond: Optional[dict], t_enc: int, ddim_steps: int = 200,
                              guidance: float = 2.5, clip_flag=None, noise=None, noise_fn=None):
        """AudioLDM 1's style_transfer from the initial latent ``x0`` on: make_schedule(ddim_steps, eta=1.0),
        stochastic_encode at index ``t_enc`` (one draw, or ``noise``), then decode with indices t_enc - 1, ..., 0 (one
        draw per step, or ``noise_fn(i, "step")``).  ``clip_flag``: the device guard word of
        parallel.latent_guard_flag; None makes it from ``x0`` (the whole batch of a single-process call)."""
        sampler = DDIMSampler(self)
        sampler.make_schedule(ddim_num_steps=ddim_steps, ddim_eta=1.0)
        x0 = x0.to(self.device, torch.float32).contiguous()
        if clip_flag is None:
            clip_flag = parallel.guard_decision(parallel.guard_flags(x0))
        z_enc = sampler.stochastic_encode(x0, t_enc, noise=noise, clip_flag=clip_flag)
        return sampler.decode(z_enc, cond, t_enc, unconditional_guidance_scale=guidance, unconditional_conditioning=uncond,
                              noise_fn=noise_fn)

    @torch.no_grad()
    def style_transfer_waveform(self, x0, cond: dict, uncond: Optional[dict], t_enc: int, ddim_steps: int = 200,
                                guidance: float = 2.5, clip_flag=None, noise=None, noise_fn=None):
        """style_transfer_latent, then the whole latent decoded and vocoded as generate_batch does."""
        z = self.style_transfer_latent(x0, cond, uncond, t_enc, ddim_steps, guidance, clip_flag, noise, noise_fn)
        return self.mel_spectrogram_to_waveform(self.decode_first_stage(z))

    def launches_per_step(self) -> int:
        return self.lanes * (self.unet.num_launches("step") + 1 + 1)      # + timestep fill + K6, per lane

    def launches_decode(self) -> int:
        return self.vae_dec.num_launches("all") + self.vocoder.num_launches("all")

    def launches_cond(self) -> int:
        return self.lanes * self.unet.num_launches("cond")


def build_synthetic(model_name: str = "audioldm2-full", batch: int = 1, device="cuda:0", cfg: Optional[dict] = None,
                    t5_len: int = 32, **kw) -> NativeLatentDiffusion:
    """Engine on the seeded synthetic checkpoint (no network: hub checkpoints are unreachable)."""
    from . import synth
    cfg = cfg or arch.model_config(model_name)
    lens = (8, t5_len) if len([c for c in cfg["unet"]["context_dim"] if c is not None]) > 1 else (t5_len,)
    kw.setdefault("ctx_max_len", lens)
    return NativeLatentDiffusion(cfg, synth.unet_state_dict(cfg["unet"]), synth.vae_state_dict(cfg["vae"]),
                                 synth.vocoder_state_dict(cfg["vocoder"]), batch, device, **kw)
