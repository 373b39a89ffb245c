"""Drop-in surface of ``audioldm2/pipeline.py`` for the sampling hot path.

``build_model`` / ``text_to_audio`` / ``super_resolution_and_inpainting`` keep the reference's signatures, positional
order and defaults (pipeline.py:142-267); extra keyword-only arguments configure what the reference obtains from the
network.  What differs, by design of this tier:

* the conditioning encoders (CLAP / Flan-T5) are out of scope and need hub downloads that are unreachable offline:
  conditioning comes from ``latent_diffusion.cond_provider`` (``.cond(batch)`` for the prompts, ``.uncond(n)`` for the
  unconditional branch); the default provider of a synthetic build is the seeded one of SURVEY.md 8d.  A provider may
  return the UNet-boundary conditioning (the reference's keyed cond-dict or the unpacked form, model.unpack_cond_dict),
  or, for the sequence-generation models (audioldm2-full / -large), the encoder outputs ``film_clap_cond1`` [B, 1, 512]
  and ``crossattn_flan_t5`` [h [B, L, 1024], mask [B, L]]: the AudioMAE tokens are then generated natively by GPT-2
  (seqgen.NativeAudioMAEGenerator), on the B prompts before the n_gen tiling as in generate_batch (ddpm.py:1500-1523);
  or, for every model with a Flan-T5 context (audioldm2-full / -large, the *_t5 models), the tokenizer's output under the
  reference's own key, ``crossattn_flan_t5`` = [input_ids (integer) [B, L], attention_mask [B, L]] (plus
  ``film_clap_cond1`` for the sequence-generation models): the T5 states are then encoded natively
  (t5.NativeFlanT5Encoder) before anything else, in the conditional and the unconditional dict alike;
  and for every model conditioned on the CLAP text embedding (audioldm2-full / -large, audioldm_48k), the RoBERTa
  tokenizer's output under the reference's key, ``film_clap_cond1`` = [input_ids (integer) [B, L], attention_mask [B, L]]:
  the embedding is then computed natively (clap.NativeCLAPTextEncoder) before everything else, with the reference's random
  replacement of prompt rows by CLAP("") (clap_replacement_draws);
* candidate re-ranking (ddpm.py:1554-1568) is the reference's ``clap.cos_similarity``, run natively
  (clap.NativeCLAPRanker: the HTSAT audio branch and the RoBERTa text branch of ``clap.model.*``, with forward's random
  replacement by CLAP("")) when the model is built with ``clap_tokenize=`` (the caller's RoBERTa tokenizer); it ranks the
  waveforms on the device and only the selected ones are copied to the host.  Otherwise a Python
  ``latent_diffusion.ranker(waveform [n,1,L], texts) -> similarity [n]`` may be attached; without either the first
  candidate of each prompt is returned and a warning says so;
* the engine is planned per (latent batch, latent length); ``NativeAudioLDM2.engine`` re-plans on demand and caches.
"""
from __future__ import annotations

import warnings
from typing import Callable, Dict, Optional, Tuple

import numpy as np
import torch

from . import arch, engine, frontend, model, parallel, synth
from . import sampler as sampler_mod
from .utils import seed_everything


class SyntheticConditioning:
    """Seeded conditioning at the UNet boundary (SURVEY.md 8d): per-prompt rows for the conditional branch, one shared
    row for the unconditional one (T5("") / zero AudioMAE tokens / zero FiLM vector)."""

    def __init__(self, cfg: dict, seed: int = 77, t5_len: int = 32, device="cpu"):
        self.cfg, self.seed, self.t5_len, self.device = cfg, seed, t5_len, device

    def cond(self, batch: dict) -> dict:
        n = len(batch["text"])
        return synth.conditioning(self.cfg, n, seed=self.seed, t5_len=self.t5_len, device=self.device)[0]

    def uncond(self, n: int) -> dict:
        return synth.conditioning(self.cfg, n, seed=self.seed, t5_len=self.t5_len, device=self.device)[1]


class SyntheticEncoderOutputs:
    """Seeded encoder outputs for the sequence-generation models (opt-in; SyntheticConditioning stays the default): an
    L2-normalised CLAP embedding [B, 1, 512] and Flan-T5 states N(0, 1) [B, L, 1024] with per-row lengths (row i holds
    ``t5_lens[i % len]`` tokens, L = the longest, as padding=True pads to the longest prompt).  The unconditional branch
    is SyntheticConditioning's single-prompt one repeated on every row (zero AudioMAE tokens, one T5("") row): like the
    reference's, it does not depend on how many rows are asked for, so a rank of a sharded call sees the same rows as one
    process."""

    def __init__(self, cfg: dict, seed: int = 78, t5_lens=(32, 19, 7), t5_len: int = 32, device="cpu"):
        if not arch.has_seqgen(cfg):
            raise ValueError(f"{cfg.get('name')}: encoder outputs need the AudioMAE token generator, which this model has not")
        self.cfg, self.seed, self.t5_lens, self.device = cfg, seed, tuple(t5_lens), device
        self._uncond = SyntheticConditioning(cfg, t5_len=t5_len, device=device)

    def cond(self, batch: dict) -> dict:
        n = len(batch["text"])
        clap, t5, mask = synth.encoder_outputs(n, [self.t5_lens[i % len(self.t5_lens)] for i in range(n)], seed=self.seed,
                                               device=self.device)
        return {"film_clap_cond1": clap, "crossattn_flan_t5": [t5, mask]}

    def uncond(self, n: int) -> dict:
        u = self._uncond.uncond(1)
        return {k: ([t.expand(n, *t.shape[1:]).contiguous() for t in v] if isinstance(v, list) else
                    (v.expand(n, *v.shape[1:]).contiguous() if torch.is_tensor(v) else v)) for k, v in u.items()}


class SyntheticTokenIds:
    """Seeded tokenizer output for every model with a Flan-T5 context (opt-in): ``crossattn_flan_t5`` = [ids, mask] with
    per-row token counts (row i holds ``lens[i % len]`` tokens ending in EOS, L = the longest: padding=True), and for the
    sequence-generation models an L2-normalised CLAP embedding [B, 1, 512].  The unconditional branch is the tokenization
    of "" ([[1]] on every row) next to zero AudioMAE tokens where the model has them: the same rows whatever the row
    count, as in the reference."""

    def __init__(self, cfg: dict, seed: int = 79, lens=(32, 19, 7), device="cpu"):
        if not arch.has_t5(cfg):
            raise ValueError(f"{cfg.get('name')}: token ids need a Flan-T5 context, which this model has not")
        self.cfg, self.seed, self.lens, self.device = cfg, seed, tuple(lens), device

    def cond(self, batch: dict) -> dict:
        n = len(batch["text"])
        ids, mask = synth.token_ids([self.lens[i % len(self.lens)] for i in range(n)], seed=self.seed, device=self.device)
        out = {}
        if arch.has_seqgen(self.cfg):
            g = torch.Generator(device="cpu"); g.manual_seed(self.seed + 1)
            clap = torch.randn(n, 1, 512, generator=g)
            out["film_clap_cond1"] = (clap / clap.norm(dim=-1, keepdim=True)).to(self.device)
        out["crossattn_flan_t5"] = [ids, mask]
        return out

    def uncond(self, n: int) -> dict:
        one = torch.ones(n, 1, device=self.device)
        out = {}
        if arch.has_seqgen(self.cfg):                 # zero AudioMAE tokens (encoders/modules.py:476-479)
            out["crossattn_audiomae_generated"] = [torch.zeros(n, 8, 768, device=self.device), torch.ones(n, 8, device=self.device)]
        out["crossattn_flan_t5"] = [(one * arch.T5["eos_id"]).long(), one]
        return out


class SyntheticPromptTokens:
    """Seeded tokenizer output for every model conditioned on the CLAP text embedding (opt-in): ``film_clap_cond1`` =
    [ids, mask] padded to the RoBERTa tokenizer's 512 (padding="max_length"; row i holds ``lens[i % len]`` tokens, BOS and
    EOS included), plus Flan-T5 ids (SyntheticTokenIds' layout, ``t5_lens``) where the model has a Flan-T5 context.  The
    unconditional branch is the reference's: the tokenization of "" on every row for audioldm_48k, zero AudioMAE tokens
    and T5("") for the sequence-generation models."""

    def __init__(self, cfg: dict, seed: int = 81, lens=(24, 11, 5), t5_lens=(32, 19, 7), device="cpu"):
        if not arch.has_clap(cfg):
            raise ValueError(f"{cfg.get('name')}: CLAP token ids need a model conditioned on the CLAP text embedding")
        self.cfg, self.seed, self.lens, self.device = cfg, seed, tuple(lens), device
        self._t5 = SyntheticTokenIds(cfg, seed=seed + 1, lens=t5_lens, device=device) if arch.has_t5(cfg) else None

    def cond(self, batch: dict) -> dict:
        n = len(batch["text"])
        ids, mask = synth.clap_token_ids([self.lens[i % len(self.lens)] for i in range(n)], seed=self.seed, device=self.device)
        out = {"film_clap_cond1": [ids, mask]}
        if self._t5 is not None:
            out["crossattn_flan_t5"] = self._t5.cond(batch)["crossattn_flan_t5"]
        return out

    def uncond(self, n: int) -> dict:
        if self._t5 is not None:                    # SequenceGenAudioMAECond's cfg_uncond and T5(""): no CLAP entry
            return self._t5.uncond(n)
        from .clap import empty_prompt
        return {"film_clap_cond1": list(empty_prompt(n, device=self.device))}


def is_clap_token_level(cond) -> bool:
    """The CLAP entry holds the tokenizer's output (integer ids) rather than the embedding."""
    if not isinstance(cond, dict) or not isinstance(cond.get("film_clap_cond1"), (list, tuple)):
        return False
    ids = cond["film_clap_cond1"][0]
    return torch.is_tensor(ids) and not ids.dtype.is_floating_point and not ids.dtype.is_complex


def clap_replacement_draws(n: int, extra: bool) -> list:
    """The CPU draws of the reference's get_input for the CLAP conditioner, in its order: with ``extra`` (every call of a
    model after its first: conditional_dry_run_finished) LatentDiffusion.make_decision(0.0) draws one torch.rand(1)
    (ddpm.py:852-854); then CLAPAudioEmbeddingClassifierFreev2.forward draws one per prompt row, in row order, and replaces
    the row by CLAP("") below unconditional_prob = 0.1 (encoders/modules.py:731-733).  -> the n decisions."""
    from .clap import replacement_draws
    if extra:
        torch.rand(1)                               # make_decision(0.0): drawn, never true
    return replacement_draws(n)


def encode_clap_tokens(cfg: dict, cond: dict, encoder: Callable[[], object], unconditional: bool = False,
                       decide: Optional[Callable[[int], list]] = None) -> dict:
    """Replace token-level ``film_clap_cond1`` = [ids, mask] by the embedding [B, 1, 512] (every other entry is kept, in
    order); anything else is returned as it is, the encoder is never built and nothing is drawn.  In the conditional dict
    ``decide(B)`` gives the rows replaced by CLAP("") (clap_replacement_draws; None: no replacement).  In the
    unconditional dict, rows that are all the tokenization of "" go through ``encoder().unconditional()``, computed once
    and cached like the reference's unconditional_token (get_unconditional_condition, encoders/modules.py:606-610)."""
    if not is_clap_token_level(cond):
        return cond
    if not arch.has_clap(cfg):
        raise ValueError(f"{cfg.get('name')} has no CLAP text conditioning: token ids under film_clap_cond1 do not apply")
    from .clap import is_empty_prompt
    ids, mask = cond["film_clap_cond1"]
    enc = encoder()
    if unconditional and is_empty_prompt(ids, mask):
        e = enc.unconditional().expand(ids.shape[0], -1).clone()
    else:
        e = enc.embed(ids, mask)
        if not unconditional and decide is not None:
            rows = [i for i, r in enumerate(decide(ids.shape[0])) if r]
            if rows:
                e[rows] = enc.unconditional().to(e.device)
    return {k: (e[:, None, :] if k == "film_clap_cond1" else v) for k, v in cond.items()}


def is_token_level(cond) -> bool:
    """The Flan-T5 entry holds the tokenizer's output (integer ids) rather than hidden states."""
    if not isinstance(cond, dict) or not isinstance(cond.get("crossattn_flan_t5"), (list, tuple)):
        return False
    ids = cond["crossattn_flan_t5"][0]
    return torch.is_tensor(ids) and not ids.dtype.is_floating_point and not ids.dtype.is_complex


def encode_tokens(cfg: dict, cond: dict, encoder: Callable[[], object], unconditional: bool = False) -> dict:
    """Replace token-level ``crossattn_flan_t5`` = [ids, mask] by [encoder().encode(ids, mask), mask.float()] (every other
    entry is kept, in order); anything else is returned as it is and the encoder is never built.  In the unconditional
    dict, the tokenization of "" ([[1]] on every row, mask 1) goes through ``encoder().unconditional(n)``, computed once
    and cached like the reference's T5("") (encoders/modules.py:139-154)."""
    if not is_token_level(cond):
        return cond
    if not arch.has_t5(cfg):
        raise ValueError(f"{cfg.get('name')} has no Flan-T5 context: token ids under crossattn_flan_t5 do not apply")
    ids, mask = cond["crossattn_flan_t5"]
    enc = encoder()
    if unconditional and ids.shape[1] == 1 and bool((ids == arch.T5["eos_id"]).all()) and bool((mask == 1).all()):
        h = enc.unconditional(ids.shape[0])
    else:
        h = enc.encode(ids, mask)
    return {k: ([h, mask.float().to(h.device)] if k == "crossattn_flan_t5" else v) for k, v in cond.items()}


def is_encoder_level(cond: dict) -> bool:
    """Encoder outputs rather than UNet-boundary conditioning: CLAP + Flan-T5 present, no AudioMAE tokens, not unpacked."""
    return isinstance(cond, dict) and "film_clap_cond1" in cond and "crossattn_flan_t5" in cond and \
        "crossattn_audiomae_generated" not in cond and "context_list" not in cond


def route_conditioning(cfg: dict, cond: dict, generator: Callable[[], object]) -> dict:
    """UNet-boundary conditioning is returned as it is (the generator is never built).  Encoder outputs go through
    ``generator().generate`` -> {"crossattn_audiomae_generated": [tokens, ones], "crossattn_flan_t5": [h, mask]}, the
    UNet's context order (SequenceGenAudioMAECond.forward, encoders/modules.py:281-300)."""
    if not is_encoder_level(cond):
        return cond
    if not arch.has_seqgen(cfg):
        raise ValueError(f"{cfg.get('name')} has no AudioMAE token generator: give UNet-boundary conditioning "
                         "(context_list / crossattn_* entries), not CLAP + Flan-T5 encoder outputs")
    h, m = cond["crossattn_flan_t5"]
    tokens = generator().generate(cond["film_clap_cond1"], h, m)
    return {"crossattn_audiomae_generated": [tokens, torch.ones(tokens.shape[:2], device=tokens.device)],
            "crossattn_flan_t5": [h, m]}


def _tile(c, n_gen: int):
    """The n_gen tiling of generate_batch (ddpm.py:1516-1525): torch.cat([t] * n_gen) on every tensor, so the candidates
    of prompt i sit at rows i + k * batchsize."""
    if n_gen == 1 or c is None:
        return c
    if torch.is_tensor(c):
        return torch.cat([c] * n_gen, dim=0)
    if isinstance(c, dict):
        return {k: _tile(v, n_gen) for k, v in c.items()}
    if isinstance(c, (list, tuple)):
        return [_tile(v, n_gen) for v in c]
    return c


def select_best(waveform: np.ndarray, similarity, batchsize: int):
    """ddpm.py:1554-1564: per prompt i take the candidate (rows i, i+B, i+2B, ...) with the highest similarity."""
    sim = torch.as_tensor(similarity).reshape(-1)
    best_index = []
    for i in range(batchsize):
        candidates = sim[i::batchsize]
        best_index.append(i + int(torch.argmax(candidates).item()) * batchsize)
    return waveform[best_index], best_index


class NativeAudioLDM2:
    """What ``build_model`` returns: the reference's ``LatentDiffusion`` seen from pipeline.py (``generate_batch``,
    ``generate_batch_masked``, ``latent_t_size``) over per-shape native engines."""

    def __init__(self, cfg: dict, unet_sd, vae_sd, vocoder_sd, device, scale_factor: float = 1.0, ctx_max_len=None,
                 cond_provider=None, ranker: Optional[Callable] = None, seqgen_sd=None, t5_sd=None, t5_uncond_sd=None,
                 clap_sd=None, clap_rank_sd=None, clap_tokenize=None, **engine_kw):
        """``t5_sd`` / ``t5_uncond_sd``: the Flan-T5 weights of the conditional and of the unconditional branch (or callables
        that return them, for weights made on first use); ``t5_uncond_sd`` None means the same weights.  ``clap_sd``: the
        CLAP text branch's weights (or a callable).  ``clap_tokenize``: the RoBERTa tokenizer, ``texts -> (ids, mask)``; with
        it candidates are ranked natively by the weights of ``clap_rank_sd``, (audio branch, text branch) of the reference's
        ``clap.model``, each a state dict or a callable that returns one."""
        if ranker is not None and clap_tokenize is not None:
            raise ValueError("pass either a ranker or clap_tokenize (the native CLAP ranker), not both")
        if clap_tokenize is not None and cfg.get("sampling_rate") not in (16000, 48000):
            raise ValueError(f"{cfg.get('name')}: the native CLAP ranker takes 16 or 48 kHz audio, "
                             f"not {cfg.get('sampling_rate')} Hz")
        self.cfg, self.device = cfg, torch.device(device)
        self._sd = (unet_sd, vae_sd, vocoder_sd)
        self.scale_factor = scale_factor
        self.ctx_max_len = ctx_max_len
        self.engine_kw = engine_kw
        self.cond_provider, self.ranker = cond_provider, ranker
        self.latent_t_size = cfg["latent"][1]                 # pipeline.py:200 overwrites it per call
        self.cond_stage_key = "text"
        self._engines: Dict[Tuple[int, int, bool], model.NativeLatentDiffusion] = {}
        self._pinned: Dict[Tuple[int, ...], torch.Tensor] = {}
        self._seqgen_sd = seqgen_sd
        self._seqgen = None
        self._t5_sd, self._t5_uncond_sd = t5_sd, t5_uncond_sd
        self._t5 = None
        self._clap_sd = clap_sd
        self._clap = None
        self._clap_rank_sd, self.clap_tokenize = clap_rank_sd, clap_tokenize
        self._native_ranker = None
        self.conditional_dry_run_finished = False           # LatentDiffusion's flag (ddpm.py:852-854, 916-917)

    # ---- AudioMAE token generator (built on first use: UNet-boundary providers never pay for it) ----------------------
    def seqgen(self):
        if self._seqgen is None:
            if self._seqgen_sd is None:
                raise ValueError("encoder-level conditioning needs the AudioMAE generator's weights (cond_stage_models.<i>.*), "
                                 "which this model was built without")
            from .seqgen import NativeAudioMAEGenerator
            self._seqgen = NativeAudioMAEGenerator(self._seqgen_sd, self.device)
        return self._seqgen

    # ---- Flan-T5 encoder (built on first token-level use) ---------------------------------------------------
    def t5_encoders(self):
        """(conditional, unconditional) native encoders.  One packed arena serves both when the two weight sets are
        equal (the checkpoint holds two frozen copies of the same pretrained encoder), otherwise each has its own."""
        if self._t5 is None:
            if self._t5_sd is None:
                raise ValueError("token-level conditioning needs the Flan-T5 weights, which this model was built without")
            from .t5 import NativeFlanT5Encoder
            get = lambda w: w() if callable(w) else w
            sd_c = get(self._t5_sd)
            enc_c = NativeFlanT5Encoder(sd_c, self.device)
            enc_u = enc_c
            if self._t5_uncond_sd is not None:
                sd_u = get(self._t5_uncond_sd)
                same = sd_u is sd_c or (set(sd_u) == set(sd_c) and all(torch.equal(sd_u[k], sd_c[k]) for k in sd_c))
                if not same:
                    enc_u = NativeFlanT5Encoder(sd_u, self.device)
            self._t5 = (enc_c, enc_u)
        return self._t5

    # ---- CLAP text encoder (built on first token-level use) ------------------------------------------------
    def clap_encoder(self):
        if self._clap is None:
            if self._clap_sd is None:
                raise ValueError("token-level film_clap_cond1 needs the CLAP text weights, which this model was built without")
            from .clap import NativeCLAPTextEncoder
            self._clap = NativeCLAPTextEncoder(self._clap_sd() if callable(self._clap_sd) else self._clap_sd, self.device)
        return self._clap

    # ---- native CLAP re-ranker (built on the first call with n_gen > 1) ------------------------------------------
    def native_ranker(self):
        """clap.NativeCLAPRanker over the reference's ``clap.model``.  Its text branch shares the conditioning CLAP text
        encoder (arena and cached CLAP("")) when the two weight sets are equal."""
        if self._native_ranker is None:
            from .clap import NativeCLAPAudioEncoder, NativeCLAPRanker, NativeCLAPTextEncoder
            get = lambda w: w() if callable(w) else w
            src_a, src_t = self._clap_rank_sd
            text = None
            if self._clap_sd is not None:
                if src_t is self._clap_sd:                  # the same weights, or the same generator of synthetic ones
                    text = self.clap_encoder()
                elif not callable(src_t) and not callable(self._clap_sd):
                    sd_c = self._clap_sd
                    if set(sd_c) == set(src_t) and all(torch.equal(sd_c[k], src_t[k]) for k in src_t):
                        text = self.clap_encoder()
            if text is None:
                text = NativeCLAPTextEncoder(get(src_t), self.device)
            sd_a = get(src_a)
            audio = NativeCLAPAudioEncoder(sd_a, self.device, sampling_rate=self.cfg["sampling_rate"])
            self._native_ranker = NativeCLAPRanker(audio, text, self.clap_tokenize)
        return self._native_ranker

    def conditioning(self, batch) -> dict:
        """The provider's conditioning of the call's B prompts, as the reference's get_input makes it (after the posterior
        draw): CLAP token ids embedded, with the reference's random replacement by CLAP(""), and Flan-T5 token ids
        encoded; then the AudioMAE tokens generated when it holds encoder outputs."""
        extra = self.conditional_dry_run_finished
        self.conditional_dry_run_finished = True
        cond = encode_clap_tokens(self.cfg, self.cond_provider.cond(batch), self.clap_encoder,
                                  decide=lambda n: clap_replacement_draws(n, extra))
        cond = encode_tokens(self.cfg, cond, lambda: self.t5_encoders()[0])
        return route_conditioning(self.cfg, cond, self.seqgen)

    def _sharded_conditioning(self, batch, lo: int, hi: int) -> dict:
        """Rows [lo, hi) of the conditioning of the whole call: every rank makes the draws of all B prompts, so the
        replacement decisions and the CPU generator state are those of one process."""
        return parallel.shard_rows(self.conditioning(batch), lo, hi)

    def unconditioning(self, n: int, uncond=None) -> dict:
        """The unconditional branch (the provider's unless given), with token ids encoded by the unconditional encoders."""
        u = self.cond_provider.uncond(n) if uncond is None else uncond
        u = encode_clap_tokens(self.cfg, u, self.clap_encoder, unconditional=True)
        return encode_tokens(self.cfg, u, lambda: self.t5_encoders()[1], unconditional=True)

    # ---- engines -------------------------------------------------------------------------------------
    def engine(self, Bl: int, latent_t: Optional[int] = None, with_encoder: bool = False) -> model.NativeLatentDiffusion:
        T = int(latent_t or self.latent_t_size)
        for (b, t, enc), e in self._engines.items():
            if b == Bl and t == T and (enc or not with_encoder):
                return e
        if len(self._engines) >= 2:                          # keep the two most recent plans (1-3 GB of HBM each)
            self._engines.pop(next(iter(self._engines)))
            torch.cuda.empty_cache()
        cfg = dict(self.cfg)
        C_, _, F_ = self.cfg["latent"]
        assert T % 8 == 0, f"latent length {T} must be a multiple of 8 (three stride-2 levels)"
        cfg["latent"] = (C_, T, F_)
        n_cross = len([c for c in cfg["unet"]["context_dim"] if c is not None])
        lens = self.ctx_max_len or ((8, 128) if n_cross > 1 else (128,))
        e = model.NativeLatentDiffusion(cfg, *self._sd, Bl, self.device, scale_factor=self.scale_factor, ctx_max_len=lens,
                                        with_encoder=with_encoder, **self.engine_kw)
        self._engines[(Bl, T, with_encoder)] = e
        return e

    def _egress(self, wave: torch.Tensor) -> np.ndarray:
        """Waveform to host memory (ddpm.py:936 does a blocking ``.cpu().numpy()``): asynchronous copy into a cached
        pinned buffer on the current stream, one event wait, no device-wide synchronisation."""
        key = tuple(wave.shape)
        buf = self._pinned.get(key)
        if buf is None:
            buf = self._pinned[key] = torch.empty(wave.shape, dtype=torch.float32).pin_memory()
        buf.copy_(wave, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        ev.synchronize()
        return buf.numpy().copy()

    # ---- generate_batch (ddpm.py:1477-1570) -------------------------------------------------------------
    @torch.no_grad()
    def generate_batch(self, batch, ddim_steps=200, ddim_eta=1.0, x_T=None, n_gen=1, unconditional_guidance_scale=1.0,
                       unconditional_conditioning=None, use_plms=False, **kwargs):
        return self._generate(batch, ddim_steps, ddim_eta, x_T, n_gen, unconditional_guidance_scale,
                              unconditional_conditioning, use_plms, None, None)

    @torch.no_grad()
    def generate_batch_masked(self, batch, ddim_steps=200, ddim_eta=1.0, x_T=None, n_gen=1, unconditional_guidance_scale=1.0,
                              unconditional_conditioning=None, use_plms=False, time_mask_ratio_start_and_end=(0.25, 0.75),
                              freq_mask_ratio_start_and_end=(0.75, 1.0), **kwargs):
        return self._generate(batch, ddim_steps, ddim_eta, x_T, n_gen, unconditional_guidance_scale,
                              unconditional_conditioning, use_plms, time_mask_ratio_start_and_end, freq_mask_ratio_start_and_end)

    def _generate(self, batch, ddim_steps, ddim_eta, x_T, n_gen, guidance, uncond, use_plms, tmask, fmask):
        """sample_log (ddpm.py:1449-1461): DDIMSampler, or PLMSSampler with ``use_plms`` (which ignores ``ddim_eta``)."""
        assert x_T is None, "the native path draws x_T itself, as pipeline.py's calls do"
        shard = parallel.current_shard(len(batch["text"]))
        if shard is not None:              # one process per GPU: this rank generates prompts [lo, hi) of the call (SURVEY.md 8e)
            return self._generate_sharded(shard, batch, ddim_steps, ddim_eta, n_gen, guidance, uncond, tmask, fmask, use_plms)
        return self._generate_local(batch, ddim_steps, ddim_eta, n_gen, guidance, uncond, tmask, fmask, None, use_plms=use_plms)

    def _generate_sharded(self, shard, batch, ddim_steps, ddim_eta, n_gen, guidance, uncond, tmask, fmask, use_plms=False):
        """Every rank runs the same call with the same seed; prompts are cut into contiguous shards, the noise of the
        single-process latent batch (rows i + k * B) is drawn in full on every rank and sliced, and the selected waveforms are
        all-gathered at the end.  Results equal the single-process call row for row."""
        local, glob, cond_l = self._shard_view(shard, batch, n_gen)
        out = self._generate_local(local, ddim_steps, ddim_eta, n_gen, guidance, uncond, tmask, fmask, glob, cond_l, use_plms)
        full = parallel.all_gather_rows(torch.from_numpy(out).to(self.device), len(batch["text"]))
        return self._egress(full)

    def _shard_view(self, shard, batch, n_gen):
        """This rank's part of a sharded call: (its prompts' batch, (B, its latent rows of the whole call), its rows of the
        whole call's conditioning).  The candidates of prompt i sit at rows i + k * B."""
        _, _, lo, hi = shard
        B = len(batch["text"])
        local = {k: (v[lo:hi] if (torch.is_tensor(v) or isinstance(v, list)) and len(v) == B else v) for k, v in batch.items()}
        rows = [i + k * B for k in range(n_gen) for i in range(lo, hi)]
        # conditioning of the whole call, this rank's rows: made after the posterior draw, as in one process
        cond_l = lambda: self._sharded_conditioning(batch, lo, hi)
        return local, (B, rows), cond_l

    def _encode_front(self, batch, n_gen, glob, eng, encode: bool):
        """The front half shared by generation and the audio-to-audio calls, up to the conditioning: the posterior draw,
        the CUDA noise of a sharded call, and the encoder pass when ``encode`` -> (x0 or None, x_T, noise_fn)."""
        B = len(batch["text"])
        C_, T, F_ = eng.latent
        # get_input -> encode_first_stage -> posterior.sample() (ddpm.py:845-846): a CPU torch.randn of the latent shape
        # (distributions.py:38).  Plain text_to_audio encodes an all-zero fbank only to read z.shape[0]; that encoder pass is
        # skipped here (345 GFLOP per prompt), the CPU draw is kept so every later CPU draw sees the reference's RNG state.
        x_T = noise_fn = None
        if glob is None:
            post_noise = torch.randn(B, C_, T, F_)
        else:                                 # sharded call: draw the global tensors, keep this rank's rows
            Bg, rows = glob
            post_noise = torch.randn(Bg, C_, T, F_)[rows[:B]]
            noise_fn = parallel.ShardedNoise(Bg * n_gen, 0, 0, (C_, T, F_), self.device, rows=rows,
                                             generator=torch.cuda.default_generators[self.device.index or 0])
            x_T = noise_fn.x_T()
        x0 = None
        if encode:
            fbank = torch.as_tensor(batch["log_mel_spec"], dtype=torch.float32)           # [B, T', F']
            mel = _tile(fbank[:, None], n_gen).to(self.device)                            # torch.cat([z] * n_gen) (ddpm.py:1651)
            mom = eng.encode_first_stage_moments(mel)
            x0 = eng.get_first_stage_encoding(mom, _tile(post_noise, n_gen))
        return x0, x_T, noise_fn

    def _generate_local(self, batch, ddim_steps, ddim_eta, n_gen, guidance, uncond, tmask, fmask, glob, cond_rows=None,
                        use_plms=False):
        masked = tmask is not None
        B = len(batch["text"])
        Bl = B * n_gen
        eng = self.engine(Bl, with_encoder=masked)
        C_, T, F_ = eng.latent
        x0, x_T, noise_fn = self._encode_front(batch, n_gen, glob, eng, masked)
        mask = None
        if masked:
            mask = torch.ones(Bl, T, F_, device=self.device)                              # ddpm.py:1611-1617
            mask[:, int(T * tmask[0]):int(T * tmask[1]), :] = 0
            mask[:, :, int(F_ * fmask[0]):int(F_ * fmask[1])] = 0
            mask = mask[:, None].contiguous()
        cond = _tile(cond_rows() if cond_rows is not None else self.conditioning(batch), n_gen)
        if guidance != 1.0:
            uncond = self.unconditioning(Bl, uncond)                                      # ddpm.py:1529-1536
        texts = list(batch["text"]) * n_gen
        wave = eng.generate_waveform(cond, uncond, ddim_steps=ddim_steps, guidance=guidance, eta=ddim_eta, mask=mask, x0=x0,
                                     x_T=x_T, noise_fn=noise_fn, use_plms=use_plms)
        if n_gen > 1 and self.clap_tokenize is not None:
            # the reference ranks the host copy (ddpm.py:1556); the same values are ranked here on the device, and only
            # the B selected waveforms are copied out
            n_total, rows = (Bl, None) if glob is None else (glob[0] * n_gen, glob[1])
            similarity = self.native_ranker()(wave.reshape(Bl, -1), texts, rows=rows, n_total=n_total)
            _, best = select_best(np.zeros(Bl), similarity.cpu(), B)
            return self._egress(wave[best])
        waveform = self._egress(wave)                                                     # ddpm.py:936
        if n_gen > 1:
            if self.ranker is None:
                warnings.warn("no ranker (the reference's clap.cos_similarity, ddpm.py:1556) is attached to this model: "
                              "returning the first of the n_candidate_gen_per_text candidates of every prompt")
                return waveform[:B]
            similarity = self.ranker(torch.from_numpy(waveform).squeeze(1), texts)
            waveform, _ = select_best(waveform, similarity, B)
        return waveform

    # ---- style transfer (AudioLDM 1's style_transfer on AudioLDM2's primitives) ---------------------------------------
    @torch.no_grad()
    def generate_batch_style_transfer(self, batch, transfer_strength, ddim_steps=200, unconditional_guidance_scale=1.0,
                                      unconditional_conditioning=None):
        """The recording in ``batch["log_mel_spec"]`` encoded to its latent (one CPU posterior draw), AudioLDM 1's latent
        guard, the conditioning of ``batch["text"]``, then DDIMSampler.stochastic_encode at t_enc = int(transfer_strength
        * ddim_steps) (one CUDA draw) and decode over indices t_enc - 1, ..., 0 (one CUDA draw per step), decoder and
        vocoder -> np.ndarray [B, 1, samples].  In a sharded call each rank runs its prompts' rows with the whole call's
        draws, the guard's two flags are all-reduced once, and the waveforms are all-gathered at the end."""
        t_enc = sampler_mod.transfer_steps(transfer_strength, ddim_steps, self.cfg["timesteps"])
        B = len(batch["text"])
        shard = parallel.current_shard(B)
        local, glob, cond_l = (batch, None, None) if shard is None else self._shard_view(shard, batch, 1)
        wave = self._style_transfer_local(local, ddim_steps, t_enc, unconditional_guidance_scale,
                                          unconditional_conditioning, glob, cond_l)
        return self._egress(parallel.all_gather_rows(wave, B))

    def _style_transfer_local(self, batch, ddim_steps, t_enc, guidance, uncond, glob, cond_rows=None):
        B = len(batch["text"])
        eng = self.engine(B, with_encoder=True)
        x0, noise, noise_fn = self._encode_front(batch, 1, glob, eng, True)
        clip_flag = parallel.latent_guard_flag(x0)           # decided on the device: no synchronisation before the UNet
        cond = cond_rows() if cond_rows is not None else self.conditioning(batch)
        if guidance != 1.0:
            uncond = self.unconditioning(B, uncond)
        return eng.style_transfer_waveform(x0, cond, uncond, t_enc, ddim_steps=ddim_steps, guidance=guidance,
                                           clip_flag=clip_flag, noise=noise, noise_fn=noise_fn)


def build_model(ckpt_path=None, config=None, device=None, model_name="audioldm2-full", *, synthetic: Optional[bool] = None,
                cond_provider=None, ranker: Optional[Callable] = None, t5_len: int = 32, ctx_max_len=None, seqgen_index: int = 0,
                t5_index: Optional[int] = None, clap_tokenize: Optional[Callable] = None, **engine_kw):
    """pipeline.py:142-179.  ``ckpt_path`` is a reference ``<model_name>.pth`` (``["state_dict"]``, key layout of SURVEY.md
    8b); without it (no network here, utils.py:209-219) the seeded synthetic checkpoint is used.  For audioldm2-full / -large
    the AudioMAE generator's weights are taken too (``cond_stage_models.<seqgen_index>.``), for encoder-level providers.  Engines are planned lazily
    for the latent batch of each call (``batchsize * n_candidate_gen_per_text``).

    The Flan-T5 weights, for token-level providers: audioldm2-full / -large encode the conditional branch with the
    generator's inner T5 (``cond_stage_models.<seqgen_index>.cond_stage_models.<t5_index>.model.``, t5_index 1 by default:
    get_input skips a key an earlier model already produced, ddpm.py:861-862) and T5("") with the top-level copy
    (``cond_stage_models.<t5_index>.model.``, ddpm.py:1529-1533); the *_t5 models use ``cond_stage_models.<t5_index>``
    (default 0) for both.  The CLAP text weights, for token-level ``film_clap_cond1``: the generator's first inner model
    (``cond_stage_models.<seqgen_index>.cond_stage_models.0.model.``) for audioldm2-full / -large,
    ``cond_stage_models.0.model.`` for audioldm_48k.  Synthetic weights are generated on first token-level use.
    ``clap_tokenize`` (keyword only; the RoBERTa tokenizer, ``texts -> (ids, mask)``): rank the candidates of
    n_candidate_gen_per_text > 1 natively with the reference's ``clap.model.*`` (its HTSAT audio branch and its text
    branch; synthetic weights made on first use without a checkpoint).  It excludes ``ranker``."""
    if ranker is not None and clap_tokenize is not None:
        raise ValueError("pass either a ranker or clap_tokenize (the native CLAP ranker), not both")
    if device is None or device == "auto":
        device = torch.device("cuda:0")          # the native path has no CPU / MPS fallback
    cfg = arch.model_config(model_name) if config is None else config
    if isinstance(cfg, str):
        raise NotImplementedError("YAML configs are read by the reference's conditioning stack, which is out of scope; "
                                  "pass a dict from arch.model_config")
    if ckpt_path is None:
        if synthetic is False:
            raise RuntimeError("no checkpoint given and hub download is unavailable offline (utils.py:209-219)")
        un, vae, voc, sf = synth.unet_state_dict(cfg["unet"]), synth.vae_state_dict(cfg["vae"]), \
            synth.vocoder_state_dict(cfg["vocoder"]), 1.0
        seq = synth.seqgen_state_dict() if arch.has_seqgen(cfg) else None
        t5c = synth.t5_state_dict if arch.has_t5(cfg) else None
        t5u = None
        clap = synth.clap_text_state_dict if arch.has_clap(cfg) else None
        rank = (synth.clap_audio_state_dict, synth.clap_text_state_dict)
        if ctx_max_len is None:
            n_cross = len([c for c in cfg["unet"]["context_dim"] if c is not None])
            ctx_max_len = (8, t5_len) if n_cross > 1 else (t5_len,)
    else:
        sd = torch.load(ckpt_path, map_location="cpu")["state_dict"]                      # pipeline.py:172
        un, vae, voc, sf = model.split_state_dict(sd)
        seq = model.split_seqgen_state_dict(sd, seqgen_index) if arch.has_seqgen(cfg) else None
        t5c = t5u = None
        if arch.has_seqgen(cfg):
            j = 1 if t5_index is None else t5_index
            t5c = model.split_t5_state_dict(sd, f"cond_stage_models.{seqgen_index}.cond_stage_models.{j}.model.")
            t5u = model.split_t5_state_dict(sd, f"cond_stage_models.{j}.model.")
        elif arch.has_t5(cfg):
            t5c = model.split_t5_state_dict(sd, f"cond_stage_models.{t5_index or 0}.model.")
        clap = None
        if arch.has_seqgen(cfg):
            clap = model.split_clap_text_state_dict(sd, f"cond_stage_models.{seqgen_index}.cond_stage_models.0.model.")
        elif arch.has_clap(cfg):
            clap = model.split_clap_text_state_dict(sd, "cond_stage_models.0.model.")
        rank = None
        if clap_tokenize is not None:
            rank = (model.split_clap_audio_state_dict(sd, "clap.model."), model.split_clap_text_state_dict(sd, "clap.model."))
    ld = NativeAudioLDM2(cfg, un, vae, voc, device, scale_factor=sf, ctx_max_len=ctx_max_len, seqgen_sd=seq,
                         t5_sd=t5c, t5_uncond_sd=t5u, clap_sd=clap, clap_rank_sd=rank if clap_tokenize is not None else None,
                         clap_tokenize=clap_tokenize,
                         cond_provider=cond_provider or SyntheticConditioning(cfg, t5_len=t5_len, device=device), ranker=ranker,
                         **engine_kw)
    ld.model_name = model_name
    return ld


def make_batch_for_text_to_audio(text, transcription="", waveform=None, fbank=None, batchsize=1):
    """pipeline.py:84-124 restricted to the keys the hot path reads (the phoneme / kaldi-fbank entries feed the
    conditioning encoders).  ``text`` may also be a list of ``batchsize`` prompts."""
    text = [text] * batchsize if isinstance(text, str) else list(text)
    assert len(text) == batchsize, "a prompt list must have batchsize entries"
    if fbank is None:
        fbank = torch.zeros((batchsize, 1024, 64))          # not used (pipeline.py:93-96)
    else:
        fbank = torch.as_tensor(fbank, dtype=torch.float32)
        fbank = fbank.expand(batchsize, *fbank.shape[1:])
    if waveform is None:
        waveform = torch.zeros((batchsize, 160000))         # not used
    else:
        waveform = torch.as_tensor(waveform, dtype=torch.float32).expand(batchsize, -1)
    return {"text": text, "fname": [t.replace(" ", "_").replace("'", "_").replace('"', "_") for t in text],
            "waveform": waveform, "log_mel_spec": fbank, "transcription": [transcription] * batchsize}


def text_to_audio(latent_diffusion, text, transcription="", seed=42, ddim_steps=200, duration=10, batchsize=1,
                  guidance_scale=3.5, n_candidate_gen_per_text=3, latent_t_per_second=25.6, config=None, *, use_plms=False):
    """pipeline.py:181-211 -> np.ndarray [batchsize, 1, samples] float32 in (-1, 1).  ``use_plms`` (keyword only) samples
    with PLMS, as generate_batch(use_plms=True) does: ``ddim_steps`` PLMS steps cost ``ddim_steps`` + 1 UNet pairs."""
    seed_everything(int(seed))
    batch = make_batch_for_text_to_audio(text, transcription=transcription, waveform=None, batchsize=batchsize)
    latent_diffusion.latent_t_size = int(duration * latent_t_per_second)
    with torch.no_grad():
        waveform = latent_diffusion.generate_batch(batch, unconditional_guidance_scale=guidance_scale, ddim_steps=ddim_steps,
                                                   n_gen=n_candidate_gen_per_text, duration=duration, use_plms=use_plms)
    return waveform


def wav_to_fbank(latent_diffusion, original_audio_file_path=None, target_length=1024, waveform=None, sr=None):
    """tools.py:86-104 with the native front end: file / array -> read_wav_file's normalisation (tools.py:28-40) ->
    clip(-1, 1) -> aldm_stft_mel (K9) -> fbank [target_length, n_mels] (cropped like _pad_spec, tools.py:71-84)."""
    cfg = latent_diffusion.cfg
    vc = cfg["vocoder"]
    if waveform is None:
        waveform, sr = frontend.read_wav(original_audio_file_path)
    x = frontend.prepare_waveform(np.asarray(waveform, dtype=np.float32).reshape(-1), sr or vc["sampling_rate"],
                                  vc["sampling_rate"], target_length * vc["hop_size"])
    dev = latent_diffusion.device
    wav = torch.clip(torch.from_numpy(x), -1, 1).to(dev).contiguous()                      # get_mel_from_wav (tools.py:43-46)
    fb = engine.stft_mel(wav, vc["n_fft"], vc["hop_size"], frontend.mel_basis_for(cfg).to(dev), out_frames=target_length)[0]
    if fb.shape[-1] % 2 != 0:
        fb = fb[..., :-1]
    return fb, x


def super_resolution_and_inpainting(latent_diffusion, text, transcription="", original_audio_file_path=None, seed=42,
                                    ddim_steps=200, duration=None, batchsize=1, guidance_scale=2.5, n_candidate_gen_per_text=3,
                                    time_mask_ratio_start_and_end=(0.40, 0.6), freq_mask_ratio_start_and_end=(1.0, 1.0),
                                    latent_t_per_second=25.6, config=None, *, waveform=None, waveform_sr=None, use_plms=False):
    """pipeline.py:213-267: STFT/mel front end (K9) -> VAE encoder -> masked DDIM -> decode -> vocoder.  ``waveform`` (+
    ``waveform_sr``) replaces the file read for callers that already hold the samples; ``use_plms`` samples with masked
    PLMS instead (generate_batch_masked(use_plms=True))."""
    seed_everything(int(seed))
    if duration is None:
        duration = latent_diffusion.cfg["latent"][1] / latent_diffusion.cfg["latent_t_per_second"] if waveform is None \
            else len(np.reshape(waveform, -1)) / float(waveform_sr or latent_diffusion.cfg["sampling_rate"])
    frames_per_s = latent_diffusion.cfg["sampling_rate"] / latent_diffusion.cfg["vocoder"]["hop_size"]     # 102.4 at 16 kHz
    mel, _ = wav_to_fbank(latent_diffusion, original_audio_file_path, target_length=int(duration * frames_per_s),
                          waveform=waveform, sr=waveform_sr)
    batch = make_batch_for_text_to_audio(text, transcription=transcription, fbank=mel[None, ...], batchsize=batchsize)
    ds = 2 ** (len(latent_diffusion.cfg["vae"]["ch_mult"]) - 1)
    latent_diffusion.latent_t_size = mel.shape[0] // ds
    with torch.no_grad():
        waveform_out = latent_diffusion.generate_batch_masked(
            batch, unconditional_guidance_scale=guidance_scale, ddim_steps=ddim_steps, n_gen=n_candidate_gen_per_text,
            duration=duration, time_mask_ratio_start_and_end=time_mask_ratio_start_and_end,
            freq_mask_ratio_start_and_end=freq_mask_ratio_start_and_end, use_plms=use_plms)
    return waveform_out


def round_up_duration(duration):
    """pipeline.py:124-125: the duration, in steps of 2.5 s, that a recording of ``duration`` seconds is generated at."""
    return int(round(duration / 2.5) + 1) * 2.5


def style_transfer_sizes(cfg: dict, duration: float):
    """(latent frames, mel frames) of style transfer at ``duration`` s: int(duration * latent_t_per_second), times the
    VAE's 2 ** (len(ch_mult) - 1) -- 1024 mel frames at 10 s for both 16 kHz and 48 kHz, AudioLDM 1's int(duration *
    102.4) at 16 kHz.  ValueError unless the latent length is a multiple of 8 (the UNet's three stride-2 levels)."""
    latent_t = int(duration * cfg["latent_t_per_second"])
    if latent_t % 8 != 0:
        raise ValueError(f"duration {duration} s gives {latent_t} latent frames; the UNet needs a multiple of 8 "
                         f"(durations in steps of {8 / cfg['latent_t_per_second']:g} s)")
    return latent_t, latent_t * 2 ** (len(cfg["vae"]["ch_mult"]) - 1)


def style_transfer(latent_diffusion, text, original_audio_file_path, transfer_strength, seed=42, duration=10, batchsize=1,
                   guidance_scale=2.5, ddim_steps=200, config=None, *, waveform=None, waveform_sr=None):
    """Audio-to-audio style transfer, AudioLDM 1's ``style_transfer`` on this engine: the recording's mel is encoded to
    its latent, noised to DDIM index t_enc = int(transfer_strength * ddim_steps) and denoised over t_enc steps under
    ``text`` (a prompt, or a list of ``batchsize`` prompts) -> np.ndarray [batchsize, 1, samples] float32.  A duration
    longer than the recording becomes round_up_duration(its length).  ``waveform`` (+ ``waveform_sr``, keyword only)
    replaces the file read.  ``config`` is accepted and unused, as in super_resolution_and_inpainting.  ValueError
    before any draw when t_enc is outside [0, schedule length) or the latent length is not a multiple of 8."""
    cfg = latent_diffusion.cfg
    if waveform is None:
        waveform, waveform_sr = frontend.read_wav(original_audio_file_path)
    audio_duration = len(np.reshape(waveform, -1)) / float(waveform_sr or cfg["sampling_rate"])
    if duration > audio_duration:
        duration = round_up_duration(audio_duration)
    seed_everything(int(seed))
    latent_t, mel_frames = style_transfer_sizes(cfg, duration)
    sampler_mod.transfer_steps(transfer_strength, ddim_steps, cfg["timesteps"])
    mel, _ = wav_to_fbank(latent_diffusion, target_length=mel_frames, waveform=waveform, sr=waveform_sr)
    batch = make_batch_for_text_to_audio(text, fbank=mel[None, ...], batchsize=batchsize)
    latent_diffusion.latent_t_size = latent_t
    with torch.no_grad():
        return latent_diffusion.generate_batch_style_transfer(batch, transfer_strength, ddim_steps=ddim_steps,
                                                              unconditional_guidance_scale=guidance_scale)
