"""NativeCLAPTextEncoder: the CLAP text embedding, run natively from token ids.

``embed(ids, mask)`` returns what ``CLAP.get_text_embedding`` returns (clap/open_clip/model.py:656-663, 730-750) for the
RoBERTa text branch: the L2-normalised ``text_projection`` of the pooler output, [B, 512] float32.  The tokenizer (a BPE
hub asset) stays with the caller, which passes its ids and attention mask as the reference's tokenizer gives them
(padding="max_length": L = 512, pad id 1).  ``unconditional()`` is CLAP(""), the reference's ``unconditional_token``
(encoders/modules.py:655-658): "" tokenizes to [0, 2]; computed once and cached.

The sequence is cut at L_eff = 1 + the last position any row's mask holds a token at, before planning.  That is exact
up to rounding: the embedding reads token 0 of the last layer only, padded keys get probability exactly 0 in every layer,
and the position id of a valid token depends only on the ids before it.  A prompt of 10-40 tokens so costs a twentieth
of the 512 positions the reference encodes.  L_eff is the one value read on the host, from the mask, before the run.

Every kernel is sm_90a code of this package (plan.build_clap_text: embedding, its LayerNorm, 12 blocks of 8 launches, the
head), one op table per (B, L_eff) replayed as a CUDA graph; plans are built lazily and the two most recent are kept,
all sharing one uploaded weight arena.  Nothing is read back after a run: pack_clap_weights has already ruled out values
beyond the fp16 range of the operand planes from the weights.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Dict, Optional

import torch

from . import arch, engine, plan


def check_tokens(ids: torch.Tensor, mask: torch.Tensor):
    """Raise ValueError unless ids [B, L] are integers in [0, vocab), mask [B, L] holds only 0 / 1 with at least one 1 per
    row, and 1 <= L <= 512 (the tokenizer's max_length)."""
    V, Lmax = arch.CLAP_TEXT["vocab"], arch.CLAP_TEXT["max_len"]
    if ids.dim() != 2 or ids.dtype.is_floating_point or ids.dtype.is_complex or ids.dtype == torch.bool:
        raise ValueError(f"token ids must be an integer tensor [B, L], got {ids.dtype} {tuple(ids.shape)}")
    if tuple(mask.shape) != tuple(ids.shape):
        raise ValueError(f"attention mask {tuple(mask.shape)} does not match the ids {tuple(ids.shape)}")
    B, L = ids.shape
    if B < 1 or not 1 <= L <= Lmax:
        raise ValueError(f"token ids [B={B}, L={L}]: need B >= 1 and 1 <= L <= {Lmax}")
    if bool(((ids < 0) | (ids >= V)).any()):
        raise ValueError(f"token ids outside [0, {V})")
    m = mask.float()
    if bool(((m != 0) & (m != 1)).any()):
        raise ValueError("attention mask values must be 0 or 1")
    if bool((m.sum(1) < 1).any()):
        raise ValueError("every row of the attention mask needs at least one token")


def effective_length(mask: torch.Tensor) -> int:
    """1 + the last index at which any row's mask is 1."""
    cols = (mask.float() == 1).any(0).nonzero()
    return int(cols[-1]) + 1


def empty_prompt(n: int = 1, L: int = 512, device="cpu"):
    """The tokenization of "" on n rows, padded to L as the reference's tokenizer pads: ids [0, 2, 1, 1, ...], mask
    [1, 1, 0, ...]."""
    A = arch.CLAP_TEXT
    ids = torch.full((n, L), A["pad_id"], dtype=torch.int64, device=device)
    ids[:, 0], ids[:, 1] = A["bos_id"], A["eos_id"]
    mask = torch.zeros(n, L, device=device)
    mask[:, :2] = 1
    return ids, mask


def is_empty_prompt(ids: torch.Tensor, mask: torch.Tensor) -> bool:
    """Every row is the tokenization of "" (any padding length)."""
    if ids.dim() != 2 or ids.shape[1] < 2:
        return False
    e_ids, e_mask = empty_prompt(ids.shape[0], ids.shape[1], ids.device)
    m = mask.to(ids.device).float()
    return bool(torch.equal(m, e_mask)) and bool(((ids == e_ids) | (m == 0)).all())


class NativeCLAPTextEncoder:
    def __init__(self, state_dict: Optional[Dict[str, torch.Tensor]] = None, device="cuda:0", use_graph: bool = True,
                 max_plans: int = 2, weights: Optional[plan.ClapWeights] = None):
        """``state_dict``: the text branch's keys (model.split_clap_text_state_dict or synth.clap_text_state_dict), or
        ``weights``, an already packed arena."""
        if not torch.cuda.is_available():
            raise RuntimeError("the native CLAP text encoder needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device(device)
        self.use_graph = use_graph
        self.max_plans = max_plans
        self.weights = weights if weights is not None else plan.pack_clap_weights(state_dict)
        self.arena = self.weights.arena.to(self.device)
        self._progs: "OrderedDict[tuple, engine.DeviceProgram]" = OrderedDict()
        self._uncond: Optional[torch.Tensor] = None

    def program(self, B: int, L: int) -> engine.DeviceProgram:
        key = (int(B), int(L))
        prog = self._progs.get(key)
        if prog is not None:
            self._progs.move_to_end(key)
            return prog
        while len(self._progs) >= self.max_plans:
            self._progs.popitem(last=False)[1].close()
        pl = plan.build_clap_text(None, B, L, weights=self.weights)
        prog = engine.DeviceProgram(pl, self.device, dict(all=(pl.marks["begin"], pl.marks["end"])), arena_dev=self.arena)
        self._progs[key] = prog
        return prog

    @torch.no_grad()
    def embed(self, ids: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
        """ids [B, L] integer, mask [B, L] (1 = token, 0 = padding) -> the text embedding [B, 512] float32 on the device."""
        check_tokens(ids, mask)
        L = effective_length(mask)
        ids, mask = ids[:, :L], mask[:, :L]
        prog = self.program(ids.shape[0], L)
        prog.view("ids").copy_(ids.to(torch.int64))
        prog.view("mask").copy_(mask.float())
        if self.use_graph:
            prog.replay("all")
        else:
            prog.run("all")
        return prog.view("embed").clone()

    def unconditional(self) -> torch.Tensor:
        """CLAP("") -> [1, 512], computed once and cached."""
        if self._uncond is None:
            self._uncond = self.embed(*empty_prompt(1, 2, self.device))
        return self._uncond


class NativeCLAPAudioEncoder:
    """The CLAP audio embedding, run natively from the waveform: ``embed(waveform [n, L])`` returns what the reference's
    CLAPAudioEmbeddingClassifierFreev2 computes in audio mode before its random replacement (encoders/modules.py:689-716):
    torchaudio's resample to 48 kHz unless ``sampling_rate`` is 48 000, the truncation to 480 000 samples, then
    CLAP.get_audio_embedding with the HTSAT-base branch -- [n, 512] float32 on the device, L2-normalised.

    Every kernel is sm_90a code of this package (plan.build_clap_audio: the log-mel front end, the patch embedding, 18 Swin
    blocks, 3 PatchMergings and the head), one op table per (n, L, sampling rate) replayed as a CUDA graph; plans are built
    lazily and the two most recent are kept, sharing one uploaded weight arena.  Nothing is read back after a run:
    pack_clap_audio_weights has already ruled out values beyond the fp16 range of the operand planes from the weights."""

    def __init__(self, state_dict: Optional[Dict[str, torch.Tensor]] = None, device="cuda:0", sampling_rate: int = 16000,
                 use_graph: bool = True, max_plans: int = 2, weights: Optional[plan.ClapAudioWeights] = None):
        if not torch.cuda.is_available():
            raise RuntimeError("the native CLAP audio encoder needs a CUDA device (sm_90a); there is no CPU fallback")
        if int(sampling_rate) not in (16000, 48000):
            raise ValueError(f"CLAP audio encoder: sampling rate {sampling_rate} (16000 or 48000)")
        self.device = torch.device(device)
        self.sampling_rate = int(sampling_rate)
        self.use_graph = use_graph
        self.max_plans = max_plans
        self.weights = weights if weights is not None else plan.pack_clap_audio_weights(state_dict)
        self.arena = self.weights.arena.to(self.device)
        self._progs: "OrderedDict[tuple, engine.DeviceProgram]" = OrderedDict()

    def check(self, waveform: torch.Tensor):
        """Raise ValueError unless waveform is a float32 [n, L] tensor whose 48 kHz signal is longer than 512 samples
        (reflect padding of the first frame)."""
        if waveform.dim() != 2 or waveform.dtype != torch.float32:
            raise ValueError(f"waveform must be a float32 tensor [n, L], got {waveform.dtype} {tuple(waveform.shape)}")
        n, L = waveform.shape
        L48 = min(L * (48000 // self.sampling_rate), arch.CLAP_AUDIO["max_samples"])
        if n < 1 or L48 <= arch.CLAP_AUDIO["n_fft"] // 2:
            raise ValueError(f"waveform [n={n}, L={L}] at {self.sampling_rate} Hz: need n >= 1 and more than "
                             f"{arch.CLAP_AUDIO['n_fft'] // 2} samples at 48 kHz")

    def program(self, n: int, L: int) -> engine.DeviceProgram:
        key = (int(n), int(L), self.sampling_rate)
        prog = self._progs.get(key)
        if prog is not None:
            self._progs.move_to_end(key)
            return prog
        while len(self._progs) >= self.max_plans:
            self._progs.popitem(last=False)[1].close()
        pl = plan.build_clap_audio(None, n, L, self.sampling_rate, weights=self.weights)
        prog = engine.DeviceProgram(pl, self.device, dict(all=(pl.marks["begin"], pl.marks["end"])), arena_dev=self.arena)
        self._progs[key] = prog
        return prog

    @torch.no_grad()
    def embed(self, waveform: torch.Tensor) -> torch.Tensor:
        """waveform [n, L] float32 (host or device) -> the audio embedding [n, 512] float32 on the device."""
        self.check(waveform)
        prog = self.program(*waveform.shape)
        prog.view("wav").copy_(waveform)
        if self.use_graph:
            prog.replay("all")
        else:
            prog.run("all")
        return prog.view("embed").clone()


def replacement_draws(n: int) -> list:
    """The draws of CLAPAudioEmbeddingClassifierFreev2.forward after an embedding of n rows (encoders/modules.py:730-733):
    one torch.rand(1) per row in row order; a row is replaced by CLAP("") below unconditional_prob = 0.1.  Used for the
    conditioning rows (pipeline.clap_replacement_draws) and for both halves of the ranker's cos_similarity."""
    return [float(torch.rand(1)) < 0.1 for _ in range(n)]


class NativeCLAPRanker:
    """The reference's re-ranker ``clap.cos_similarity(waveform, text)`` (encoders/modules.py:639-653, ddpm.py:1554-1568),
    natively: ``__call__(waveform [n, L], texts) -> similarity [n]`` on the device, the contract of the pipeline's ``ranker``
    hook.  The audio rows are embedded, then forward's n draws replace rows by CLAP(""); the texts are tokenized by
    ``tokenize(texts) -> (ids, mask)`` (the RoBERTa tokenizer stays with the caller) and embedded, then n more draws; then
    the cosine similarity.  ``rows`` / ``n_total`` rank a subset of a larger call (one rank of a sharded call): all
    2 n_total draws are made, in global row order, and row k of ``waveform`` takes the decisions of global row rows[k]."""

    def __init__(self, audio_encoder: NativeCLAPAudioEncoder, text_encoder: NativeCLAPTextEncoder, tokenize):
        self.audio, self.text, self.tokenize = audio_encoder, text_encoder, tokenize

    @torch.no_grad()
    def __call__(self, waveform: torch.Tensor, texts, rows=None, n_total: Optional[int] = None) -> torch.Tensor:
        n = waveform.shape[0]
        if len(texts) != n:
            raise ValueError(f"{len(texts)} texts for {n} waveforms")
        rows = list(range(n)) if rows is None else [int(r) for r in rows]
        n_total = n if n_total is None else int(n_total)
        u = self.text.unconditional()
        a = self.audio.embed(waveform)
        da = replacement_draws(n_total)
        ra = [k for k, g in enumerate(rows) if da[g]]
        if ra:
            a[ra] = u
        t = self.text.embed(*self.tokenize(list(texts)))
        dt = replacement_draws(n_total)
        rt = [k for k, g in enumerate(rows) if dt[g]]
        if rt:
            t[rt] = u.to(t.device)
        return torch.nn.functional.cosine_similarity(a[:, None], t[:, None], dim=2).reshape(-1)
