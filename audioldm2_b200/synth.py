"""Seeded synthetic checkpoints with the reference ``state_dict`` layout.

Hub checkpoints cannot be assumed reachable (no network), so they are not fetched
(utils.py:209-219).  Parity and throughput are therefore measured on deterministic
random weights that have exactly the key names / shapes of the reference modules
(SURVEY.md 8b/8d).  Rules (SURVEY.md 8d "synthetic inputs"):

* conv / linear weights ~ N(0, gain/sqrt(fan_in)) -- *including* the ones the reference
  zero-initialises with ``zero_module`` (openaimodel.py:255-257,810; attention.py:452-454),
  otherwise half of the graph would be multiplied by zero and left untested;
* biases and norm beta ~ 0.02 N(0,1); norm gamma ~ 1 + 0.1 N(0,1).

Tensors are generated one by one from a CPU ``torch.Generator`` in sorted-key order, so
the same (config, seed) gives bit-identical weights on every machine with this torch.
"""
from __future__ import annotations

import math
from typing import Dict, Tuple

import torch

from . import arch


def _fill(shapes: Dict[str, Tuple[int, ...]], seed: int, gain: float = 1.0) -> Dict[str, torch.Tensor]:
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    out = {}
    for name in sorted(shapes):
        shp = shapes[name]
        if name.endswith(".bias"):
            t = 0.02 * torch.randn(shp, generator=g)
        elif len(shp) == 1:                      # norm gamma
            t = 1.0 + 0.1 * torch.randn(shp, generator=g)
        else:
            fan_in = 1
            for d in shp[1:]:
                fan_in *= d
            t = torch.randn(shp, generator=g) * (gain / math.sqrt(fan_in))
        out[name] = t.contiguous()
    return out


def unet_state_dict(cfg: dict, seed: int = 1234) -> Dict[str, torch.Tensor]:
    return _fill(arch.unet_param_shapes(cfg), seed)


def vae_state_dict(cfg: dict, seed: int = 1235) -> Dict[str, torch.Tensor]:
    return _fill(arch.vae_param_shapes(cfg), seed)


def vocoder_state_dict(cfg: dict, seed: int = 1236) -> Dict[str, torch.Tensor]:
    sd = _fill(arch.vocoder_param_shapes(cfg), seed)
    # Keep activations O(1) through five upsampling stages and 15-20 residual blocks so the
    # final tanh is not saturated (SURVEY.md 7 H2; the reference init N(0, 0.01) at
    # hifigan/models.py:10-13 gives vanishing outputs instead).
    for name in sd:
        w = sd[name]
        if name.startswith("ups.") and name.endswith(".weight"):
            # ConvTranspose1d weight is [Cin, Cout, k]; an output sample sees Cin*k/u taps.
            i = int(name.split(".")[1])
            u = cfg["upsample_rates"][i]
            cin, cout, k = w.shape
            sd[name] = (w * math.sqrt(cout * u / cin)).contiguous()
        elif name.startswith("resblocks.") and name.endswith(".weight"):
            sd[name] = (w * 0.7).contiguous()
        elif name == "conv_post.weight":
            sd[name] = (w * 0.5).contiguous()
    return sd


def seqgen_state_dict(seed: int = 1237, n_layer: int = 12) -> Dict[str, torch.Tensor]:
    """Seeded AudioMAE-generator checkpoint (keys relative to ``cond_stage_models.<i>.``).  Not ``_fill``: GPT-2's
    ``Conv1D`` weights are [in, out], so their fan-in is ``shape[0]``; ``wpe`` / ``wte`` are 0.02 N(0, 1) (GPT-2's
    embedding init) and the SOS / EOS tables N(0, 1) (the ``nn.Embedding`` default).  Everything else as SURVEY.md 8d."""
    shapes = arch.seqgen_param_shapes(n_layer)
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    out = {}
    for name in sorted(shapes):
        shp = shapes[name]
        t = torch.randn(shp, generator=g)
        if name in ("model.wpe.weight", "model.wte.weight"):
            t = 0.02 * t
        elif name.endswith("_of_sequence_tokens.weight"):
            pass
        elif name.endswith(".bias"):
            t = 0.02 * t
        elif len(shp) == 1:
            t = 1.0 + 0.1 * t
        elif name.startswith("model."):                 # Conv1D [in, out]
            t = t / math.sqrt(shp[0])
        else:                                           # nn.Linear [out, in]
            t = t / math.sqrt(shp[1])
        out[name] = t.contiguous()
    return out


def t5_state_dict(seed: int = 1238, n_layer: int = 24) -> Dict[str, torch.Tensor]:
    """Seeded Flan-T5 encoder checkpoint (HF ``T5EncoderModel`` keys, arch.t5_param_shapes).  Not ``_fill``: the gains
    follow HF's T5 initialisation so that the unscaled logits stay O(1) -- q ~ N(0, 1/(1024 * 64)), k / v ~ N(0, 1/1024)
    -- and the two residual projections (o, wo) are scaled by 1/sqrt(2 n_layer) so that the residual stream stays O(1)
    over all blocks; the embedding and the relative-position bias are N(0, 1), RMSNorm weights 1 + 0.1 N(0, 1).
    ``encoder.embed_tokens.weight`` is ``shared.weight`` (tied), as in the module's state dict."""
    C, Dk = arch.T5["d_model"], arch.T5["d_kv"]
    shapes = arch.t5_param_shapes(n_layer, with_embed_tokens=False)
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    res = 1.0 / math.sqrt(2 * n_layer)
    out = {}
    for name in sorted(shapes):
        shp = shapes[name]
        t = torch.randn(shp, generator=g)
        if name == "shared.weight" or name.endswith("relative_attention_bias.weight"):
            pass
        elif len(shp) == 1:
            t = 1.0 + 0.1 * t
        elif name.endswith(".q.weight"):
            t = t / math.sqrt(C * Dk)
        elif name.endswith((".o.weight", ".wo.weight")):
            t = t * (res / math.sqrt(shp[1]))
        else:
            t = t / math.sqrt(shp[1])
        out[name] = t.contiguous()
    out["encoder.embed_tokens.weight"] = out["shared.weight"]
    return out


def token_ids(lens, seed: int = 79, device="cpu"):
    """Seeded tokenizer output: ids [B, L] int64 and attention_mask [B, L] float, L = max(lens) (padding=True).  Row i
    holds lens[i] - 1 ids drawn from [2, vocab), then EOS (1), then pad (0) -- the layout of a T5 tokenization."""
    g = torch.Generator(device="cpu"); g.manual_seed(seed)
    lens = [int(n) for n in lens]
    assert min(lens) >= 1 and max(lens) <= arch.T5["max_len"]
    L = max(lens)
    ids = torch.randint(2, arch.T5["vocab"], (len(lens), L), generator=g)
    mask = (torch.arange(L)[None, :] < torch.tensor(lens)[:, None])
    ids[torch.arange(len(lens)), torch.tensor(lens) - 1] = arch.T5["eos_id"]
    ids = torch.where(mask, ids, torch.full_like(ids, arch.T5["pad_id"]))
    return ids.to(device), mask.float().to(device)


def clap_text_state_dict(seed: int = 1239, n_layer: int = 12) -> Dict[str, torch.Tensor]:
    """Seeded CLAP text branch (HF ``RobertaModel`` keys under ``text_branch.`` plus ``text_projection``,
    arch.clap_text_param_shapes).  Not ``_fill``: every matrix is N(0, 1 / fan_in), so that each projection of a LayerNorm
    output is O(1) -- logits q.k / 8 of a few units, pooler pre-activations O(1) so that tanh is exercised on its
    nonlinear part; biases and LayerNorm offsets 0.1 N(0, 1), LayerNorm weights 1 + 0.1 N(0, 1), embeddings N(0, 1)."""
    shapes = arch.clap_text_param_shapes(n_layer)
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    out = {}
    for name in sorted(shapes):
        shp = shapes[name]
        t = torch.randn(shp, generator=g)
        if "embeddings." in name and len(shp) == 2:
            pass
        elif name.endswith("LayerNorm.weight"):
            t = 1.0 + 0.1 * t
        elif len(shp) == 1:
            t = 0.1 * t
        else:
            t = t / math.sqrt(shp[1])
        out[name] = t.contiguous()
    return out


def clap_token_ids(lens, L: int = 512, seed: int = 80, device="cpu"):
    """Seeded RoBERTa tokenizer output as the reference pads it (padding="max_length"): ids [B, L] int64 and
    attention_mask [B, L] float.  Row i holds lens[i] tokens -- BOS (0), lens[i] - 2 ids drawn from [3, vocab), EOS (2) --
    then pad (1)."""
    g = torch.Generator(device="cpu"); g.manual_seed(seed)
    lens = [int(n) for n in lens]
    assert min(lens) >= 2 and max(lens) <= L <= arch.CLAP_TEXT["max_len"]
    ids = torch.randint(3, arch.CLAP_TEXT["vocab"], (len(lens), L), generator=g)
    n = torch.tensor(lens)[:, None]
    pos = torch.arange(L)[None, :]
    ids[:, 0] = arch.CLAP_TEXT["bos_id"]
    ids = torch.where(pos == n - 1, torch.full_like(ids, arch.CLAP_TEXT["eos_id"]), ids)
    ids = torch.where(pos < n, ids, torch.full_like(ids, arch.CLAP_TEXT["pad_id"]))
    return ids.to(device), (pos < n).float().to(device)


def encoder_outputs(batch: int, t5_lens, seed: int = 78, device="cpu"):
    """Synthetic encoder outputs for the sequence-generation models (SURVEY.md 8d): CLAP [B, 1, 512] L2-normalised (as
    the CLAP embedding is), Flan-T5 hidden states [B, L, 1024] N(0, 1) with L = max(t5_lens) and the padding mask of
    per-row lengths ``t5_lens`` (zeros behind each row's length, as the tokenizer's padding=True gives)."""
    g = torch.Generator(device="cpu"); g.manual_seed(seed)
    lens = [int(n) for n in t5_lens]
    assert len(lens) == batch and min(lens) >= 1
    L = max(lens)
    clap = torch.randn(batch, 1, 512, generator=g)
    clap = clap / clap.norm(dim=-1, keepdim=True)
    t5 = torch.randn(batch, L, 1024, generator=g)
    mask = (torch.arange(L)[None, :] < torch.tensor(lens)[:, None]).float()
    return clap.to(device), t5.to(device), mask.to(device)


def conditioning(cfg: dict, batch: int, seed: int = 77, t5_len: int = 32, device="cpu"):
    """Synthetic conditioning at the UNet boundary (SURVEY.md 8d).

    Returns (cond, uncond), each a dict with ``context_list`` / ``mask_list`` (lists of
    [B, L, D] / [B, L] float tensors) and ``y`` ([B, film_dim] or None), i.e. the keyword
    arguments of ``UNetModel.forward`` (openaimodel.py:837-845).
    """
    g = torch.Generator(device="cpu"); g.manual_seed(seed)
    ucfg = cfg["unet"]
    dims = [c for c in ucfg["context_dim"] if c is not None]
    cond = dict(context_list=[], mask_list=[], y=None)
    unc = dict(context_list=[], mask_list=[], y=None)
    for i, d in enumerate(dims):
        L = 8 if i == 0 and len(dims) > 1 else t5_len
        c = torch.randn(batch, L, d, generator=g)
        cond["context_list"].append(c.to(device)); cond["mask_list"].append(torch.ones(batch, L).to(device))
        if i == 0 and len(dims) > 1:        # AudioMAE tokens: uncond = zeros (encoders/modules.py:476-479)
            unc["context_list"].append(torch.zeros(batch, L, d).to(device))
            unc["mask_list"].append(torch.ones(batch, L).to(device))
        else:                               # T5(""): one token
            u = torch.randn(1, 1, d, generator=g).expand(batch, 1, d).contiguous()
            unc["context_list"].append(u.to(device)); unc["mask_list"].append(torch.ones(batch, 1).to(device))
    fd = ucfg.get("extra_film_condition_dim")
    if fd is not None:
        y = torch.randn(batch, fd, generator=g); y = y / y.norm(dim=-1, keepdim=True)
        cond["y"] = y.to(device)
        unc["y"] = torch.zeros(batch, fd).to(device)
    return cond, unc


def clap_audio_state_dict(seed: int = 1240, depths=(2, 2, 12, 2)) -> Dict[str, torch.Tensor]:
    """Seeded CLAP audio branch (``audio_branch.`` + ``audio_projection``, arch.clap_audio_param_shapes).  torchlibrosa's
    fixed tensors are made exactly: the STFT weights are the periodic-Hann DFT basis (model.htsat_dft_basis) and melW the
    Slaney mel filterbank of 48 kHz / 1024 / 64 bins / 50 Hz - 14 kHz.  bn0's running statistics (mean -15 dB, std 15 dB)
    bring the log-mel of vocoder-like audio (|x| ~ 0.1) to O(1).  Matrices are N(0, 1 / fan_in), with the residual branch
    outputs (attn.proj, mlp.fc2) at half that gain so that the pre-LN residual stream stays O(1) over 18 blocks; the
    relative-position tables 0.5 N(0, 1) (a visible bias next to logits of a few units); biases and LayerNorm offsets
    0.1 N(0, 1), LayerNorm and bn0 weights 1 + 0.1 N(0, 1)."""
    from . import frontend, model
    shapes = arch.clap_audio_param_shapes(tuple(depths))
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    out = {}
    for name in sorted(shapes):
        shp = shapes[name]
        t = torch.randn(shp, generator=g)
        if "spectrogram_extractor" in name or "logmel_extractor" in name:
            continue
        if name.endswith("running_mean"):
            t = -15.0 + 0.5 * t
        elif name.endswith("running_var"):
            t = 225.0 * (1.0 + 0.05 * t.abs())
        elif name.endswith("relative_position_bias_table"):
            t = 0.5 * t
        elif name.endswith(("norm.weight", "norm1.weight", "norm2.weight", "bn0.weight")):
            t = 1.0 + 0.1 * t
        elif len(shp) == 1:
            t = 0.1 * t
        else:
            fan_in = math.prod(shp[1:])
            t = t / math.sqrt(fan_in) * (0.5 if name.endswith(("attn.proj.weight", "mlp.fc2.weight")) else 1.0)
        out[name] = t.contiguous()
    real, imag = model.htsat_dft_basis(arch.CLAP_AUDIO["n_fft"])
    out["audio_branch.spectrogram_extractor.stft.conv_real.weight"] = real.float()
    out["audio_branch.spectrogram_extractor.stft.conv_imag.weight"] = imag.float()
    A = arch.CLAP_AUDIO
    out["audio_branch.logmel_extractor.melW"] = frontend.mel_basis(A["sample_rate"], A["n_fft"], A["n_mels"], A["fmin"],
                                                                   A["fmax"]).t().contiguous()
    return out


def clap_tokenize(texts, seed: int = 82, L: int = 512):
    """A seeded stand-in for the RoBERTa tokenizer (padding="max_length", max_length 512): each text maps
    deterministically (crc32 of its UTF-8 bytes and the seed, not Python's salted hash) to BOS, 1 .. 30 ids from
    [3, vocab), EOS, then pad; "" gives [BOS, EOS] as the real tokenizer does.  -> (ids [n, L] int64, mask [n, L] float)."""
    import zlib
    A = arch.CLAP_TEXT
    ids = torch.full((len(texts), L), A["pad_id"], dtype=torch.int64)
    mask = torch.zeros(len(texts), L)
    for i, t in enumerate(texts):
        h = zlib.crc32(t.encode("utf-8")) ^ (seed * 0x9E3779B1 & 0xFFFFFFFF)
        g = torch.Generator().manual_seed(h)
        n = 0 if t == "" else 1 + int(torch.randint(30, (1,), generator=g))
        row = [A["bos_id"]] + torch.randint(3, A["vocab"], (n,), generator=g).tolist() + [A["eos_id"]]
        ids[i, :len(row)] = torch.tensor(row)
        mask[i, :len(row)] = 1
    return ids, mask
