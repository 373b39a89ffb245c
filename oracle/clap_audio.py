"""TEST INFRASTRUCTURE -- pure-torch restatement of the CLAP audio embedding and the re-ranker (never imported by the
product path).

``clap_audio_embed`` is what ``CLAPAudioEmbeddingClassifierFreev2.forward`` computes in audio mode before its random
replacement (latent_diffusion/modules/encoders/modules.py:689-716): torchaudio's resample to 48 kHz when the input is not
48 kHz, the truncation of ``get_audio_features`` (clap/training/data.py:421-450, never a padding), then
``CLAP.get_audio_embedding`` (clap/open_clip/model.py:752-777) with the non-fusion HTSAT-base branch
(clap/open_clip/htsat.py): torchlibrosa Spectrogram / LogmelFilterBank from the checkpoint's STFT weights and melW, bn0,
reshape_wav2img (:1074-1101), PatchEmbed, pre-LN Swin blocks with (shifted) window attention (:412-637), PatchMerging
(:639-679), the final norm and the mean over tokens (:1021-1039), audio_projection and F.normalize.  ``cos_similarity``
restates encoders/modules.py:639-653 with forward's replacement draws (:730-733), and ``select`` the ranking of
ddpm.py:1554-1568.  Everything runs in the dtype asked for (float64 for the tests' references, float32 / TF32 on a GPU for
the timing script's baseline).  Pinned to the unmodified reference by tests/golden/make_clap_audio_golden.py.
"""
from __future__ import annotations

import math
from typing import Callable, Dict, List, Tuple

import torch
import torch.nn.functional as F

SD = Dict[str, torch.Tensor]


def resample_16k_to_48k(x: torch.Tensor, lowpass_filter_width: int = 6, rolloff: float = 0.99) -> torch.Tensor:
    """torchaudio.functional.resample(x, 16000, 48000) (sinc_interp_hann): [n, L] -> [n, 3 L].  The kernel is made in
    float32 as torchaudio makes it for a float32 waveform, the convolution runs in x's dtype."""
    orig, new = 1, 3
    base = min(orig, new) * rolloff
    width = math.ceil(lowpass_filter_width * orig / base)
    idx = torch.arange(-width, width + orig, dtype=torch.float32)[None, None] / orig
    t = torch.arange(0, -new, -1, dtype=torch.float32)[:, None, None] / new + idx
    t = (t * base).clamp(-lowpass_filter_width, lowpass_filter_width)
    window = torch.cos(t * math.pi / lowpass_filter_width / 2) ** 2
    t = t * math.pi
    k = torch.where(t == 0, torch.tensor(1.0), t.sin() / t) * window * (base / orig)
    n, L = x.shape
    xp = F.pad(x, (width, width + orig))
    y = F.conv1d(xp[:, None], k.to(x), stride=orig)           # [n, 3, L + 1]
    return y.transpose(1, 2).reshape(n, -1)[:, :new * L]


def relative_position_index(window: int = 8) -> torch.Tensor:
    """WindowAttention.relative_position_index (htsat.py:384-401)."""
    c = torch.stack(torch.meshgrid(torch.arange(window), torch.arange(window), indexing="ij")).flatten(1)
    rel = (c[:, :, None] - c[:, None, :]).permute(1, 2, 0) + (window - 1)
    return rel[..., 0] * (2 * window - 1) + rel[..., 1]


def shift_mask(R: int, window: int, shift: int) -> torch.Tensor:
    """SwinTransformerBlock.attn_mask (htsat.py:545-576): [nW, w^2, w^2] of 0 / -100."""
    img = torch.zeros(1, R, R, 1)
    cnt = 0
    sl = (slice(0, -window), slice(-window, -shift), slice(-shift, None))
    for h in sl:
        for w in sl:
            img[:, h, w, :] = cnt
            cnt += 1
    mw = partition(img, window).reshape(-1, window * window)
    m = mw[:, None, :] - mw[:, :, None]
    return m.masked_fill(m != 0, -100.0).masked_fill(m == 0, 0.0)


def partition(x: torch.Tensor, w: int) -> torch.Tensor:
    B, H, W, C = x.shape
    return x.view(B, H // w, w, W // w, w, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, w, w, C)


def unpartition(x: torch.Tensor, w: int, H: int, W: int) -> torch.Tensor:
    B = x.shape[0] // ((H // w) * (W // w))
    return x.view(B, H // w, W // w, w, w, -1).permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, -1)


def logmel(sd: SD, wav48: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    """torchlibrosa Spectrogram (conv with the checkpoint's STFT weights over reflect-centred frames) -> power ->
    LogmelFilterBank (melW, 10 log10(max(., 1e-10))) -> bn0 (eval).  [n, L48] -> [n, T, 64]."""
    a = "audio_branch"
    xp = F.pad(wav48[:, None], (512, 512), mode="reflect")[:, 0]
    fr = xp.unfold(1, 1024, 480)                                           # [n, T, 1024]
    re = fr @ sd[f"{a}.spectrogram_extractor.stft.conv_real.weight"][:, 0].t()
    im = fr @ sd[f"{a}.spectrogram_extractor.stft.conv_imag.weight"][:, 0].t()
    mel = (re ** 2 + im ** 2) @ sd[f"{a}.logmel_extractor.melW"]
    db = 10.0 * torch.log10(torch.clamp(mel, min=1e-10))
    return (db - sd[f"{a}.bn0.running_mean"]) / torch.sqrt(sd[f"{a}.bn0.running_var"] + eps) * sd[f"{a}.bn0.weight"] \
        + sd[f"{a}.bn0.bias"]


def wav2img(x: torch.Tensor) -> torch.Tensor:
    """reshape_wav2img: [n, T, 64] -> bicubic (align_corners) to [n, 1024, 64] -> the fold to [n, 1, 256, 256]."""
    n = x.shape[0]
    x = F.interpolate(x[:, None], (1024, 64), mode="bicubic", align_corners=True)     # [n, 1, 1024, 64]
    x = x.permute(0, 1, 3, 2).reshape(n, 1, 64, 4, 256).permute(0, 1, 3, 2, 4).reshape(n, 1, 256, 256)
    return x


def clap_audio_embed(sd: SD, wav: torch.Tensor, sampling_rate: int, depths=(2, 2, 12, 2), heads=(4, 8, 16, 32),
                     window: int = 8, eps: float = 1e-5, dtype=torch.float64, device="cpu") -> torch.Tensor:
    """wav [n, L] -> the L2-normalised audio embedding [n, 512] in ``dtype``."""
    sd = {k: v.to(device, dtype) for k, v in sd.items() if k.startswith(("audio_branch.", "audio_projection."))}
    x = wav.to(device, dtype)
    if sampling_rate != 48000:
        x = resample_16k_to_48k(x)
    x = x[:, :480000]
    a = "audio_branch"
    img = wav2img(logmel(sd, x))
    h = F.conv2d(img, sd[f"{a}.patch_embed.proj.weight"], sd[f"{a}.patch_embed.proj.bias"], stride=4)
    n, E, R, _ = h.shape
    h = h.flatten(2).transpose(1, 2)
    ln = lambda nm, v: F.layer_norm(v, (v.shape[-1],), sd[nm + ".weight"], sd[nm + ".bias"], eps)
    lin = lambda nm, v, bias=True: v @ sd[nm + ".weight"].t() + (sd[nm + ".bias"] if bias else 0)
    h = ln(f"{a}.patch_embed.norm", h)
    rpi = relative_position_index(window).to(device)
    C = E
    for i, depth in enumerate(depths):
        H = heads[i]
        for j in range(depth):
            p = f"{a}.layers.{i}.blocks.{j}"
            w = min(window, R)
            shift = 0 if R <= window or j % 2 == 0 else window // 2
            x = ln(f"{p}.norm1", h).view(n, R, R, C)
            if shift:
                x = torch.roll(x, (-shift, -shift), (1, 2))
            xw = partition(x, w).view(-1, w * w, C)
            qkv = lin(f"{p}.attn.qkv", xw).reshape(xw.shape[0], w * w, 3, H, C // H).permute(2, 0, 3, 1, 4)
            q, k, v = qkv[0] * (C // H) ** -0.5, qkv[1], qkv[2]
            att = q @ k.transpose(-2, -1)
            bias = sd[f"{p}.attn.relative_position_bias_table"][rpi.reshape(-1)].view(w * w, w * w, -1).permute(2, 0, 1)
            att = att + bias[None]
            if shift:
                m = shift_mask(R, w, shift).to(att)
                att = (att.view(n, -1, H, w * w, w * w) + m[None, :, None]).view(-1, H, w * w, w * w)
            o = (torch.softmax(att, -1) @ v).transpose(1, 2).reshape(-1, w * w, C)
            o = unpartition(lin(f"{p}.attn.proj", o).view(-1, w, w, C), w, R, R)
            if shift:
                o = torch.roll(o, (shift, shift), (1, 2))
            h = h + o.reshape(n, R * R, C)
            h = h + lin(f"{p}.mlp.fc2", F.gelu(lin(f"{p}.mlp.fc1", ln(f"{p}.norm2", h))))
        if i < len(depths) - 1:
            d = f"{a}.layers.{i}.downsample"
            x = h.view(n, R, R, C)
            x = torch.cat([x[:, 0::2, 0::2], x[:, 1::2, 0::2], x[:, 0::2, 1::2], x[:, 1::2, 1::2]], -1)
            h = lin(f"{d}.reduction", ln(f"{d}.norm", x.reshape(n, -1, 4 * C)), bias=False)
            R, C = R // 2, 2 * C
    e = ln(f"{a}.norm", h).mean(1)
    y = lin("audio_projection.2", torch.relu(lin("audio_projection.0", e)))
    return F.normalize(y, dim=-1)


def replacement_draws(n: int, p: float = 0.1) -> List[bool]:
    """forward's draws after an embedding (encoders/modules.py:730-733): one torch.rand(1) per row, in row order."""
    return [float(torch.rand(1)) < p for _ in range(n)]


def cos_similarity(audio: Callable[[], torch.Tensor], text: Callable[[], torch.Tensor], uncond: torch.Tensor
                   ) -> Tuple[torch.Tensor, List[int], List[int]]:
    """encoders/modules.py:639-653: the audio embeddings with forward's replacement by CLAP(""), then the text
    embeddings with theirs (2 n CPU draws, audio rows first), then F.cosine_similarity over the 512 channels.
    -> (similarity [n], replaced audio rows, replaced text rows)."""
    a = audio().clone()
    ra = [i for i, r in enumerate(replacement_draws(a.shape[0])) if r]
    a[ra] = uncond.to(a)
    t = text().clone()
    rt = [i for i, r in enumerate(replacement_draws(t.shape[0])) if r]
    t[rt] = uncond.to(t)
    return F.cosine_similarity(a[:, None], t[:, None], dim=2).reshape(-1), ra, rt


def select(similarity: torch.Tensor, batchsize: int) -> List[int]:
    """ddpm.py:1554-1564: per prompt i the argmax over rows i, i + B, ..."""
    return [i + int(torch.argmax(similarity[i::batchsize]).item()) * batchsize for i in range(batchsize)]
