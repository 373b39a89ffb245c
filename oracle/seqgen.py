"""TEST INFRASTRUCTURE -- pure-torch restatement of the AudioMAE token generator (never imported by the product path).

``audiomae_generate`` is what ``SequenceGenAudioMAECond.forward`` puts under ``crossattn_audiomae_generated``: the
input sequence of ``Sequence2AudioMAE.get_input_sequence_and_mask`` + ``add_sos_eos_tokens``
(audiomae_gen/sequence_input.py:110-201) and the ``generate`` loop (:294-325), i.e. ``gen_len`` full forward passes of
HF ``GPT2Model`` (eager attention) without a cache, each over a sequence one position longer than the last.  It runs in
the dtype of its inputs (float64 for the tests' references, float32 on a GPU for the timing script's baseline).  It is
pinned to the unmodified reference by tests/golden/make_seqgen_golden.py.
"""
from __future__ import annotations

import math
from typing import Dict

import torch
import torch.nn.functional as F

SD = Dict[str, torch.Tensor]


def gelu_new(x: torch.Tensor) -> torch.Tensor:
    """transformers NewGELUActivation (GPT-2's ``gelu_new``)."""
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * torch.pow(x, 3.0))))


def gpt2_forward(sd: SD, embeds: torch.Tensor, mask: torch.Tensor, n_layer: int, n_head: int = 12,
                 eps: float = 1e-5) -> torch.Tensor:
    """GPT2Model(inputs_embeds, attention_mask).last_hidden_state: position ids arange(T); attention weights
    where(causal, w, finfo.min) + (1 - mask) * finfo.min; Conv1D layers y = x W + b."""
    B, T, C = embeds.shape
    dt = embeds.dtype
    minv = torch.finfo(dt).min
    h = embeds + sd["model.wpe.weight"][:T]
    causal = torch.tril(torch.ones(T, T, dtype=torch.bool, device=embeds.device))
    add = (1.0 - mask.to(dt))[:, None, None, :] * minv
    hd = C // n_head

    def c1d(n, x):
        return x @ sd[n + ".weight"] + sd[n + ".bias"]

    def ln(n, x):
        return F.layer_norm(x, (C,), sd[n + ".weight"], sd[n + ".bias"], eps)

    for i in range(n_layer):
        p = f"model.h.{i}"
        q, k, v = c1d(p + ".attn.c_attn", ln(p + ".ln_1", h)).split(C, dim=2)
        q, k, v = (t.reshape(B, T, n_head, hd).transpose(1, 2) for t in (q, k, v))
        w = (q @ k.transpose(-1, -2)) / (hd ** 0.5)
        w = torch.where(causal, w, torch.tensor(minv, dtype=dt, device=w.device)) + add
        o = (torch.softmax(w, dim=-1) @ v).transpose(1, 2).reshape(B, T, C)
        h = h + c1d(p + ".attn.c_proj", o)
        h = h + c1d(p + ".mlp.c_proj", gelu_new(c1d(p + ".mlp.c_fc", ln(p + ".ln_2", h))))
    return ln("model.ln_f", h)


def input_sequence(sd: SD, clap: torch.Tensor, t5: torch.Tensor, t5_mask: torch.Tensor):
    """[sos0, Linear0(clap), eos0, sos1, Linear1(t5), eos1] and its mask (sequence_input.py:110-201)."""
    B = clap.shape[0]
    dt = clap.dtype
    parts, masks = [], []
    for i, (x, m) in enumerate(((clap.reshape(B, 1, -1), torch.ones(B, 1, dtype=dt, device=clap.device)), (t5, t5_mask.to(dt)))):
        e = F.linear(x, sd[f"input_sequence_embed_linear.{i}.weight"], sd[f"input_sequence_embed_linear.{i}.bias"])
        sos = sd["start_of_sequence_tokens.weight"][i].expand(B, 1, -1)
        eos = sd["end_of_sequence_tokens.weight"][i].expand(B, 1, -1)
        one = torch.ones(B, 1, dtype=dt, device=clap.device)
        parts.append(torch.cat([sos, e, eos], 1))
        masks.append(torch.cat([one, m, one], 1))
    return torch.cat(parts, 1), torch.cat(masks, 1)


def audiomae_generate(sd: SD, clap: torch.Tensor, t5: torch.Tensor, t5_mask: torch.Tensor, n_layer: int = 12,
                      gen_len: int = 8) -> torch.Tensor:
    """-> [B, gen_len, 768] in the dtype of ``clap`` (the state dict is cast to it)."""
    dt, dev = clap.dtype, clap.device
    sd = {k: v.to(dev, dt) for k, v in sd.items() if k != "model.wte.weight"}
    x, m = input_sequence(sd, clap.to(dt), t5.to(dev, dt), t5_mask.to(dev, dt))
    P = x.shape[1]
    for _ in range(gen_len):
        out = gpt2_forward(sd, x, m, n_layer)
        x = torch.cat([x, out[:, -1:]], 1)
        m = torch.cat([m, torch.ones(m.shape[0], 1, dtype=dt, device=dev)], 1)
    return x[:, P:]
