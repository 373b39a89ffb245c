"""TEST INFRASTRUCTURE -- pure-torch restatement of the Flan-T5 encoder (never imported by the product path).

``t5_encode`` is what ``FlanT5HiddenState.encode_text`` returns as its hidden states (encoders/modules.py:173-198):
HF ``T5EncoderModel(input_ids, attention_mask)[0]`` for the gated-GELU T5 configuration of google/flan-t5-large
(transformers models/t5/modeling_t5.py: T5Stack, T5Block, T5LayerSelfAttention, T5Attention, T5LayerFF,
T5DenseGatedActDense, T5LayerNorm), with dropout off.  It runs in the dtype of the state dict it is given (float64 for
the tests' references, float32 / TF32 on a GPU for the timing script's baseline).  It is pinned to the unmodified
reference by tests/golden/make_t5_golden.py.
"""
from __future__ import annotations

import math
from typing import Dict

import torch

SD = Dict[str, torch.Tensor]


def gelu_new(x: torch.Tensor) -> torch.Tensor:
    """transformers NewGELUActivation (``dense_act_fn = "gelu_new"`` of the gated-gelu configuration)."""
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * torch.pow(x, 3.0))))


def relative_position_bucket(rp: torch.Tensor, num_buckets: int = 32, max_distance: int = 128) -> torch.Tensor:
    """T5Attention._relative_position_bucket, bidirectional (the encoder)."""
    num_buckets //= 2
    out = (rp > 0).to(torch.long) * num_buckets
    rp = torch.abs(rp)
    max_exact = num_buckets // 2
    large = max_exact + (torch.log(rp.float() / max_exact) / math.log(max_distance / max_exact)
                         * (num_buckets - max_exact)).to(torch.long)
    large = torch.min(large, torch.full_like(large, num_buckets - 1))
    return out + torch.where(rp < max_exact, rp, large)


def rms_norm(x: torch.Tensor, w: torch.Tensor, eps: float) -> torch.Tensor:
    """T5LayerNorm: x * rsqrt(mean(x^2) + eps) * w -- no mean subtraction, no bias."""
    return w * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps))


def t5_encode(sd: SD, ids: torch.Tensor, mask: torch.Tensor, n_layer: int, n_head: int = 16, d_kv: int = 64,
              eps: float = 1e-6, dtype=torch.float64, device="cpu") -> torch.Tensor:
    """ids [B, L] int, mask [B, L] (1 = token) -> hidden states [B, L, 1024] in ``dtype``.

    T5Stack.forward: h = embed_tokens(ids) (not scaled); extended mask (1 - mask) * finfo.min; per block
    h += o(attn(rms(h))) with scores q k^T (no 1/sqrt(d)) + layer 0's position bias + mask; then
    h += wo(gelu_new(wi_0(rms(h))) * wi_1(rms(h))); final_layer_norm."""
    sd = {k: v.to(device, dtype) for k, v in sd.items()}
    ids = ids.to(device)
    B, L = ids.shape
    h = sd["shared.weight"][ids]
    minv = torch.finfo(dtype).min
    ext = (1.0 - mask.to(device, dtype))[:, None, None, :] * minv
    pos = torch.arange(L, device=device)
    bucket = relative_position_bucket(pos[None, :] - pos[:, None])
    bias = sd["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"][bucket].permute(2, 0, 1)[None]
    bias = bias + ext                                   # position_bias, computed in block 0 and passed to every block

    def lin(n, x):
        return x @ sd[n + ".weight"].t()

    for i in range(n_layer):
        p = f"encoder.block.{i}.layer"
        a = rms_norm(h, sd[f"{p}.0.layer_norm.weight"], eps)
        q, k, v = (lin(f"{p}.0.SelfAttention.{n}", a).reshape(B, L, n_head, d_kv).transpose(1, 2) for n in "qkv")
        s = q @ k.transpose(-1, -2) + bias
        w = torch.softmax(s, dim=-1)                    # HF: softmax(s.float()).type_as(s), the same in fp32 / fp64
        o = (w @ v).transpose(1, 2).reshape(B, L, n_head * d_kv)
        h = h + lin(f"{p}.0.SelfAttention.o", o)
        a = rms_norm(h, sd[f"{p}.1.layer_norm.weight"], eps)
        f = f"{p}.1.DenseReluDense"
        h = h + lin(f + ".wo", gelu_new(lin(f + ".wi_0", a)) * lin(f + ".wi_1", a))
    return rms_norm(h, sd["encoder.final_layer_norm.weight"], eps)
