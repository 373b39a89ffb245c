"""TEST INFRASTRUCTURE -- pure-torch restatement of the CLAP text embedding (never imported by the product path).

``clap_text_embed`` is what ``CLAP.get_text_embedding`` returns (clap/open_clip/model.py:656-663, 730-750) for the
"roberta" text branch: HF ``RobertaModel(input_ids, attention_mask)["pooler_output"]`` (transformers
models/roberta/modeling_roberta.py: RobertaEmbeddings with create_position_ids_from_input_ids, post-LN RobertaLayer,
RobertaPooler), then ``text_projection`` (Linear, ReLU, Linear) and ``F.normalize``, with dropout off.  It runs in the
dtype asked for (float64 for the tests' references, float32 / TF32 on a GPU for the timing script's baseline).  It is
pinned to the unmodified reference by tests/golden/make_clap_golden.py.
"""
from __future__ import annotations

import math
from typing import Dict

import torch
import torch.nn.functional as F

SD = Dict[str, torch.Tensor]


def position_ids(ids: torch.Tensor, pad: int = 1) -> torch.Tensor:
    """create_position_ids_from_input_ids: cumsum(id != pad) * (id != pad) + pad, per row."""
    m = (ids != pad).int()
    return (torch.cumsum(m, dim=1).type_as(m) * m).long() + pad


def gelu(x: torch.Tensor) -> torch.Tensor:
    """transformers GELUActivation (hidden_act "gelu"): the erf form."""
    return x * 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0)))


def clap_text_embed(sd: SD, ids: torch.Tensor, mask: torch.Tensor, n_layer: int, n_head: int = 12, eps: float = 1e-5,
                    dtype=torch.float64, device="cpu") -> torch.Tensor:
    """ids [B, L] int, mask [B, L] (1 = token) -> the L2-normalised text embedding [B, 512] in ``dtype``.

    RobertaEmbeddings: LN((word[ids] + token_type[0]) + position[pid]); extended mask (1 - mask) * finfo.min; per layer
    h = LN(h + o(softmax(q k^T / sqrt(64) + mask) v)), h = LN(h + out(gelu(inter(h)))); pooler tanh(dense(h[:, 0]));
    text_projection; F.normalize."""
    sd = {k: v.to(device, dtype) for k, v in sd.items() if k.startswith(("text_branch.", "text_projection."))}
    ids = ids.to(device)
    B, L = ids.shape
    C = sd["text_branch.embeddings.word_embeddings.weight"].shape[1]
    d = C // n_head
    e = "text_branch.embeddings"

    def ln(n, x):
        return F.layer_norm(x, (C,), sd[n + ".weight"], sd[n + ".bias"], eps)

    def lin(n, x):
        return x @ sd[n + ".weight"].t() + sd[n + ".bias"]

    h = sd[f"{e}.word_embeddings.weight"][ids] + sd[f"{e}.token_type_embeddings.weight"][0]
    h = ln(f"{e}.LayerNorm", h + sd[f"{e}.position_embeddings.weight"][position_ids(ids)])
    ext = (1.0 - mask.to(device, dtype))[:, None, None, :] * torch.finfo(dtype).min
    for i in range(n_layer):
        p = f"text_branch.encoder.layer.{i}"
        q, k, v = (lin(f"{p}.attention.self.{n}", h).reshape(B, L, n_head, d).transpose(1, 2) for n in ("query", "key", "value"))
        w = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(d) + ext, dim=-1)
        o = (w @ v).transpose(1, 2).reshape(B, L, C)
        h = ln(f"{p}.attention.output.LayerNorm", lin(f"{p}.attention.output.dense", o) + h)
        h = ln(f"{p}.output.LayerNorm", lin(f"{p}.output.dense", gelu(lin(f"{p}.intermediate.dense", h))) + h)
    pooled = torch.tanh(lin("text_branch.pooler.dense", h[:, 0]))
    y = lin("text_projection.2", torch.relu(lin("text_projection.0", pooled)))
    return F.normalize(y, dim=-1)
