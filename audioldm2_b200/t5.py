"""NativeFlanT5Encoder: the Flan-T5-large text encoder, run natively from token ids.

``encode(ids, mask)`` returns what ``FlanT5HiddenState.encode_text`` returns as its hidden states
(encoders/modules.py:173-198): ``T5EncoderModel(input_ids, attention_mask)[0]``, [B, L, 1024] float32.  The tokenizer (a
sentencepiece hub asset) stays with the caller, which passes its ids and attention mask (max_length 128, padding=True,
pad id 0).  ``unconditional(n)`` is ``get_unconditional_condition``: T5("") = T5([[1]]), computed once and cached.

Every kernel is sm_90a code of this package (plan.build_t5: embedding, 24 blocks of 8 launches, final_layer_norm), one op
table per (B, L) replayed as a CUDA graph; plans are built lazily and the two most recent are kept, all sharing one
uploaded weight arena.  After each run the per-block count of gated-GELU values beyond the fp16 range is read back: the
operand planes of the wo GEMM would clamp them, so a nonzero count raises instead of returning a silently clamped result.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Dict, Optional

import torch

from . import arch, engine, plan


def check_tokens(ids: torch.Tensor, mask: torch.Tensor):
    """Raise ValueError unless ids [B, L] are integers in [0, vocab), mask [B, L] holds only 0 / 1 with at least one 1 per
    row, and 1 <= L <= 128 (the tokenizer's max_length)."""
    V, Lmax = arch.T5["vocab"], arch.T5["max_len"]
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


class NativeFlanT5Encoder:
    def __init__(self, state_dict: Optional[Dict[str, torch.Tensor]] = None, device="cuda:0", use_graph: bool = True,
                 max_plans: int = 2, weights: Optional[plan.T5Weights] = None, arena_dev: Optional[torch.Tensor] = None):
        """``state_dict``: HF ``T5EncoderModel`` keys (model.split_t5_state_dict or synth.t5_state_dict).  Or ``weights`` /
        ``arena_dev``: an already packed (and uploaded) arena, shared with another encoder."""
        if not torch.cuda.is_available():
            raise RuntimeError("the native Flan-T5 encoder needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device(device)
        self.use_graph = use_graph
        self.max_plans = max_plans
        self.weights = weights if weights is not None else plan.pack_t5_weights(state_dict)
        self.arena = arena_dev if arena_dev is not None else self.weights.arena.to(self.device)
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
        pl = plan.build_t5(None, B, L, weights=self.weights)
        prog = engine.DeviceProgram(pl, self.device, dict(all=(pl.marks["begin"], pl.marks["end"])), arena_dev=self.arena)
        self._progs[key] = prog
        return prog

    @torch.no_grad()
    def encode(self, ids: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
        """ids [B, L] integer, mask [B, L] (1 = token, 0 = padding) -> hidden states [B, L, 1024] float32 on the device.
        Padded positions are computed like the reference computes them (their queries attend to the valid keys)."""
        check_tokens(ids, mask)
        B, L = ids.shape
        prog = self.program(B, L)
        prog.view("ids").copy_(ids.to(torch.int64))
        prog.view("mask").copy_(mask.float())
        if self.use_graph:
            prog.replay("all")
        else:
            prog.run("all")
        sat = prog.view("sat")
        counts = sat.cpu()                                   # one small copy on the stream, after the run
        if bool(counts.any()):
            sat.zero_()
            layers = [(i, int(c)) for i, c in enumerate(counts.tolist()) if c]
            raise RuntimeError("Flan-T5 encoder: gated-GELU values beyond the fp16 operand range (|v| > 65504) in block(s) "
                               + ", ".join(f"{i} ({c} values)" for i, c in layers)
                               + "; the wo GEMM's operand planes would clamp them")
        return prog.view("hidden").clone()

    def unconditional(self, n: int) -> torch.Tensor:
        """T5("") for n rows: the tokenizer maps "" to [EOS] = [[1]]; computed once and cached, like the reference's
        ``empty_hidden_state_cfg`` (encoders/modules.py:139-154).  -> [n, 1, 1024]."""
        if self._uncond is None:
            one = torch.ones(1, 1, dtype=torch.int64, device=self.device)
            self._uncond = self.encode(one * arch.T5["eos_id"], one.float())
        return self._uncond.expand(int(n), 1, self._uncond.shape[-1]).contiguous()
