"""NativeAudioMAEGenerator: the AudioMAE conditioning tokens of the sequence-generation models, generated natively.

``generate(clap, t5, t5_mask)`` returns the tensor ``SequenceGenAudioMAECond.forward`` puts under
``crossattn_audiomae_generated`` (audiomae_gen/sequence_input.py:294-325, encoders/modules.py:271-300): GPT-2 small run
autoregressively over [sos0, CLAP, eos0, sos1, Flan-T5, eos1] for 8 tokens.  The reference runs 8 full forward passes;
here one prefill pass fills per-layer KV caches and 7 single-position passes extend them (plan.build_seqgen), all
as sm_90a kernels in one op table, replayed as a CUDA graph.

Plans depend on (B, L): the position of every generated token is L + 5 + k, so a prompt's tokens depend on the T5
padding length of its call, exactly as in the reference (padding=True pads to the longest prompt).  Plans are built
lazily per shape and the two most recent are kept; all of them share one uploaded weight arena.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Dict

import torch

from . import arch, engine, plan


class NativeAudioMAEGenerator:
    def __init__(self, state_dict: Dict[str, torch.Tensor], device="cuda:0", gen_len: int = None, use_graph: bool = True,
                 max_plans: int = 2):
        """``state_dict``: keys relative to ``cond_stage_models.<i>.`` (model.split_seqgen_state_dict or
        synth.seqgen_state_dict)."""
        if not torch.cuda.is_available():
            raise RuntimeError("the native AudioMAE generator needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device(device)
        self.gen_len = int(gen_len or arch.SEQGEN["gen_len"])
        self.use_graph = use_graph
        self.max_plans = max_plans
        self.weights = plan.pack_seqgen_weights(state_dict)
        self.arena = self.weights.arena.to(self.device)
        self._progs: "OrderedDict[tuple, engine.DeviceProgram]" = OrderedDict()

    def program(self, B: int, L: int) -> engine.DeviceProgram:
        key = (int(B), int(L))
        prog = self._progs.get(key)
        if prog is not None:
            self._progs.move_to_end(key)
            return prog
        while len(self._progs) >= self.max_plans:
            self._progs.popitem(last=False)[1].close()
        pl = plan.build_seqgen(None, B, L, self.gen_len, weights=self.weights)
        m = pl.marks
        prog = engine.DeviceProgram(pl, self.device, dict(all=(m["begin"], m["end"]), prefill=(m["begin"], m["prefill_end"]),
                                                          decode=(m["prefill_end"], m["end"])), arena_dev=self.arena)
        self._progs[key] = prog
        return prog

    @torch.no_grad()
    def generate(self, clap: torch.Tensor, t5: torch.Tensor, t5_mask: torch.Tensor) -> torch.Tensor:
        """clap [B, 1, 512] (or [B, 512]), t5 [B, L, 1024], t5_mask [B, L] (1 = token, 0 = padding; position 0 of the
        sequence is a SOS token, so no row is fully masked) -> tokens [B, gen_len, 768] float32 on the device."""
        B = clap.shape[0]
        d0, d1 = arch.SEQGEN["input_dims"]
        if clap.numel() != B * d0:
            raise ValueError(f"CLAP embedding must be [B, 1, {d0}], got {tuple(clap.shape)}")
        if t5.dim() != 3 or t5.shape[0] != B or t5.shape[2] != d1 or tuple(t5_mask.shape) != tuple(t5.shape[:2]):
            raise ValueError(f"Flan-T5 states must be [B, L, {d1}] with a [B, L] mask, got {tuple(t5.shape)} / {tuple(t5_mask.shape)}")
        prog = self.program(B, t5.shape[1])
        prog.view("clap").copy_(clap.reshape(B, 1, d0))
        prog.view("t5").copy_(t5)
        prog.view("t5_mask").copy_(t5_mask)
        if self.use_graph:
            prog.replay("all")
        else:
            prog.run("all")
        return prog.view("tokens").clone()
