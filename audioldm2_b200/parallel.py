"""Multi-GPU: one process per GPU, independent batch shards, ONE NCCL broadcast of the packed weight
arenas at load and no per-step collective (SURVEY.md 8e).  Every latent sample is independent
through all DDIM steps, decode and vocode, so ranks never exchange data on the hot path."""
from __future__ import annotations

import os
from typing import Optional

import torch
import torch.distributed as dist


def init_from_env(backend: Optional[str] = None):
    """Initialise torch.distributed from torchrun's environment; returns (rank, world, local_rank)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        backend = backend or ("nccl" if torch.cuda.is_available() else "gloo")
        dist.init_process_group(backend=backend, rank=rank, world_size=world)
    return rank, world, local


def shard_range(n_items: int, rank: int, world: int):
    """Contiguous shard [lo, hi) of ``n_items`` units for ``rank`` (first ranks take the remainder)."""
    base, rem = divmod(n_items, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


class ShardedNoise:
    """SURVEY.md 8e seeding rule: an N-rank run must produce the rows the single-process batch would.  Every rank draws
    the FULL-batch tensors (x_T, then per DDIM step the q_sample noise when masked and the step noise, in the reference's
    order, ddim.py:191,351 / ddpm.py:431) from the same seed with the same generator and keeps rows [lo, hi) -- 131 KB per
    sample and draw, no communication.  Use as ``x_T=sn.x_T(), noise_fn=sn`` of ``generate_latent``."""

    def __init__(self, global_batch: int, lo: int, hi: int, latent, device, seed: int = 42, generator=None, rows=None):
        """Rows [lo, hi) of the global batch, or an explicit index list ``rows`` (the candidates of prompt i sit at
        rows i + k * batchsize, ddpm.py:1560-1562, so a rank that owns prompts [lo, hi) owns a strided row set)."""
        self.shape = (int(global_batch),) + tuple(int(v) for v in latent)
        self.lo, self.hi, self.device = lo, hi, torch.device(device)
        self.rows = None if rows is None else torch.as_tensor(rows, dtype=torch.long, device=self.device)
        if generator is None:
            generator = torch.Generator(device=self.device)
            generator.manual_seed(int(seed))
        self.gen = generator

    def _draw(self) -> torch.Tensor:
        full = torch.randn(self.shape, device=self.device, generator=self.gen)
        return (full[self.lo:self.hi] if self.rows is None else full[self.rows]).contiguous()

    def x_T(self) -> torch.Tensor:
        return self._draw()

    def __call__(self, i: int, kind: str) -> torch.Tensor:
        return self._draw()


def shard_rows(t, lo: int, hi: int):
    """Rows [lo, hi) of every tensor in a (nested) conditioning structure."""
    if t is None:
        return None
    if torch.is_tensor(t):
        return t[lo:hi].contiguous()
    if isinstance(t, dict):
        return {k: shard_rows(v, lo, hi) for k, v in t.items()}
    if isinstance(t, (list, tuple)):
        return [shard_rows(v, lo, hi) for v in t]
    return t


def current_shard(n_items: int):
    """(rank, world, lo, hi) of this process for ``n_items`` independent units, or None in a single-process run."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return None
    r, w = dist.get_rank(), dist.get_world_size()
    lo, hi = shard_range(n_items, r, w)
    return r, w, lo, hi


def all_gather_rows(local: torch.Tensor, n_items: int) -> torch.Tensor:
    """Concatenate the ranks' row shards (shard_range order) into the full [n_items, ...] tensor on every rank: the one
    collective at the END of a sharded generation (SURVEY.md 8e); shards may differ by one row."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return local
    w = dist.get_world_size()
    sizes = [shard_range(n_items, r, w) for r in range(w)]
    mx = max(b - a for a, b in sizes)
    pad = torch.zeros((mx,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[:local.shape[0]] = local
    bufs = [torch.empty_like(pad) for _ in range(w)]
    dist.all_gather(bufs, pad)
    return torch.cat([bufs[r][:b - a] for r, (a, b) in enumerate(sizes)], dim=0)


def make_arena_bcast(device, src: int = 0):
    """Hook for NativeLatentDiffusion(arena_bcast=...): rank ``src`` uploads its packed arena, every
    other rank receives it over NCCL (NVLink/NVSwitch) instead of packing + uploading its own."""
    def bcast(name: str, cpu_arena: torch.Tensor, nbytes: int) -> torch.Tensor:
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
            return cpu_arena.to(device)
        if dist.get_rank() == src:
            t = cpu_arena.to(device)
        else:
            t = torch.empty(nbytes, dtype=torch.uint8, device=device)
        dist.broadcast(t, src=src)
        return t
    return bcast


def max_over_ranks(value: float, device) -> float:
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return value
    t = torch.tensor([value], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def guard_flags(x: torch.Tensor) -> torch.Tensor:
    """The two inputs of AudioLDM 1's latent guard (``torch.max(torch.abs(x)) > 1e2`` then clip to [-10, 10]), made on
    x's device without a host synchronisation: int32 [over, has_nan], over = max |x| > 100 (strict) and has_nan = any
    NaN in x.  A NaN makes the reference's max NaN, so it must veto the clip."""
    return torch.stack([torch.amax(torch.abs(x)) > 1e2, torch.isnan(x).any()]).to(torch.int32)


def reduce_guard_flags(flags: torch.Tensor) -> torch.Tensor:
    """guard_flags of every rank's rows combined with MAX, in place: one two-word collective per call, after which every
    rank holds the flags of the whole batch and makes the single-process decision.  No-op in a single process."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(flags, op=dist.ReduceOp.MAX)
    return flags


def guard_decision(flags: torch.Tensor) -> torch.Tensor:
    """int32 [1] on the flags' device: 1 = clip (over and no NaN), the guard word aldm_stochastic_encode reads."""
    return (flags[0] * (1 - flags[1])).reshape(1).to(torch.int32).contiguous()


def latent_guard_flag(x: torch.Tensor) -> torch.Tensor:
    """AudioLDM 1's guard decision for the whole batch of the call (all ranks' rows in a sharded run)."""
    return guard_decision(reduce_guard_flags(guard_flags(x)))


def barrier():
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.barrier()
