"""Planner: reference config + state_dict  ->  flat op table (IR) for the native executor.

The IR is a list of plain dicts whose fields mirror the C structs in include/aldm_b200.h, with
device pointers replaced by ``Ref(region, byte_offset)``:

* region "w"  -- the packed weight arena (built here on the CPU, uploaded / NCCL-broadcast once);
* region "ws" -- the activation workspace, managed by a plan-time first-fit allocator so buffers
  are reused and the working set of one UNet evaluation stays L2-resident.

``Plan.resolve(w_base, ws_base)`` turns the IR into the ctypes ``Op`` array.  tests/emulator.py
executes the same IR with torch on the CPU, which checks the graph wiring, the weight layouts and
the buffer liveness without a GPU.

Network structure follows the reference modules (citations in each builder).
"""
from __future__ import annotations

import ctypes as C
import math
import os
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import torch

from . import _lib, arch, packing
from .packing import round_up

ALIGN = 256


@dataclass(frozen=True)
class Ref:
    region: str
    off: int

    def __add__(self, nbytes: int) -> "Ref":
        return Ref(self.region, self.off + int(nbytes))


@dataclass
class F32:            # fp32 activation [rows, C] (channels-last)
    ref: Ref
    rows: int
    C: int

    @property
    def nbytes(self):
        return self.rows * self.C * 4


@dataclass
class Planes:         # fp16 operand planes [rows, Cp]: hi = fp16(x) and, for two-plane operands, lo = fp16(x - hi)
    hi: Ref
    lo: Optional[Ref]
    rows: int
    Cp: int

    @property
    def nbytes(self):
        return (1 if self.lo is None else 2) * self.rows * self.Cp * 2


@dataclass
class VT:             # transposed V planes [(b*C + c), ld_t] (keys contiguous), written by an ALDM_OUT_QKV GEMM
    hi: Ref
    lo: Optional[Ref]
    ld_t: int


@dataclass
class WMat:           # packed weight matrix
    packed: Ref
    plain: Optional[Ref]
    bias: Optional[Ref]
    N: int
    K: int
    Kpad: int
    bn: int
    Cp: int
    ntaps: int


class Arena:
    """Byte arena assembled on the CPU."""

    def __init__(self):
        self.chunks: List[Tuple[int, torch.Tensor]] = []
        self.size = 0

    def add(self, t: torch.Tensor) -> int:
        b = t.contiguous().view(torch.uint8).reshape(-1) if t.dtype != torch.uint8 else t.contiguous().reshape(-1)
        off = round_up(self.size, ALIGN)
        self.chunks.append((off, b))
        self.size = off + b.numel()
        return off

    def build(self) -> torch.Tensor:
        out = torch.zeros(round_up(max(self.size, ALIGN), ALIGN), dtype=torch.uint8)
        for off, b in self.chunks:
            out[off:off + b.numel()] = b
        return out


class Pool:
    """Plan-time first-fit allocator with coalescing (offsets into the workspace)."""

    def __init__(self):
        self.free: List[Tuple[int, int]] = []     # (off, size), sorted
        self.top = 0
        self.live: Dict[int, int] = {}
        self.peak = 0

    def alloc(self, nbytes: int) -> int:
        n = round_up(max(int(nbytes), 1), ALIGN)
        for i, (off, sz) in enumerate(self.free):
            if sz >= n:
                if sz == n:
                    self.free.pop(i)
                else:
                    self.free[i] = (off + n, sz - n)
                self.live[off] = n
                return off
        # grow: if the last free block touches the top, extend it
        if self.free and self.free[-1][0] + self.free[-1][1] == self.top:
            off, sz = self.free.pop()
            self.top = off + n
        else:
            off = self.top
            self.top += n
        self.live[off] = n
        self.peak = max(self.peak, self.top)
        return off

    def release(self, off: int):
        n = self.live.pop(off)
        self.free.append((off, n))
        self.free.sort()
        merged = []
        for o, s in self.free:
            if merged and merged[-1][0] + merged[-1][1] == o:
                merged[-1] = (merged[-1][0], merged[-1][1] + s)
            else:
                merged.append((o, s))
        self.free = merged


@dataclass
class Plan:
    ops: List[dict]
    arena: torch.Tensor                  # CPU uint8
    ws_bytes: int
    io: Dict[str, object]                # name -> F32 / Planes / (Ref, shape, dtype)
    marks: Dict[str, int] = field(default_factory=dict)    # named op indices (program split points)
    meta: Dict[str, object] = field(default_factory=dict)

    def resolve(self, w_base: int, ws_base: int, first: int = 0, last: Optional[int] = None):
        """IR -> ctypes Op array with absolute device addresses."""
        base = {"w": w_base, "ws": ws_base}

        def P(r):
            if r is None:
                return None
            return base[r.region] + r.off

        ops = self.ops[first:last]
        arr = (_lib.Op * len(ops))()
        for i, o in enumerate(ops):
            op = arr[i]
            op.tag = int(o.get("tag", 0))
            k = o["kind"]
            if k == "gemm":
                op.kind = _lib.OP_GEMM
                g = op.u.gemm
                for name in ("a_hi", "a_lo", "w_packed", "w_plain", "bias", "rowvec", "res", "out", "out_hi", "out_lo",
                             "out2_hi", "out2_lo", "ws"):
                    setattr(g, name, P(o.get(name)))
                for name in ("n_split", "tok_per_batch", "ld_t"):
                    setattr(g, name, int(o.get(name, 0)))
                for name in ("B", "H", "W", "Cp", "up", "bmod", "OH", "OW", "sy", "sx", "ntaps", "N", "K", "Kpad", "bn",
                             "ldo", "ld_res", "ld_rowvec", "OHF", "OWF", "osy", "ooy", "act", "out_mode", "accumulate",
                             "splitk", "impl"):
                    setattr(g, name, int(o[name]))
                g.alpha = float(o["alpha"])
                for t, (dy, dx) in enumerate(o["taps"]):
                    g.dy[t] = dy
                    g.dx[t] = dx
            elif k == "prep":
                op.kind = _lib.OP_PREP
                p = op.u.prep
                for name in ("src0", "src1", "gamma", "beta", "out_hi", "out_lo", "scratch"):
                    setattr(p, name, P(o.get(name)))
                for name in ("rows", "c0", "c1", "Cp", "B", "HW", "groups", "mode", "src_nchw"):
                    setattr(p, name, int(o[name]))
                p.eps = float(o["eps"]); p.slope = float(o["slope"])
            elif k == "attn":
                op.kind = _lib.OP_ATTN
                a = op.u.attn
                for name in ("q_hi", "q_lo", "k_hi", "k_lo", "vt_hi", "vt_lo", "mask", "out_hi", "out_lo"):
                    setattr(a, name, P(o.get(name)))
                for name in ("B", "heads", "Nq", "Nk", "ldq", "ldk", "ld_t", "ldo", "q_col", "k_col", "kv_bmod", "impl"):
                    setattr(a, name, int(o[name]))
                a.scale = float(o["scale"])
            elif k == "softmax":
                op.kind = _lib.OP_SOFTMAX
                s = op.u.softmax
                s.x, s.out_hi, s.out_lo = P(o["x"]), P(o["out_hi"]), P(o["out_lo"])
                s.rows, s.n, s.scale = int(o["rows"]), int(o["n"]), float(o["scale"])
            elif k == "temb":
                op.kind = _lib.OP_TEMB
                t = op.u.temb
                t.t, t.freqs, t.out_hi, t.out_lo = P(o["t"]), P(o["freqs"]), P(o["out_hi"]), P(o["out_lo"])
                t.B, t.dim = int(o["B"]), int(o["dim"])
            elif k == "packb":
                op.kind = _lib.OP_PACKB
                b = op.u.packb
                b.src, b.dst_packed, b.dst_plain = P(o["src"]), P(o["dst_packed"]), P(o.get("dst_plain"))
                b.lds, b.transpose, b.N, b.K, b.bn = int(o["lds"]), int(o["transpose"]), int(o["N"]), int(o["K"]), int(o["bn"])
            elif k == "seq_assemble":
                op.kind = _lib.OP_SEQ_ASSEMBLE
                a = op.u.seq_assemble
                for name in ("x", "sos", "eos", "wpe", "t5_mask", "mask"):
                    setattr(a, name, P(o[name]))
                for name in ("B", "L", "lmax", "C"):
                    setattr(a, name, int(o[name]))
            elif k == "kv_attn":
                op.kind = _lib.OP_KV_ATTN
                a = op.u.kv_attn
                for name in ("seq", "mask", "out_hi", "out_lo"):
                    setattr(a, name, P(o.get(name)))
                for name in ("B", "heads", "lmax", "ld_seq", "p0", "nq", "ldo"):
                    setattr(a, name, int(o[name]))
                a.scale = float(o["scale"])
            elif k == "seq_feedback":
                op.kind = _lib.OP_SEQ_FEEDBACK
                a = op.u.seq_feedback
                for name in ("x", "gamma", "beta", "wpe", "out", "next"):
                    setattr(a, name, P(o.get(name)))
                for name in ("B", "nq", "C", "pos", "k", "gen_len"):
                    setattr(a, name, int(o[name]))
                a.eps = float(o["eps"])
            elif k == "t5_embed":
                op.kind = _lib.OP_T5_EMBED
                a = op.u.t5_embed
                a.ids, a.table, a.out = P(o["ids"]), P(o["table"]), P(o["out"])
                a.rows, a.vocab, a.C = int(o["rows"]), int(o["vocab"]), int(o["C"])
            elif k == "t5_rmsnorm":
                op.kind = _lib.OP_T5_RMSNORM
                a = op.u.t5_rmsnorm
                for name in ("x", "gamma", "out_hi", "out_lo", "out_f32"):
                    setattr(a, name, P(o.get(name)))
                a.rows, a.C, a.ldo, a.eps = int(o["rows"]), int(o["C"]), int(o["ldo"]), float(o["eps"])
            elif k == "t5_attn":
                op.kind = _lib.OP_T5_ATTN
                a = op.u.t5_attn
                for name in ("qkv", "bias", "mask", "out_hi", "out_lo"):
                    setattr(a, name, P(o.get(name)))
                for name in ("B", "L", "heads", "d_kv", "C", "ld_qkv", "ldo"):
                    setattr(a, name, int(o[name]))
            elif k == "t5_gate":
                op.kind = _lib.OP_T5_GATE
                a = op.u.t5_gate
                for name in ("x", "out_hi", "out_lo", "sat"):
                    setattr(a, name, P(o.get(name)))
                a.rows, a.F, a.ld_x, a.ldo = int(o["rows"]), int(o["F"]), int(o["ld_x"]), int(o["ldo"])
            elif k == "clap_embed":
                op.kind = _lib.OP_CLAP_EMBED
                a = op.u.clap_embed
                for name in ("ids", "word", "pos", "type", "out"):
                    setattr(a, name, P(o[name]))
                for name in ("B", "L", "vocab", "n_pos", "C", "pad"):
                    setattr(a, name, int(o[name]))
            elif k == "clap_ln":
                op.kind = _lib.OP_CLAP_LN
                a = op.u.clap_ln
                for name in ("x", "gamma", "beta", "out_f32", "out_hi", "out_lo"):
                    setattr(a, name, P(o.get(name)))
                a.rows, a.C, a.ldo, a.eps = int(o["rows"]), int(o["C"]), int(o["ldo"]), float(o["eps"])
            elif k == "clap_attn":
                op.kind = _lib.OP_CLAP_ATTN
                a = op.u.clap_attn
                for name in ("qkv", "mask", "out_hi", "out_lo"):
                    setattr(a, name, P(o.get(name)))
                for name in ("B", "L", "heads", "C", "ld_qkv", "ldo"):
                    setattr(a, name, int(o[name]))
            elif k == "clap_gelu":
                op.kind = _lib.OP_CLAP_GELU
                a = op.u.clap_gelu
                for name in ("x", "out_hi", "out_lo"):
                    setattr(a, name, P(o.get(name)))
                a.rows, a.F, a.ld_x, a.ldo = int(o["rows"]), int(o["F"]), int(o["ld_x"]), int(o["ldo"])
            elif k == "clap_head":
                op.kind = _lib.OP_CLAP_HEAD
                a = op.u.clap_head
                for name in ("x", "wp_t", "bp", "w1_t", "b1", "w2_t", "b2", "out"):
                    setattr(a, name, P(o[name]))
                for name in ("B", "L", "C", "P"):
                    setattr(a, name, int(o[name]))
            elif k == "htsat_logmel":
                op.kind = _lib.OP_HTSAT_LOGMEL
                a = op.u.htsat_logmel
                for name in ("wav", "taps", "melW", "bn_mean", "bn_var", "bn_w", "bn_b", "out"):
                    setattr(a, name, P(o.get(name)))
                for name in ("n", "L", "up", "L48", "T"):
                    setattr(a, name, int(o[name]))
                a.eps = float(o["eps"])
            elif k == "htsat_patch":
                op.kind = _lib.OP_HTSAT_PATCH
                a = op.u.htsat_patch
                for name in ("mel", "w", "bias", "gamma", "beta", "out"):
                    setattr(a, name, P(o[name]))
                a.n, a.T, a.eps = int(o["n"]), int(o["T"]), float(o["eps"])
            elif k == "htsat_attn":
                op.kind = _lib.OP_HTSAT_ATTN
                a = op.u.htsat_attn
                for name in ("qkv", "bias", "mask", "out_hi", "out_lo"):
                    setattr(a, name, P(o.get(name)))
                for name in ("n", "R", "shift", "heads", "head_dim", "C", "ld_qkv", "ldo"):
                    setattr(a, name, int(o[name]))
                a.scale = float(o["scale"])
            elif k == "htsat_merge":
                op.kind = _lib.OP_HTSAT_MERGE
                a = op.u.htsat_merge
                for name in ("x", "gamma", "beta", "out_hi", "out_lo"):
                    setattr(a, name, P(o.get(name)))
                for name in ("n", "R", "C", "ldo"):
                    setattr(a, name, int(o[name]))
                a.eps = float(o["eps"])
            elif k == "htsat_head":
                op.kind = _lib.OP_HTSAT_HEAD
                a = op.u.htsat_head
                for name in ("x", "gamma", "beta", "w1_t", "b1", "w2_t", "b2", "out"):
                    setattr(a, name, P(o[name]))
                for name in ("n", "ntok", "C", "P"):
                    setattr(a, name, int(o[name]))
                a.eps = float(o["eps"])
            elif k == "copy":
                op.kind = _lib.OP_COPY
                c = op.u.copy
                c.src, c.dst, c.bytes = P(o["src"]), P(o["dst"]), int(o["bytes"])
            else:
                raise ValueError(k)
        return arr


H100_SMS = 132      # SMs of the H100 SXM: the tile-count heuristics below size one wave of the persistent GEMM


class Planner:
    def __init__(self, impl: str = "tc", keep_plain: bool = False, splitk: bool = True, n_sm: int = H100_SMS):
        self.impl = {"tc": _lib.GEMM_TC, "simt": _lib.GEMM_SIMT}[impl]
        self.keep_plain = keep_plain or impl == "simt"
        self.use_splitk = splitk and impl != "simt"
        self.static_b = os.environ.get("ALDM_BPRE", "1") != "0"      # weight prefetch ahead of the PDL wait (A/B switch)
        self.n_sm = n_sm
        # planes of the token-side operands of the UNet (LayerNorm outputs, Q|K, V^T, attention output, GEGLU output):
        # 1 = single fp16 plane (default; precision budget in DESIGN.md section 3), 2 = hi + lo everywhere
        self.tok_planes = 2 if os.environ.get("ALDM_TOKEN_PLANES", "1") == "2" else 1
        self.arena = Arena()
        self.pool = Pool()
        self.ops: List[dict] = []
        self.tag = 0
        self.marks: Dict[str, int] = {}
        self._gn_scr: Dict[int, int] = {}       # GroupNorm scratch bytes per batch size (its layout depends on B: csrc/prep.cu)
        self.splitk_ws: Optional[Ref] = None
        self.splitk_ws_bytes = 0

    # ---- weights -------------------------------------------------------------------------
    def vec(self, t: torch.Tensor) -> Ref:
        return Ref("w", self.arena.add(t.float().contiguous()))

    def bn_for_rows(self, N: int, m_rows: Optional[int], geglu: bool = False, min_bn: int = 32) -> int:
        """N tile: 128 unless the GEMM is too small to give every SM a tile -- then the widest tile that
        yields >= ~0.8 * n_sm tiles (per-tile time of a short K loop is dominated by fixed latencies, so
        more, narrower tiles in flight win)."""
        cands = [b for b in ((128, 64) if geglu else (128, 64, 32)) if N % b == 0 and b >= min_bn]
        if not cands:
            return 128 if geglu else packing.choose_bn(N)
        if not m_rows:
            return cands[0]
        mt = math.ceil(m_rows / 128)
        for b in cands:
            if mt * (N // b) >= int(0.8 * self.n_sm):
                return b
        return cands[-1]

    def wmat(self, wm: torch.Tensor, bias: Optional[torch.Tensor], ntaps: int, cp: int, geglu: bool = False,
             bn: Optional[int] = None, m_rows: Optional[int] = None) -> WMat:
        N, K = wm.shape
        assert K == ntaps * cp
        # Narrower tiles as a general rule for small-M GEMMs cost a second wave at the 256-pixel level, twice the weight traffic
        # and no split-K for the long-K convolutions (ALDM_NARROW=64 / 32 selects them, for experiments).  One case is different:
        # a SHORT-K GEMM whose 128-wide tiles fill at most half the SMs (the 64-pixel level: 1024 x 640 x 640 = 40 tiles on 132
        # SMs) is a latency chain load -> MMA -> 64 KB of stores per CTA; halving the tile width halves the MMA and store phases
        # of each CTA while the tiles still fit one wave.  ALDM_HALF_TILES=0 switches it off (A/B).
        narrow = int(os.environ.get("ALDM_NARROW", "0"))       # experiment switch: smallest N tile the heuristic may pick
        explicit = bn is not None
        bn = bn or self.bn_for_rows(N, m_rows if narrow else None, geglu, min_bn=narrow or 32)
        if (not explicit and not narrow and m_rows and bn == 128 and N % 64 == 0 and os.environ.get("ALDM_HALF_TILES", "1") != "0"
                and math.ceil(K / 64) < 24 and not geglu):
            tiles = math.ceil(m_rows / 128) * math.ceil(N / 128)
            if tiles * 2 <= self.n_sm:
                bn = 64
        if geglu:
            order = packing.geglu_row_order(N // 2, bn)
            wm = wm[order]
            bias = bias[order] if bias is not None else None
        packed, plain, Npad, Kpad = packing.pack_tiles(wm, bn)
        bref = None
        if bias is not None:
            bp = torch.zeros(Npad, dtype=torch.float32)
            bp[:N] = bias.float()
            bref = self.vec(bp)
        return WMat(Ref("w", self.arena.add(packed)), Ref("w", self.arena.add(plain)) if self.keep_plain else None,
                    bref, N, K, Kpad, bn, cp, ntaps)

    def bn_for_split(self, N: int, n_split: int) -> int:
        for b in (128, 64, 32):
            if n_split % b == 0 and N % b == 0:
                return b
        raise ValueError((N, n_split))

    def conv_w(self, sd, name: str, scale: float = 1.0, m_rows: Optional[int] = None) -> WMat:
        w = sd[name + ".weight"].float() * scale
        wm, taps, cp = packing.conv_weight_matrix(w)
        return self.wmat(wm, sd.get(name + ".bias"), taps, cp, m_rows=m_rows)

    # ---- workspace -----------------------------------------------------------------------
    def f32(self, rows: int, Cc: int) -> F32:
        return F32(Ref("ws", self.pool.alloc(rows * Cc * 4)), rows, Cc)

    def planes(self, rows: int, Cc: int, n: int = 2) -> Planes:
        """n = 2: hi + lo (22-bit operands, three tensor-core passes); n = 1: hi only (11-bit activations against 22-bit
        weights, two passes) -- the token-side operands of the UNet (DESIGN.md section 3)."""
        cp = round_up(Cc, 8)
        off = self.pool.alloc(n * rows * cp * 2)
        return Planes(Ref("ws", off), Ref("ws", off + rows * cp * 2) if n == 2 else None, rows, cp)

    def raw(self, nbytes: int) -> Ref:
        return Ref("ws", self.pool.alloc(nbytes))

    def vt(self, batch: int, Cc: int, ntok: int, n: int = 2) -> VT:
        ld_t = round_up(ntok, 8)
        nb = batch * Cc * ld_t * 2
        off = self.pool.alloc(n * nb)
        return VT(Ref("ws", off), Ref("ws", off + nb) if n == 2 else None, ld_t)

    def attn(self, q: Planes, q_col: int, k: Planes, k_col: int, vt: VT, out: Planes, *, B: int, heads: int, Nq: int,
             Nk: int, mask: Optional[Ref], scale: float, kv_bmod: int = 0):
        self.ops.append(dict(kind="attn", tag=self.tag, q_hi=q.hi, q_lo=q.lo, k_hi=k.hi, k_lo=k.lo, vt_hi=vt.hi, vt_lo=vt.lo,
                             mask=mask, out_hi=out.hi, out_lo=out.lo, B=B, heads=heads, Nq=Nq, Nk=Nk, ldq=q.Cp, ldk=k.Cp,
                             ld_t=vt.ld_t, ldo=out.Cp, q_col=q_col, k_col=k_col, kv_bmod=kv_bmod, impl=self.impl, scale=scale))

    def free(self, *bufs):
        for b in bufs:
            if b is None:
                continue
            r = b.hi if isinstance(b, (Planes, VT)) else (b.ref if isinstance(b, F32) else b)
            self.pool.release(r.off)

    def mark(self, name: str):
        self.marks[name] = len(self.ops)

    # ---- ops -----------------------------------------------------------------------------
    @staticmethod
    def gn_scratch_bytes(B: int) -> int:
        """Bytes of the GroupNorm scratch of a batch of B (layout: csrc/prep.cu): [B][64 blocks][32 groups][2] double
        partials | [B][32][2] float (mean, rstd) | [B] uint tickets."""
        return round_up(B * 64 * 32 * 2 * 8 + B * 32 * 2 * 4 + B * 4, ALIGN)

    def _gn_scratch(self, B: int) -> Ref:
        # The tickets must be ZERO when a GroupNorm starts (they reset themselves): the buffer therefore cannot come from the
        # pool's free list -- a hole there belongs to buffers that other ops rewrite on every run -- and is placed above the
        # high-water mark by finish(), like the split-K scratch (the workspace is zero-initialised once by engine.DeviceProgram).
        self._gn_scr[B] = self.gn_scratch_bytes(B)
        return "GNSCR%d" % B

    def prep(self, mode: int, src0: F32, src1: Optional[F32] = None, gamma: Optional[Ref] = None,
             beta: Optional[Ref] = None, eps: float = 0.0, slope: float = 0.0, B: int = 0, HW: int = 0,
             src_nchw: bool = False, out: Optional[Planes] = None, n: int = 2) -> Planes:
        Cc = src0.C + (src1.C if src1 is not None else 0)
        out = out or self.planes(src0.rows, Cc, n)
        self.ops.append(dict(kind="prep", tag=self.tag, src0=src0.ref, src1=src1.ref if src1 is not None else None,
                             gamma=gamma, beta=beta, out_hi=out.hi, out_lo=out.lo,
                             scratch=self._gn_scratch(B) if mode in (_lib.PREP_GN, _lib.PREP_GN_SILU) else None,
                             rows=src0.rows, c0=src0.C, c1=src1.C if src1 is not None else 0, Cp=out.Cp,
                             B=B, HW=HW, groups=32, mode=mode, eps=eps, slope=slope, src_nchw=int(src_nchw)))
        return out

    def gemm(self, a: Planes, w: WMat, *, B: int, H: int, W: int = 1, taps=((0, 0),), OH: Optional[int] = None,
             OW: Optional[int] = None, sy: int = 1, sx: int = 1, up: int = 0, bmod: int = 0,
             out: Optional[F32] = None, out_planes: Optional[Planes] = None, out_ref: Optional[Ref] = None,
             ldo: Optional[int] = None, out_mode: Optional[int] = None,
             res: Optional[F32] = None, res_ref: Optional[Ref] = None, ld_res: Optional[int] = None,
             rowvec: Optional[Ref] = None, ld_rowvec: int = 0, act: int = _lib.ACT_NONE, alpha: float = 1.0,
             accumulate: bool = False, OHF: Optional[int] = None, osy: int = 1, ooy: int = 0,
             a_off_rows: int = 0, use_bias: bool = True, qkv=None, also_planes: Optional[Planes] = None):
        OH = H if OH is None else OH
        OW = W if OW is None else OW
        assert len(taps) == w.ntaps and a.Cp == w.Cp, (len(taps), w.ntaps, a.Cp, w.Cp)
        M = B * OH * OW
        n_out = w.N // 2 if act == _lib.ACT_GEGLU else w.N
        o = dict(kind="gemm", tag=self.tag, a_hi=a.hi + a_off_rows * a.Cp * 2,
                 a_lo=(a.lo + a_off_rows * a.Cp * 2) if a.lo is not None else None,
                 w_packed=w.packed, w_plain=w.plain, bias=w.bias if use_bias else None, rowvec=rowvec,
                 res=(res.ref if res is not None else res_ref), out=None, out_hi=None, out_lo=None, ws=None,
                 B=B, H=H, W=W, Cp=a.Cp, up=up, bmod=bmod, OH=OH, OW=OW, sy=sy, sx=sx, ntaps=w.ntaps,
                 taps=[(int(dy), int(dx)) for dy, dx in taps], N=w.N, K=w.K, Kpad=w.Kpad, bn=w.bn,
                 ldo=0, ld_res=0, ld_rowvec=ld_rowvec, OHF=OH if OHF is None else OHF, OWF=OW, osy=osy, ooy=ooy,
                 act=act, out_mode=_lib.OUT_F32, accumulate=int(accumulate), splitk=1,
                 impl=self.impl | (_lib.GEMM_STATIC_B if w.packed.region == "w" and self.static_b else 0), alpha=alpha)
        if qkv is not None:          # (planes for columns < n_split, transposed planes for the rest, n_split, tokens per batch)
            pl_, vt_, n_split, tpb = qkv
            assert n_split % w.bn == 0 and n_split % 32 == 0 and pl_.Cp == n_split
            o.update(out_mode=_lib.OUT_QKV, out_hi=pl_.hi, out_lo=pl_.lo, out2_hi=vt_.hi, out2_lo=vt_.lo, ldo=pl_.Cp,
                     n_split=n_split, tok_per_batch=tpb, ld_t=vt_.ld_t)
        elif out_planes is not None:
            o["out_mode"] = _lib.OUT_PLANES
            o["out_hi"], o["out_lo"] = out_planes.hi, out_planes.lo
            o["ldo"] = out_planes.Cp if ldo is None else ldo
        else:
            o["out_mode"] = _lib.OUT_F32 if out_mode is None else out_mode
            o["out"] = out.ref if out is not None else out_ref
            o["ldo"] = (out.C if out is not None else n_out) if ldo is None else ldo
            if also_planes is not None:       # dual output: fp32 + operand planes with the same leading dimension
                assert also_planes.Cp == o["ldo"] and o["out_mode"] == _lib.OUT_F32
                o["out_hi"], o["out_lo"] = also_planes.hi, also_planes.lo
        if o["res"] is not None:
            o["ld_res"] = (res.C if res is not None else n_out) if ld_res is None else ld_res
        # split-K for tiles that cannot fill the machine (deep UNet levels at small batch)
        if self.use_splitk:
            tiles = math.ceil(M / 128) * math.ceil(w.N / w.bn)
            nkb = w.Kpad // 64
            # only worth a second (reduction) kernel when the K loop is long: a short loop is dominated by
            # fixed per-tile costs either way
            if tiles * 2 <= self.n_sm and nkb >= 24:
                sk = min(nkb // 8, max(1, self.n_sm // tiles), 16)
                if sk > 1:
                    o["splitk"] = sk
                    need = sk * round_up(M, 128) * round_up(w.N, w.bn) * 4
                    self.splitk_ws_bytes = max(self.splitk_ws_bytes, need)
                    o["ws"] = "SPLITK"
        self.ops.append(o)
        return o

    def finish(self, io: Dict[str, object], meta=None) -> Plan:
        if self.splitk_ws_bytes:
            # The split-K scratch is used by ops all along the program, so it must not come from the
            # free list (those holes belong to buffers that are live at other points of the schedule):
            # place it above the pool's high-water mark.
            off = round_up(self.pool.peak, ALIGN)
            self.pool.peak = off + round_up(self.splitk_ws_bytes, ALIGN)
            ws = Ref("ws", off)
            for o in self.ops:
                if o.get("ws") == "SPLITK":
                    o["ws"] = ws
        for B, nbytes in sorted(self._gn_scr.items()):
            off = round_up(self.pool.peak, ALIGN)
            self.pool.peak = off + nbytes
            for o in self.ops:
                if o.get("scratch") == "GNSCR%d" % B:
                    o["scratch"] = Ref("ws", off)
        return Plan(self.ops, self.arena.build(), round_up(self.pool.peak, ALIGN), io, dict(self.marks), meta or {})


# ==============================================================================================
# tap helpers
# ==============================================================================================
TAPS_3x3 = tuple((ky - 1, kx - 1) for ky in range(3) for kx in range(3))      # pad 1
TAPS_3x3_ASYM = tuple((ky, kx) for ky in range(3) for kx in range(3))         # F.pad(0,1,0,1) + pad 0 (model.py:88-91)


def taps_1d(k: int, dil: int = 1):
    pad = (k * dil - dil) // 2
    return tuple((j * dil - pad, 0) for j in range(k))


# ==============================================================================================
# UNet (openaimodel.py:837-885)
# ==============================================================================================
def build_unet(sd: Dict[str, torch.Tensor], cfg: dict, latent: Tuple[int, int, int], batch: int, cfg_batched: bool = True,
               ctx_max_len: Tuple[int, ...] = (8, 128), **pk) -> Plan:
    """``batch`` = latent batch B_l.  With ``cfg_batched`` the program evaluates 2*B_l rows per call
    (rows [0,B_l) with the unconditional, [B_l,2B_l) with the conditional conditioning) from one copy
    of x, replacing the two separate apply_model calls of ddim.py:293-296."""
    P = Planner(**pk)
    TP = P.tok_planes
    spec = arch.unet_spec(cfg)
    Cin, T, Fq = latent
    Bl = batch
    Bt = 2 * Bl if cfg_batched else Bl
    mc, ted, emb_ch = cfg["model_channels"], spec.time_embed_dim, spec.emb_ch
    ctx_dims = [c for c in cfg["context_dim"] if c is not None] if cfg.get("context_dim") else []
    film = cfg.get("extra_film_condition_dim")
    io: Dict[str, object] = {}

    # ---------------- persistent I/O + conditioning buffers ----------------
    x_in = F32(P.raw(Bl * Cin * T * Fq * 4), Bl * T * Fq, Cin)          # NCHW [Bl, C, T, F]
    t_in = P.raw(Bt * 8)
    eps_out = P.raw(Bt * cfg["out_channels"] * T * Fq * 4)              # NCHW
    emb = F32(P.raw(Bt * emb_ch * 4), Bt, emb_ch)
    io.update(x=("f32", x_in.ref, (Bl, Cin, T, Fq)), t=("i64", t_in, (Bt,)),
              eps=("f32", eps_out, (Bt, cfg["out_channels"], T, Fq)))
    ctx_bufs, mask_refs = [], []
    for s, dmodel in enumerate(ctx_dims):
        L = ctx_max_len[s] if s < len(ctx_max_len) else ctx_max_len[-1]
        cb = F32(P.raw(Bt * L * dmodel * 4), Bt * L, dmodel)
        mr = P.raw(Bt * L * 4)
        ctx_bufs.append((cb, L)); mask_refs.append(mr)
        io[f"ctx{s}"] = ("f32", cb.ref, (Bt, L, dmodel)); io[f"mask{s}"] = ("f32", mr, (Bt, L))
    if film is not None:
        y_in = F32(P.raw(Bt * film * 4), Bt, film)
        io["y"] = ("f32", y_in.ref, (Bt, film))
    freqs = P.vec(torch.exp(-math.log(10000.0) * torch.arange(mc // 2, dtype=torch.float32) / (mc // 2)))  # util.py:183-187

    # all ResBlock emb projections fused into one GEMM (K4): rows of emb_all = cat_l Linear_l(SiLU(emb))
    res_layers = [l for blk in spec.input_blocks + [spec.middle] + spec.output_blocks for l in blk if l.kind == "res"]
    emb_off, acc = {}, 0
    for l in res_layers:
        emb_off[l.name] = acc; acc += l.cout
    emb_total = acc
    emb_all = F32(P.raw(Bt * emb_total * 4), Bt, emb_total)

    # ---------------- program 0: conditioning (once per call) ----------------
    P.mark("cond_begin")
    kv_cache: Dict[str, tuple] = {}
    ctx_planes = [P.prep(_lib.PREP_COPY, cb) for cb, _ in ctx_bufs]
    for blk in spec.input_blocks + [spec.middle] + spec.output_blocks:
        for l in blk:
            if l.kind == "st" and l.ctx_slot >= 0:
                for d in range(l.depth):
                    n = f"{l.name}.transformer_blocks.{d}.attn2"
                    wkv = torch.cat([sd[n + ".to_k.weight"], sd[n + ".to_v.weight"]], 0).float()
                    wm, taps, cp = packing.conv_weight_matrix(wkv)
                    w = P.wmat(wm, None, taps, cp, bn=P.bn_for_split(2 * l.cin, l.cin))
                    cb, L = ctx_bufs[l.ctx_slot]
                    kpl = P.planes(Bt * L, l.cin, TP)                               # persistent (step-invariant)
                    vtp = P.vt(Bt, l.cin, L, TP)
                    P.gemm(ctx_planes[l.ctx_slot], w, B=1, H=Bt * L, qkv=(kpl, vtp, l.cin, L))
                    kv_cache[n] = (kpl, vtp, L)
    if film is not None:
        yp = P.prep(_lib.PREP_COPY, y_in)
        wf = P.conv_w(sd, "film_emb")
        P.gemm(yp, wf, B=1, H=Bt, out_ref=emb.ref + ted * 4, ldo=emb_ch)        # emb[:, ted:] (openaimodel.py:869-870)
        P.free(yp)
    P.free(*ctx_planes)
    P.mark("cond_end")

    # ---------------- program 1: one UNet evaluation ----------------
    P.mark("step_begin")
    tp = P.planes(Bt, mc)
    P.ops.append(dict(kind="temb", tag=0, t=t_in, freqs=freqs, out_hi=tp.hi, out_lo=tp.lo, B=Bt, dim=mc))
    w0, w2 = P.conv_w(sd, "time_embed.0"), P.conv_w(sd, "time_embed.2")
    e1 = P.planes(Bt, ted)
    P.gemm(tp, w0, B=1, H=Bt, out_planes=e1, act=_lib.ACT_SILU)
    P.gemm(e1, w2, B=1, H=Bt, out_ref=emb.ref, ldo=emb_ch)
    P.free(tp, e1)
    es = P.prep(_lib.PREP_SILU, emb)                                             # emb_layers[0] = SiLU (openaimodel.py:244)
    wemb = torch.cat([sd[l.name + ".emb_layers.1.weight"] for l in res_layers], 0).float()
    bemb = torch.cat([sd[l.name + ".emb_layers.1.bias"] for l in res_layers], 0).float()
    wm, taps, cp = packing.conv_weight_matrix(wemb)
    P.gemm(es, P.wmat(wm, bemb, taps, cp), B=1, H=Bt, out=emb_all)
    P.free(es)

    def resblock(l: arch.Layer, x: F32, x2: Optional[F32], H: int, W: int) -> F32:
        """ResBlock._forward (openaimodel.py:280-300); x2 = skip tensor of the concat (h first, :878-880)."""
        n = l.name
        rows = x.rows
        p1 = P.prep(_lib.PREP_GN_SILU, x, x2, P.vec(sd[n + ".in_layers.0.weight"]), P.vec(sd[n + ".in_layers.0.bias"]),
                    eps=1e-5, B=Bt, HW=H * W)
        h1 = P.f32(rows, l.cout)
        P.gemm(p1, P.conv_w(sd, n + ".in_layers.2", m_rows=rows), B=Bt, H=H, W=W, taps=TAPS_3x3, out=h1,
               rowvec=emb_all.ref + emb_off[n] * 4, ld_rowvec=emb_total)
        P.free(p1)
        p2 = P.prep(_lib.PREP_GN_SILU, h1, None, P.vec(sd[n + ".out_layers.0.weight"]), P.vec(sd[n + ".out_layers.0.bias"]),
                    eps=1e-5, B=Bt, HW=H * W)
        P.free(h1)
        skip = None
        if l.cin != l.cout:
            px = P.prep(_lib.PREP_COPY, x, x2)
            skip = P.f32(rows, l.cout)
            P.gemm(px, P.conv_w(sd, n + ".skip_connection", m_rows=rows), B=Bt, H=H, W=W, out=skip)
            P.free(px)
            res = skip
        else:
            assert x2 is None
            res = x
        out = P.f32(rows, l.cout)
        P.gemm(p2, P.conv_w(sd, n + ".out_layers.3", m_rows=rows), B=Bt, H=H, W=W, taps=TAPS_3x3, out=out, res=res)
        P.free(p2, skip)
        return out

    def attention(nm: str, h: F32, norm: str, heads: int, Cc: int, HW: int, kv, mask: Optional[Ref]) -> F32:
        """x = attn(LN(x)) + x  (attention.py:343-367, 406-409).  The projection GEMMs write Q|K as operand
        planes and V transposed (ALDM_OUT_QKV), which is what the wgmma attention kernel consumes."""
        p = P.prep(_lib.PREP_LN, h, None, P.vec(sd[norm + ".weight"]), P.vec(sd[norm + ".bias"]), eps=1e-5, n=TP)
        ao = P.planes(h.rows, Cc, TP)
        scale = (Cc // heads) ** -0.5
        if kv is None:
            wq = torch.cat([sd[nm + ".to_q.weight"], sd[nm + ".to_k.weight"], sd[nm + ".to_v.weight"]], 0).float()
            wm, taps, cp = packing.conv_weight_matrix(wq)
            qk = P.planes(h.rows, 2 * Cc, TP)
            vtp = P.vt(Bt, Cc, HW, TP)
            P.gemm(p, P.wmat(wm, None, taps, cp, bn=P.bn_for_split(3 * Cc, 2 * Cc)), B=1, H=h.rows, qkv=(qk, vtp, 2 * Cc, HW))
            P.free(p)
            P.attn(qk, 0, qk, Cc, vtp, ao, B=Bt, heads=heads, Nq=HW, Nk=HW, mask=None, scale=scale)
            P.free(qk, vtp)
        else:
            kpl, vtp, L = kv
            q = P.planes(h.rows, Cc, TP)
            P.gemm(p, P.conv_w(sd, nm + ".to_q", m_rows=h.rows), B=1, H=h.rows, out_planes=q)
            P.free(p)
            P.attn(q, 0, kpl, 0, vtp, ao, B=Bt, heads=heads, Nq=HW, Nk=L, mask=mask, scale=scale)
            P.free(q)
        out = P.f32(h.rows, Cc)
        P.gemm(ao, P.conv_w(sd, nm + ".to_out.0", m_rows=h.rows), B=1, H=h.rows, out=out, res=h)
        P.free(ao)
        return out

    def spatial_transformer(l: arch.Layer, x: F32, H: int, W: int) -> F32:
        """SpatialTransformer.forward (attention.py:456-467); tokens are the channels-last rows."""
        n, Cc, HW = l.name, l.cin, H * W
        p = P.prep(_lib.PREP_GN, x, None, P.vec(sd[n + ".norm.weight"]), P.vec(sd[n + ".norm.bias"]), eps=1e-6, B=Bt, HW=HW)
        h = P.f32(x.rows, Cc)
        P.gemm(p, P.conv_w(sd, n + ".proj_in", m_rows=x.rows), B=Bt, H=H, W=W, out=h)
        P.free(p)
        for d in range(l.depth):
            b = f"{n}.transformer_blocks.{d}"
            h2 = attention(b + ".attn1", h, b + ".norm1", l.heads, Cc, HW, None, None); P.free(h); h = h2
            kv = kv_cache.get(b + ".attn2") if l.ctx_slot >= 0 else None
            h2 = attention(b + ".attn2", h, b + ".norm2", l.heads, Cc, HW, kv,
                           mask_refs[l.ctx_slot] if l.ctx_slot >= 0 else None); P.free(h); h = h2
            p = P.prep(_lib.PREP_LN, h, None, P.vec(sd[b + ".norm3.weight"]), P.vec(sd[b + ".norm3.bias"]), eps=1e-5, n=TP)
            wff = sd[b + ".ff.net.0.proj.weight"].float()
            wm, taps, cp = packing.conv_weight_matrix(wff)
            g = P.planes(h.rows, 4 * Cc, TP)
            P.gemm(p, P.wmat(wm, sd[b + ".ff.net.0.proj.bias"], taps, cp, geglu=True, m_rows=h.rows), B=1, H=h.rows, out_planes=g,
                   act=_lib.ACT_GEGLU)
            P.free(p)
            last = d == l.depth - 1
            if last:
                # the last block's output is only ever read as proj_out's operand: write the planes alone (the fp32 copy the
                # dual-output form also stored was dead -- 64 KB per tile through a 32 B/clk store port)
                hp = P.planes(h.rows, Cc)
                P.gemm(g, P.conv_w(sd, b + ".ff.net.2", m_rows=h.rows), B=1, H=h.rows, out_planes=hp, res=h)
                P.free(g, h); h = None
            else:
                h2 = P.f32(h.rows, Cc)
                P.gemm(g, P.conv_w(sd, b + ".ff.net.2", m_rows=h.rows), B=1, H=h.rows, out=h2, res=h)
                P.free(g, h); h = h2
        p = hp
        out = P.f32(x.rows, Cc)
        P.gemm(p, P.conv_w(sd, n + ".proj_out", m_rows=x.rows), B=Bt, H=H, W=W, out=out, res=x)
        P.free(p)
        return out

    keep: set = set()          # ids of skip tensors that must outlive their consumer

    def drop(tns: Optional[F32]):
        if tns is not None and id(tns) not in keep:
            P.free(tns)

    def run_block(layers: List[arch.Layer], h: Optional[F32], H: int, W: int):
        """TimestepEmbedSequential.forward (openaimodel.py:81-103)"""
        for l in layers:
            P.tag += 1
            if l.kind == "conv":            # input_blocks.0.0 : x (NCHW, B_l) -> planes, conv with batch modulo
                p = P.prep(_lib.PREP_COPY, F32(x_in.ref, Bl * H * W, Cin), src_nchw=True, HW=H * W, B=Bl)
                o = P.f32(Bt * H * W, l.cout)
                P.gemm(p, P.conv_w(sd, l.name), B=Bt, H=H, W=W, taps=TAPS_3x3, out=o, bmod=Bl)
                P.free(p); h = o
            elif l.kind == "res":
                o = resblock(l, h, None, H, W); drop(h); h = o
            elif l.kind == "st":
                o = spatial_transformer(l, h, H, W); drop(h); h = o
            elif l.kind == "down":          # Downsample conv3x3 s2 p1 (openaimodel.py:172-179)
                p = P.prep(_lib.PREP_COPY, h)
                o = P.f32(Bt * (H // 2) * (W // 2), l.cout)
                P.gemm(p, P.conv_w(sd, l.name + ".op"), B=Bt, H=H, W=W, taps=TAPS_3x3, OH=H // 2, OW=W // 2, sy=2, sx=2, out=o)
                P.free(p); drop(h); H, W = H // 2, W // 2; h = o
            elif l.kind == "up":            # nearest x2 folded into the gather (openaimodel.py:126-136)
                p = P.prep(_lib.PREP_COPY, h)
                o = P.f32(Bt * 4 * H * W, l.cout)
                P.gemm(p, P.conv_w(sd, l.name + ".conv"), B=Bt, H=2 * H, W=2 * W, taps=TAPS_3x3, up=1, out=o)
                P.free(p); drop(h); H, W = 2 * H, 2 * W; h = o
        return h, H, W

    hs: List[Tuple[F32, int, int]] = []
    H, W = T, Fq
    h: Optional[F32] = None
    for blk in spec.input_blocks:
        h, H, W = run_block(blk, h, H, W)
        hs.append((h, H, W)); keep.add(id(h))
    h, H, W = run_block(spec.middle, h, H, W)
    for blk in spec.output_blocks:
        skip, sH, sW = hs.pop()
        assert (sH, sW) == (H, W)
        first = blk[0]
        assert first.kind == "res" and first.cin == h.C + skip.C
        # the concat tensor is never materialised: the ResBlock reads (h, skip) as two sources
        P.tag += 1
        o = resblock(first, h, skip, H, W)
        drop(h)
        keep.discard(id(skip)); drop(skip)
        h = o
        h, H, W = run_block(blk[1:], h, H, W)
    P.tag += 1
    p = P.prep(_lib.PREP_GN_SILU, h, None, P.vec(sd["out.0.weight"]), P.vec(sd["out.0.bias"]), eps=1e-5, B=Bt, HW=H * W)
    P.free(h)
    P.gemm(p, P.conv_w(sd, "out.2"), B=Bt, H=H, W=W, taps=TAPS_3x3, out_ref=eps_out, out_mode=_lib.OUT_NCHW)
    P.free(p)
    P.mark("step_end")
    return P.finish(io, meta=dict(Bl=Bl, Bt=Bt, latent=latent, emb_ch=emb_ch))


# ==============================================================================================
# VAE (model.py:419-686)
# ==============================================================================================
def _vae_res(P: Planner, sd, n: str, x: F32, B: int, H: int, W: int, cin: int, cout: int) -> F32:
    """ResnetBlock.forward, temb None (model.py:155-175)"""
    p1 = P.prep(_lib.PREP_GN_SILU, x, None, P.vec(sd[n + ".norm1.weight"]), P.vec(sd[n + ".norm1.bias"]), eps=1e-6, B=B, HW=H * W)
    h1 = P.f32(x.rows, cout)
    P.gemm(p1, P.conv_w(sd, n + ".conv1"), B=B, H=H, W=W, taps=TAPS_3x3, out=h1)
    P.free(p1)
    p2 = P.prep(_lib.PREP_GN_SILU, h1, None, P.vec(sd[n + ".norm2.weight"]), P.vec(sd[n + ".norm2.bias"]), eps=1e-6, B=B, HW=H * W)
    P.free(h1)
    res, skip = x, None
    if cin != cout:
        px = P.prep(_lib.PREP_COPY, x)
        skip = P.f32(x.rows, cout)
        P.gemm(px, P.conv_w(sd, n + ".nin_shortcut"), B=B, H=H, W=W, out=skip)
        P.free(px); res = skip
    out = P.f32(x.rows, cout)
    P.gemm(p2, P.conv_w(sd, n + ".conv2"), B=B, H=H, W=W, taps=TAPS_3x3, out=out, res=res)
    P.free(p2, skip)
    return out


def _vae_attn(P: Planner, sd, n: str, x: F32, B: int, HW: int, Cc: int) -> F32:
    """AttnBlock.forward (model.py:204-230): S = q k^T * c^-0.5 (GEMM against device-packed K),
    row softmax, O = P v (GEMM against device-packed V^T), proj_out + x."""
    p = P.prep(_lib.PREP_GN, x, None, P.vec(sd[n + ".norm.weight"]), P.vec(sd[n + ".norm.bias"]), eps=1e-6, B=B, HW=HW)
    q = P.planes(x.rows, Cc)
    k = P.f32(x.rows, Cc)
    v = P.f32(x.rows, Cc)
    P.gemm(p, P.conv_w(sd, n + ".q"), B=1, H=x.rows, out_planes=q)
    P.gemm(p, P.conv_w(sd, n + ".k"), B=1, H=x.rows, out=k)
    P.gemm(p, P.conv_w(sd, n + ".v"), B=1, H=x.rows, out=v)
    P.free(p)
    o = P.planes(x.rows, Cc)
    bn_k, bn_v = packing.choose_bn(HW), packing.choose_bn(Cc)
    Kp_k, Kp_v = round_up(Cc, 64), round_up(HW, 64)
    kpk = P.raw(round_up(HW, bn_k) * Kp_k * 4)
    kpv = P.raw(round_up(Cc, bn_v) * Kp_v * 4)
    plain_k = P.raw(round_up(HW, bn_k) * Kp_k * 4) if P.keep_plain else None
    plain_v = P.raw(round_up(Cc, bn_v) * Kp_v * 4) if P.keep_plain else None
    S = P.f32(HW, HW)
    Pm = P.planes(HW, HW)
    for b in range(B):
        P.ops.append(dict(kind="packb", tag=P.tag, src=k.ref + b * HW * Cc * 4, dst_packed=kpk, dst_plain=plain_k,
                          lds=Cc, transpose=0, N=HW, K=Cc, bn=bn_k))
        wk = WMat(kpk, plain_k, None, HW, Cc, Kp_k, bn_k, q.Cp, 1)
        P.gemm(q, wk, B=1, H=HW, out=S, alpha=float(int(Cc) ** -0.5), a_off_rows=b * HW)
        P.ops.append(dict(kind="softmax", tag=P.tag, x=S.ref, out_hi=Pm.hi, out_lo=Pm.lo, rows=HW, n=HW, scale=1.0))
        P.ops.append(dict(kind="packb", tag=P.tag, src=v.ref + b * HW * Cc * 4, dst_packed=kpv, dst_plain=plain_v,
                          lds=Cc, transpose=1, N=Cc, K=HW, bn=bn_v))
        wv = WMat(kpv, plain_v, None, Cc, HW, Kp_v, bn_v, Pm.Cp, 1)
        ob = Planes(o.hi + b * HW * o.Cp * 2, o.lo + b * HW * o.Cp * 2, HW, o.Cp)
        P.gemm(Pm, wv, B=1, H=HW, out_planes=ob)
    P.free(q, k, v, S, Pm, kpk, kpv, plain_k, plain_v)
    out = P.f32(x.rows, Cc)
    P.gemm(o, P.conv_w(sd, n + ".proj_out"), B=1, H=x.rows, out=out, res=x)
    P.free(o)
    return out


def build_vae_decoder(sd, cfg: dict, latent: Tuple[int, int, int], batch: int, scale_factor: float = 1.0, **pk) -> Plan:
    """decode_first_stage (ddpm.py:922-926) -> AutoencoderKL.decode (autoencoder.py:111-117) -> Decoder.forward
    (model.py:653-686).  in: z NCHW [B, zc, T, F]; out: mel [B, 1, T*2^(L-1), F*2^(L-1)] (== channels-last, C=1)."""
    P = Planner(**pk)
    B = batch
    zc, T, Fq = latent
    ch, cm, nrb = cfg["ch"], cfg["ch_mult"], cfg["num_res_blocks"]
    z_in = F32(P.raw(B * zc * T * Fq * 4), B * T * Fq, zc)
    H, W = T, Fq
    P.mark("begin")
    p = P.prep(_lib.PREP_COPY, z_in, src_nchw=True, HW=H * W, B=B)
    h = P.f32(B * H * W, zc)
    # z / scale_factor is applied BEFORE post_quant_conv (ddpm.py:924): folded into its weights (not the bias)
    P.gemm(p, P.conv_w(sd, "post_quant_conv", scale=1.0 / scale_factor), B=B, H=H, W=W, out=h)
    P.free(p)
    bi = ch * cm[-1]
    p = P.prep(_lib.PREP_COPY, h); P.free(h)
    h = P.f32(B * H * W, bi)
    P.gemm(p, P.conv_w(sd, "decoder.conv_in"), B=B, H=H, W=W, taps=TAPS_3x3, out=h); P.free(p)
    P.tag += 1
    o = _vae_res(P, sd, "decoder.mid.block_1", h, B, H, W, bi, bi); P.free(h); h = o
    P.tag += 1
    o = _vae_attn(P, sd, "decoder.mid.attn_1", h, B, H * W, bi); P.free(h); h = o
    P.tag += 1
    o = _vae_res(P, sd, "decoder.mid.block_2", h, B, H, W, bi, bi); P.free(h); h = o
    for lvl in reversed(range(len(cm))):
        bo = ch * cm[lvl]
        for ib in range(nrb + 1):
            P.tag += 1
            o = _vae_res(P, sd, f"decoder.up.{lvl}.block.{ib}", h, B, H, W, bi, bo); P.free(h); h = o
            bi = bo
        if lvl != 0:                                  # Upsample: nearest x2 + conv3x3 (model.py:53-57)
            P.tag += 1
            p = P.prep(_lib.PREP_COPY, h); P.free(h)
            h = P.f32(B * 4 * H * W, bi)
            P.gemm(p, P.conv_w(sd, f"decoder.up.{lvl}.upsample.conv"), B=B, H=2 * H, W=2 * W, taps=TAPS_3x3, up=1, out=h)
            P.free(p); H, W = 2 * H, 2 * W
    P.tag += 1
    p = P.prep(_lib.PREP_GN_SILU, h, None, P.vec(sd["decoder.norm_out.weight"]), P.vec(sd["decoder.norm_out.bias"]),
               eps=1e-6, B=B, HW=H * W)
    P.free(h)
    mel = F32(P.raw(B * H * W * cfg["out_ch"] * 4), B * H * W, cfg["out_ch"])
    P.gemm(p, P.conv_w(sd, "decoder.conv_out"), B=B, H=H, W=W, taps=TAPS_3x3, out=mel)
    P.free(p)
    P.mark("end")
    io = dict(z=("f32", z_in.ref, (B, zc, T, Fq)), mel=("f32", mel.ref, (B, cfg["out_ch"], H, W)))
    return P.finish(io, meta=dict(B=B, H=H, W=W))


def build_vae_encoder(sd, cfg: dict, mel_hw: Tuple[int, int], batch: int, **pk) -> Plan:
    """encode_first_stage (ddpm.py:941-943) -> AutoencoderKL.encode moments (autoencoder.py:103-109) ->
    Encoder.forward (model.py:519-543).  in: mel [B,1,T,F]; out: moments channels-last [B*h*w, 2*embed]."""
    P = Planner(**pk)
    B = batch
    H, W = mel_hw
    ch, cm, nrb = cfg["ch"], cfg["ch_mult"], cfg["num_res_blocks"]
    x_in = F32(P.raw(B * H * W * cfg["in_channels"] * 4), B * H * W, cfg["in_channels"])
    P.mark("begin")
    p = P.prep(_lib.PREP_COPY, x_in)
    h = P.f32(B * H * W, ch)
    P.gemm(p, P.conv_w(sd, "encoder.conv_in"), B=B, H=H, W=W, taps=TAPS_3x3, out=h); P.free(p)
    in_mult = (1,) + tuple(cm)
    bi = ch
    for lvl in range(len(cm)):
        bi, bo = ch * in_mult[lvl], ch * cm[lvl]
        for ib in range(nrb):
            P.tag += 1
            o = _vae_res(P, sd, f"encoder.down.{lvl}.block.{ib}", h, B, H, W, bi, bo); P.free(h); h = o
            bi = bo
        if lvl != len(cm) - 1:                        # asymmetric pad (0,1,0,1) + conv3x3 s2 p0 (model.py:88-91)
            P.tag += 1
            p = P.prep(_lib.PREP_COPY, h); P.free(h)
            h = P.f32(B * (H // 2) * (W // 2), bi)
            P.gemm(p, P.conv_w(sd, f"encoder.down.{lvl}.downsample.conv"), B=B, H=H, W=W, taps=TAPS_3x3_ASYM,
                   OH=H // 2, OW=W // 2, sy=2, sx=2, out=h)
            P.free(p); H, W = H // 2, W // 2
    P.tag += 1
    o = _vae_res(P, sd, "encoder.mid.block_1", h, B, H, W, bi, bi); P.free(h); h = o
    o = _vae_attn(P, sd, "encoder.mid.attn_1", h, B, H * W, bi); P.free(h); h = o
    o = _vae_res(P, sd, "encoder.mid.block_2", h, B, H, W, bi, bi); P.free(h); h = o
    p = P.prep(_lib.PREP_GN_SILU, h, None, P.vec(sd["encoder.norm_out.weight"]), P.vec(sd["encoder.norm_out.bias"]),
               eps=1e-6, B=B, HW=H * W)
    P.free(h)
    nz = sd["encoder.conv_out.weight"].shape[0]
    h = P.f32(B * H * W, nz)
    P.gemm(p, P.conv_w(sd, "encoder.conv_out"), B=B, H=H, W=W, taps=TAPS_3x3, out=h); P.free(p)
    p = P.prep(_lib.PREP_COPY, h); P.free(h)
    ne = sd["quant_conv.weight"].shape[0]
    mom = F32(P.raw(B * H * W * ne * 4), B * H * W, ne)
    P.gemm(p, P.conv_w(sd, "quant_conv"), B=B, H=H, W=W, out=mom); P.free(p)
    P.mark("end")
    io = dict(mel=("f32", x_in.ref, (B, cfg["in_channels"], mel_hw[0], mel_hw[1])), moments=("f32", mom.ref, (B, H, W, ne)))
    return P.finish(io, meta=dict(B=B, H=H, W=W))


# ==============================================================================================
# HiFi-GAN (hifigan/models.py:96-103,149-165)
# ==============================================================================================
def build_vocoder(sd, cfg: dict, frames: int, batch: int, **pk) -> Plan:
    """in: mel channels-last [B, frames, num_mels] (the memory of the decoder output [B,1,T,F]; the
    reference permutes it to [B,F,T], ddpm.py:932-935); out: waveform [B, 1, L]."""
    P = Planner(**pk)
    B, L = batch, frames
    nm, c0 = cfg["num_mels"], cfg["upsample_initial_channel"]
    nk = len(cfg["resblock_kernel_sizes"])
    mel_in = F32(P.raw(B * L * nm * 4), B * L, nm)
    P.mark("begin")
    p = P.prep(_lib.PREP_COPY, mel_in)
    x = P.f32(B * L, c0)
    P.gemm(p, P.conv_w(sd, "conv_pre"), B=B, H=L, taps=taps_1d(7), out=x); P.free(p)
    ch = c0
    for i, (u, k) in enumerate(zip(cfg["upsample_rates"], cfg["upsample_kernel_sizes"])):
        P.tag += 1
        cin, ch = c0 // (2 ** i), c0 // (2 ** (i + 1))
        Lout = (L - 1) * u - 2 * ((k - u) // 2) + k
        p = P.prep(_lib.PREP_LRELU, x, slope=0.1); P.free(x)
        up = P.f32(B * Lout, ch)
        bias = sd[f"ups.{i}.bias"]
        for ph in packing.conv_transpose_phases(sd[f"ups.{i}.weight"].float(), u):       # K8: polyphase
            nq = (Lout - ph["r"] + u - 1) // u
            w = P.wmat(ph["weight"], bias, len(ph["taps"]), ph["cp"])
            P.gemm(p, w, B=B, H=L, taps=tuple((d, 0) for d in ph["taps"]), OH=nq, out=up, OHF=Lout, osy=u, ooy=ph["r"])
        P.free(p)
        L = Lout
        xs = P.f32(B * L, ch)
        for j, (ks, dil) in enumerate(zip(cfg["resblock_kernel_sizes"], cfg["resblock_dilation_sizes"])):
            P.tag += 1
            r = f"resblocks.{i * nk + j}"
            cur = up
            for m in range(3):                                                          # ResBlock.forward (:96-103)
                p = P.prep(_lib.PREP_LRELU, cur, slope=0.1)
                t1 = P.f32(B * L, ch)
                P.gemm(p, P.conv_w(sd, f"{r}.convs1.{m}"), B=B, H=L, taps=taps_1d(ks, dil[m]), out=t1); P.free(p)
                p = P.prep(_lib.PREP_LRELU, t1, slope=0.1); P.free(t1)
                if m < 2:
                    nxt = P.f32(B * L, ch)
                    P.gemm(p, P.conv_w(sd, f"{r}.convs2.{m}"), B=B, H=L, taps=taps_1d(ks, 1), out=nxt, res=cur)
                    if cur is not up:
                        P.free(cur)
                    cur = nxt
                else:       # last conv of the block: xs (+)= (conv + cur) / num_kernels   (:154-160)
                    P.gemm(p, P.conv_w(sd, f"{r}.convs2.{m}"), B=B, H=L, taps=taps_1d(ks, 1), out=xs, res=cur,
                           alpha=1.0 / nk, accumulate=(j > 0))
                    if cur is not up:
                        P.free(cur)
                P.free(p)
        P.free(up)
        x = xs
    P.tag += 1
    p = P.prep(_lib.PREP_LRELU, x, slope=0.01); P.free(x)                               # F.leaky_relu default (:161)
    wave = F32(P.raw(B * L * 4), B * L, 1)
    P.gemm(p, P.conv_w(sd, "conv_post"), B=B, H=L, taps=taps_1d(7), out=wave, act=_lib.ACT_TANH); P.free(p)
    P.mark("end")
    io = dict(mel=("f32", mel_in.ref, (B, frames, nm)), wave=("f32", wave.ref, (B, 1, L)))
    return P.finish(io, meta=dict(B=B, L=L))


# ==============================================================================================
# AudioMAE token generator: GPT-2 with a KV cache (audiomae_gen/sequence_input.py:110-201,294-325)
# ==============================================================================================
SEQGEN_BN = 32       # N tile of every generator GEMM: the decode passes have M = B <= 8 rows, so the tile count (and with it
                     # the number of SMs streaming the weights) is N / bn; the same packed weights serve prefill and decode


@dataclass
class SeqgenWeights:
    """The generator's packed weight arena, planned once and shared by the plans of every (batch, T5 length)."""
    arena: torch.Tensor
    n_layer: int
    refs: Dict[str, object]


def pack_seqgen_weights(sd: Dict[str, torch.Tensor], **pk) -> SeqgenWeights:
    """Weights of split_seqgen_state_dict / synth.seqgen_state_dict -> tile images.  Two planes everywhere (22-bit
    weights; the activations are two-plane operands as well, DESIGN.md section 1).  ``model.wte`` is not uploaded."""
    P = Planner(**pk)
    n_layer = len([k for k in sd if k.startswith("model.h.") and k.endswith(".ln_1.weight")])
    if n_layer == 0:
        raise KeyError("state dict holds no GPT-2 layers (model.h.<i>.*)")
    C = arch.SEQGEN["n_embd"]

    def lin(w: torch.Tensor, b: torch.Tensor) -> WMat:          # nn.Linear [out, in]
        wm, taps, cp = packing.conv_weight_matrix(w.float())
        return P.wmat(wm, b, taps, cp, bn=SEQGEN_BN)

    def c1d(n: str) -> WMat:                                     # HF Conv1D [in, out]
        wm, taps, cp = packing.conv1d_weight_matrix(sd[n + ".weight"].float())
        return P.wmat(wm, sd[n + ".bias"], taps, cp, bn=SEQGEN_BN)

    r: Dict[str, object] = {
        "wpe": P.vec(sd["model.wpe.weight"]),
        "sos": P.vec(sd["start_of_sequence_tokens.weight"][:2]),
        "eos": P.vec(sd["end_of_sequence_tokens.weight"][:2]),
        "proj0": lin(sd["input_sequence_embed_linear.0.weight"], sd["input_sequence_embed_linear.0.bias"]),
        "proj1": lin(sd["input_sequence_embed_linear.1.weight"], sd["input_sequence_embed_linear.1.bias"]),
        "ln_f": (P.vec(sd["model.ln_f.weight"]), P.vec(sd["model.ln_f.bias"])),
    }
    for i in range(n_layer):
        h = f"model.h.{i}"
        r[f"{i}.ln_1"] = (P.vec(sd[h + ".ln_1.weight"]), P.vec(sd[h + ".ln_1.bias"]))
        r[f"{i}.ln_2"] = (P.vec(sd[h + ".ln_2.weight"]), P.vec(sd[h + ".ln_2.bias"]))
        for n in ("attn.c_attn", "attn.c_proj", "mlp.c_fc", "mlp.c_proj"):
            r[f"{i}.{n}"] = c1d(f"{h}.{n}")
    assert r["wpe"].off >= 0 and C == sd["model.wpe.weight"].shape[1]
    return SeqgenWeights(P.arena.build(), n_layer, r)


def build_seqgen(sd: Optional[Dict[str, torch.Tensor]], batch: int, t5_len: int, gen_len: int = 8,
                 weights: Optional[SeqgenWeights] = None, **pk) -> Plan:
    """Sequence2AudioMAE.generate for one (batch, T5 length L): the prefill pass over P = L + 5 positions, then
    gen_len - 1 decode passes of one position each, all reading and extending per-layer KV caches.

    io: clap [B, 1, 512], t5 [B, L, 1024], t5_mask [B, L] in; tokens [B, gen_len, 768] out.  Marks: "begin",
    "prefill_end", "decode{k}_end" (k = 1 .. gen_len - 1), "end".  The plan references the arena of ``weights``
    (packed from ``sd`` when None): plans of different shapes share one uploaded copy."""
    W = weights if weights is not None else pack_seqgen_weights(sd, **pk)
    P = Planner(**pk)
    B, L = int(batch), int(t5_len)
    C, H = arch.SEQGEN["n_embd"], arch.SEQGEN["n_head"]
    Pn = L + 5
    lmax = Pn + gen_len
    if B < 1 or L < 1 or gen_len < 1:
        raise ValueError(f"seqgen: batch {B}, T5 length {L}, gen_len {gen_len}")
    if Pn > arch.SEQGEN["n_positions"] - gen_len:
        raise ValueError(f"seqgen: {Pn} input positions + {gen_len} generated exceed GPT-2's "
                         f"{arch.SEQGEN['n_positions']} positions (the reference would truncate; T5 inputs are <= 128 tokens)")
    r = W.refs
    eps = arch.SEQGEN["ln_eps"]
    d0, d1 = arch.SEQGEN["input_dims"]
    clap_in = F32(P.raw(B * d0 * 4), B, d0)
    t5_in = F32(P.raw(B * L * d1 * 4), B * L, d1)
    t5_mask = P.raw(B * L * 4)
    tokens = P.raw(B * gen_len * C * 4)
    mask = P.raw(B * lmax * 4)
    seqs = [P.raw(B * lmax * 3 * C * 4) for _ in range(W.n_layer)]        # per-layer KV cache (q | k | v per position)
    x_dec = F32(P.raw(B * C * 4), B, C)                                    # decode input: fed-back token + wpe
    io = dict(clap=("f32", clap_in.ref, (B, 1, d0)), t5=("f32", t5_in.ref, (B, L, d1)), t5_mask=("f32", t5_mask, (B, L)),
              tokens=("f32", tokens, (B, gen_len, C)))

    P.mark("begin")
    P.tag = 0
    x = P.f32(B * Pn, C)
    # the input projections write straight into their rows of the residual stream (rows 1 and [4, 4 + L) of each batch row)
    cp = P.prep(_lib.PREP_COPY, clap_in)
    P.gemm(cp, r["proj0"], B=B, H=1, out_ref=x.ref, ldo=C, OHF=Pn, ooy=1)
    tp = P.prep(_lib.PREP_COPY, t5_in)
    P.gemm(tp, r["proj1"], B=B, H=L, out_ref=x.ref, ldo=C, OHF=Pn, ooy=4)
    P.free(cp, tp)
    P.ops.append(dict(kind="seq_assemble", tag=0, x=x.ref, sos=r["sos"], eos=r["eos"], wpe=r["wpe"], t5_mask=t5_mask, mask=mask,
                      B=B, L=L, lmax=lmax, C=C))

    def gpt2_pass(xin: F32, p0: int, nq: int, k: int, last: bool):
        """GPT2Model.forward over positions [p0, p0 + nq) of every batch row (HF GPT2Block: x += attn(ln_1(x));
        x += mlp(ln_2(x))), then ln_f of the last position -> token k (+ wpe as the next pass's input)."""
        R = B * nq
        cur = xin
        for i in range(W.n_layer):
            P.tag = 1 + i
            a = P.prep(_lib.PREP_LN, cur, None, *r[f"{i}.ln_1"], eps=eps)
            P.gemm(a, r[f"{i}.attn.c_attn"], B=B, H=nq, out_ref=seqs[i], ldo=3 * C, OHF=lmax, ooy=p0)
            P.free(a)
            o = P.planes(R, C)
            P.ops.append(dict(kind="kv_attn", tag=P.tag, seq=seqs[i], mask=mask, out_hi=o.hi, out_lo=o.lo, B=B, heads=H, lmax=lmax,
                              ld_seq=3 * C, p0=p0, nq=nq, ldo=o.Cp, scale=1.0 / 8.0))
            x2 = P.f32(R, C)
            P.gemm(o, r[f"{i}.attn.c_proj"], B=1, H=R, out=x2, res=cur)
            P.free(o)
            if cur is not xin or xin is x:
                P.free(cur)
            a = P.prep(_lib.PREP_LN, x2, None, *r[f"{i}.ln_2"], eps=eps)
            hmid = P.planes(R, arch.SEQGEN["n_inner"])
            P.gemm(a, r[f"{i}.mlp.c_fc"], B=1, H=R, out_planes=hmid, act=_lib.ACT_GELU_TANH)
            P.free(a)
            x3 = P.f32(R, C)
            P.gemm(hmid, r[f"{i}.mlp.c_proj"], B=1, H=R, out=x3, res=x2)
            P.free(hmid, x2)
            cur = x3
        P.tag = 1 + W.n_layer
        P.ops.append(dict(kind="seq_feedback", tag=P.tag, x=cur.ref, gamma=r["ln_f"][0], beta=r["ln_f"][1], wpe=r["wpe"],
                          out=tokens, next=None if last else x_dec.ref, B=B, nq=nq, C=C, pos=p0 + nq - 1, k=k, gen_len=gen_len,
                          eps=eps))
        P.free(cur)

    gpt2_pass(x, 0, Pn, 0, gen_len == 1)
    P.mark("prefill_end")
    for k in range(1, gen_len):
        gpt2_pass(x_dec, Pn + k - 1, 1, k, k == gen_len - 1)
        P.mark(f"decode{k}_end")
    P.mark("end")
    assert P.arena.size == 0, "generator plans reference the shared weight arena only"
    pl = P.finish(io, meta=dict(B=B, L=L, P=Pn, lmax=lmax, gen_len=gen_len, n_layer=W.n_layer))
    pl.arena = W.arena
    return pl


# ==============================================================================================
# Flan-T5 encoder from token ids (FlanT5HiddenState.encode_text, encoders/modules.py:173-198; HF T5EncoderModel)
# ==============================================================================================
T5_BN = 64           # N tile of every encoder GEMM: the same packed weights serve 1 to 1024 rows (N = 1024 gives 16 tiles
                     # per 128-row block; split-K fills the machine for the short-M wo GEMMs)


def t5_relative_position_bucket(relative_position: torch.Tensor, num_buckets: int = 32, max_distance: int = 128) -> torch.Tensor:
    """T5Attention._relative_position_bucket with bidirectional=True (the encoder), restated with the same torch
    operations in the same order (so the same float32 logs decide the boundaries): offset j - i -> bucket in [0, 32)."""
    num_buckets //= 2
    buckets = (relative_position > 0).to(torch.long) * num_buckets
    rp = torch.abs(relative_position)
    max_exact = num_buckets // 2
    is_small = rp < max_exact
    large = max_exact + (torch.log(rp.float() / max_exact) / math.log(max_distance / max_exact)
                         * (num_buckets - max_exact)).to(torch.long)
    large = torch.min(large, torch.full_like(large, num_buckets - 1))
    return buckets + torch.where(is_small, rp, large)


def t5_bias_table(rel_bias: torch.Tensor) -> torch.Tensor:
    """relative_attention_bias.weight [32, heads] -> [heads, 255]: the bias of offsets j - i = -127 .. 127, the only
    thing the attention kernel reads (it indexes column j - i + 127).  Built here once so that no device-side log can
    move a bucket boundary."""
    L = arch.T5["max_len"]
    off = torch.arange(-(L - 1), L)
    b = t5_relative_position_bucket(off, arch.T5["num_buckets"], arch.T5["max_distance"])
    return rel_bias.float()[b].t().contiguous()


@dataclass
class T5Weights:
    """The encoder's weight arena, packed once and shared by the plans of every (batch, length)."""
    arena: torch.Tensor
    n_layer: int
    refs: Dict[str, object]


def pack_t5_weights(sd: Dict[str, torch.Tensor], **pk) -> T5Weights:
    """Weights of split_t5_state_dict / synth.t5_state_dict -> arena: shared.weight in fp32 (the embedding gather), the
    [heads, 255] bias table, the RMSNorm weights, and per block the fused [q | k | v], o, [wi_0 | wi_1] and wo matrices
    as two-plane tile images."""
    P = Planner(**pk)
    n_layer = len([k for k in sd if k.startswith("encoder.block.") and k.endswith(".layer.0.layer_norm.weight")])
    if n_layer == 0:
        raise KeyError("state dict holds no T5 blocks (encoder.block.<i>.*)")

    def lin(ws) -> WMat:
        wm, taps, cp = packing.conv_weight_matrix(torch.cat([w.float() for w in ws], 0))
        return P.wmat(wm, None, taps, cp, bn=T5_BN)

    r: Dict[str, object] = {
        "table": P.vec(sd["shared.weight"]),
        "bias": P.vec(t5_bias_table(sd["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"])),
        "final": P.vec(sd["encoder.final_layer_norm.weight"]),
    }
    for i in range(n_layer):
        b = f"encoder.block.{i}.layer"
        a = f"{b}.0.SelfAttention"
        f = f"{b}.1.DenseReluDense"
        r[f"{i}.ln0"] = P.vec(sd[f"{b}.0.layer_norm.weight"])
        r[f"{i}.ln1"] = P.vec(sd[f"{b}.1.layer_norm.weight"])
        r[f"{i}.qkv"] = lin([sd[f"{a}.q.weight"], sd[f"{a}.k.weight"], sd[f"{a}.v.weight"]])
        r[f"{i}.o"] = lin([sd[f"{a}.o.weight"]])
        r[f"{i}.wi"] = lin([sd[f"{f}.wi_0.weight"], sd[f"{f}.wi_1.weight"]])
        r[f"{i}.wo"] = lin([sd[f"{f}.wo.weight"]])
    return T5Weights(P.arena.build(), n_layer, r)


def build_t5(sd: Optional[Dict[str, torch.Tensor]], batch: int, length: int, weights: Optional[T5Weights] = None,
             **pk) -> Plan:
    """T5EncoderModel(input_ids, attention_mask).last_hidden_state for one (batch B, length L <= 128), in fp32.

    io: ids [B, L] int64, mask [B, L] fp32 (1 = token) in; hidden [B, L, 1024] fp32 out; sat [n_layer] int32, the
    per-block count of gated-GELU values beyond the fp16 range (zero unless a run saturated; the caller reads and
    clears it).  Launches: the embedding, 8 per block (RMSNorm, QKV GEMM, attention, o GEMM + residual, RMSNorm,
    [wi_0 | wi_1] GEMM, gate, wo GEMM + residual) and final_layer_norm.  Marks "begin", "end".  The plan references
    the arena of ``weights`` (packed from ``sd`` when None)."""
    W = weights if weights is not None else pack_t5_weights(sd, **pk)
    P = Planner(**pk)
    B, L = int(batch), int(length)
    if B < 1 or not 1 <= L <= arch.T5["max_len"]:
        raise ValueError(f"t5: batch {B}, length {L} (1 .. {arch.T5['max_len']} tokens)")
    C, H, Dk, Fd = arch.T5["d_model"], arch.T5["n_head"], arch.T5["d_kv"], arch.T5["d_ff"]
    eps = arch.T5["eps"]
    R = B * L
    r = W.refs
    ids = P.raw(R * 8)
    mask = P.raw(R * 4)
    hidden = P.raw(R * C * 4)
    sat = P.raw(W.n_layer * 4)
    io = dict(ids=("i64", ids, (B, L)), mask=("f32", mask, (B, L)), hidden=("f32", hidden, (B, L, C)),
              sat=("i32", sat, (W.n_layer,)))

    P.mark("begin")
    P.tag = 0
    x = P.f32(R, C)
    P.ops.append(dict(kind="t5_embed", tag=0, ids=ids, table=r["table"], out=x.ref, rows=R, vocab=arch.T5["vocab"], C=C))

    def rms(src: F32, gamma: Ref) -> Planes:
        out = P.planes(R, C)
        P.ops.append(dict(kind="t5_rmsnorm", tag=P.tag, x=src.ref, gamma=gamma, out_hi=out.hi, out_lo=out.lo, out_f32=None,
                          rows=R, C=C, ldo=out.Cp, eps=eps))
        return out

    for i in range(W.n_layer):
        P.tag = 1 + i
        # T5LayerSelfAttention: x + o(attn(rms(x)))
        a = rms(x, r[f"{i}.ln0"])
        qkv = P.f32(R, 3 * C)
        P.gemm(a, r[f"{i}.qkv"], B=1, H=R, out=qkv)
        P.free(a)
        o = P.planes(R, C)
        P.ops.append(dict(kind="t5_attn", tag=P.tag, qkv=qkv.ref, bias=r["bias"], mask=mask, out_hi=o.hi, out_lo=o.lo, B=B, L=L,
                          heads=H, d_kv=Dk, C=C, ld_qkv=3 * C, ldo=o.Cp))
        P.free(qkv)
        x2 = P.f32(R, C)
        P.gemm(o, r[f"{i}.o"], B=1, H=R, out=x2, res=x)
        P.free(o, x)
        # T5LayerFF (gated-gelu): x + wo(gelu_new(wi_0(rms(x))) * wi_1(rms(x)))
        a = rms(x2, r[f"{i}.ln1"])
        hf = P.f32(R, 2 * Fd)
        P.gemm(a, r[f"{i}.wi"], B=1, H=R, out=hf)
        P.free(a)
        g = P.planes(R, Fd)
        P.ops.append(dict(kind="t5_gate", tag=P.tag, x=hf.ref, out_hi=g.hi, out_lo=g.lo, sat=sat + 4 * i, rows=R, F=Fd,
                          ld_x=2 * Fd, ldo=g.Cp))
        P.free(hf)
        x = P.f32(R, C)
        P.gemm(g, r[f"{i}.wo"], B=1, H=R, out=x, res=x2)
        P.free(g, x2)
    P.tag = 1 + W.n_layer
    P.ops.append(dict(kind="t5_rmsnorm", tag=P.tag, x=x.ref, gamma=r["final"], out_hi=None, out_lo=None, out_f32=hidden,
                      rows=R, C=C, ldo=C, eps=eps))
    P.free(x)
    P.mark("end")
    assert P.arena.size == 0, "encoder plans reference the shared weight arena only"
    pl = P.finish(io, meta=dict(B=B, L=L, n_layer=W.n_layer))
    pl.arena = W.arena
    return pl


# ==============================================================================================
# CLAP text embedding from token ids (CLAP.get_text_embedding, clap/open_clip/model.py:656-663, 730-750; HF RobertaModel)
# ==============================================================================================
CLAP_BN = 64         # N tile of every encoder GEMM: the same packed weights serve plans of 2 to 4096 rows
FP16_MAX = 65504.0


@dataclass
class ClapWeights:
    """The text branch's weight arena, packed once and shared by the plans of every (batch, length); ``bounds``: name ->
    the largest magnitude a value entering that operand plane can take (pack_clap_weights)."""
    arena: torch.Tensor
    n_layer: int
    refs: Dict[str, object]
    bounds: Dict[str, float]


def clap_plane_bounds(sd: Dict[str, torch.Tensor], n_layer: int) -> Dict[str, float]:
    """Bounds, from the weights alone, on every value the encoder writes into fp16 operand planes.  RoBERTa is post-LN, so
    each such value is a LayerNorm output y = gamma * z + beta with ||z||_2 <= sqrt(C) (z has zero mean and unit variance
    up to eps), a linear function of one, or a convex combination / GELU of those:
      LayerNorm output            |y_c| <= |gamma_c| sqrt(C) + |beta_c|
      u = W y + b (v, and the     |u_n| <= ||w_n * gamma||_2 sqrt(C) + |w_n . beta| + |b_n|  (Cauchy-Schwarz)
      intermediate pre-activation)
      attention output            a mix of rows of v with weights summing to 1: bounded by v's bound
      GELU output                 |gelu(u)| <= |u|
    name (the HF module) -> bound, in float64."""
    C = arch.CLAP_TEXT["d_model"]
    rc = math.sqrt(C)
    d = lambda n: sd[n].double()

    def ln(n):
        return float((d(n + ".weight").abs() * rc + d(n + ".bias").abs()).max())

    def lin(n, ln_name):
        w, b = d(n + ".weight"), d(n + ".bias")
        g, be = d(ln_name + ".weight"), d(ln_name + ".bias")
        return float(((w * g[None]).norm(dim=1) * rc + (w @ be).abs() + b.abs()).max())

    prev = "text_branch.embeddings.LayerNorm"
    out = {prev: ln(prev)}
    for i in range(n_layer):
        b = f"text_branch.encoder.layer.{i}"
        out[f"{b}.attention.self.value"] = lin(f"{b}.attention.self.value", prev)
        out[f"{b}.attention.output.LayerNorm"] = ln(f"{b}.attention.output.LayerNorm")
        out[f"{b}.intermediate.dense"] = lin(f"{b}.intermediate.dense", f"{b}.attention.output.LayerNorm")
        prev = f"{b}.output.LayerNorm"
        out[prev] = ln(prev)
    return out


def pack_clap_weights(sd: Dict[str, torch.Tensor], **pk) -> ClapWeights:
    """Weights of split_clap_text_state_dict / synth.clap_text_state_dict -> arena: the word, position and token-type
    embeddings in fp32 (the embedding gather), LayerNorm vectors, per block the fused [query | key | value], attention
    output, intermediate and output matrices (with biases) as two-plane tile images, and the pooler / projection in fp32,
    transposed ([in, out]) for the head kernel.  Raises ValueError, naming the layer, if a value entering an operand plane
    could exceed the fp16 range (clap_plane_bounds): the planes would clamp it, so such weights are refused here rather
    than counted at run time."""
    n_layer = len([k for k in sd if k.startswith("text_branch.encoder.layer.") and k.endswith(".attention.output.LayerNorm.weight")])
    if n_layer == 0:
        raise KeyError("state dict holds no RoBERTa layers (text_branch.encoder.layer.<i>.*)")
    bounds = clap_plane_bounds(sd, n_layer)
    for name, v in bounds.items():
        if not v <= FP16_MAX:
            raise ValueError(f"CLAP text branch: values entering the fp16 operand planes after {name} can reach {v:.6g}, "
                             f"beyond the fp16 range ({FP16_MAX:g}); these weights cannot be encoded without clamping")
    P = Planner(**pk)

    def lin(names) -> WMat:
        w = torch.cat([sd[n + ".weight"].float() for n in names], 0)
        wm, taps, cp = packing.conv_weight_matrix(w)
        return P.wmat(wm, torch.cat([sd[n + ".bias"].float() for n in names], 0), taps, cp, bn=CLAP_BN)

    e = "text_branch.embeddings"
    vec2 = lambda n: (P.vec(sd[n + ".weight"]), P.vec(sd[n + ".bias"]))
    r: Dict[str, object] = {
        "word": P.vec(sd[f"{e}.word_embeddings.weight"]),
        "pos": P.vec(sd[f"{e}.position_embeddings.weight"]),
        "type": P.vec(sd[f"{e}.token_type_embeddings.weight"][0]),
        "ln_emb": vec2(f"{e}.LayerNorm"),
        "wp_t": P.vec(sd["text_branch.pooler.dense.weight"].float().t()), "bp": P.vec(sd["text_branch.pooler.dense.bias"]),
        "w1_t": P.vec(sd["text_projection.0.weight"].float().t()), "b1": P.vec(sd["text_projection.0.bias"]),
        "w2_t": P.vec(sd["text_projection.2.weight"].float().t()), "b2": P.vec(sd["text_projection.2.bias"]),
    }
    for i in range(n_layer):
        b = f"text_branch.encoder.layer.{i}"
        r[f"{i}.qkv"] = lin([f"{b}.attention.self.{n}" for n in ("query", "key", "value")])
        r[f"{i}.o"] = lin([f"{b}.attention.output.dense"])
        r[f"{i}.ln1"] = vec2(f"{b}.attention.output.LayerNorm")
        r[f"{i}.inter"] = lin([f"{b}.intermediate.dense"])
        r[f"{i}.out"] = lin([f"{b}.output.dense"])
        r[f"{i}.ln2"] = vec2(f"{b}.output.LayerNorm")
    return ClapWeights(P.arena.build(), n_layer, r, bounds)


def build_clap_text(sd: Optional[Dict[str, torch.Tensor]], batch: int, length: int, weights: Optional[ClapWeights] = None,
                    **pk) -> Plan:
    """CLAP.get_text_embedding(input_ids, attention_mask) for one (batch B, length L <= 512), in fp32.  The caller plans on
    the longest valid row (clap.effective_length), not on the tokenizer's 512: the embedding reads token 0 of the last
    layer only, and padded keys have probability 0 in every layer.

    io: ids [B, L] int64, mask [B, L] fp32 (1 = token) in; embed [B, 512] fp32 out.  Launches: the embedding, its
    LayerNorm, 8 per block (QKV GEMM, attention, attention-output GEMM + residual, LayerNorm, intermediate GEMM, GELU,
    output GEMM + residual, LayerNorm) and the head.  Marks "begin", "end".  The plan references the arena of
    ``weights`` (packed from ``sd`` when None)."""
    W = weights if weights is not None else pack_clap_weights(sd, **pk)
    P = Planner(**pk)
    B, L = int(batch), int(length)
    if B < 1 or not 1 <= L <= arch.CLAP_TEXT["max_len"]:
        raise ValueError(f"clap: batch {B}, length {L} (1 .. {arch.CLAP_TEXT['max_len']} tokens)")
    A = arch.CLAP_TEXT
    C, H, Fd, Pj, eps = A["d_model"], A["n_head"], A["d_ff"], A["joint_dim"], A["eps"]
    R = B * L
    r = W.refs
    ids = P.raw(R * 8)
    mask = P.raw(R * 4)
    embed = P.raw(B * Pj * 4)
    io = dict(ids=("i64", ids, (B, L)), mask=("f32", mask, (B, L)), embed=("f32", embed, (B, Pj)))

    def layernorm(src: F32, g) -> Tuple[F32, Planes]:
        y, a = P.f32(R, C), P.planes(R, C)
        P.ops.append(dict(kind="clap_ln", tag=P.tag, x=src.ref, gamma=g[0], beta=g[1], out_f32=y.ref, out_hi=a.hi, out_lo=a.lo,
                          rows=R, C=C, ldo=a.Cp, eps=eps))
        return y, a

    P.mark("begin")
    P.tag = 0
    x0 = P.f32(R, C)
    P.ops.append(dict(kind="clap_embed", tag=0, ids=ids, word=r["word"], pos=r["pos"], type=r["type"], out=x0.ref, B=B, L=L,
                      vocab=A["vocab"], n_pos=A["max_positions"], C=C, pad=A["pad_id"]))
    x, a = layernorm(x0, r["ln_emb"])
    P.free(x0)
    for i in range(W.n_layer):
        P.tag = 1 + i
        # RobertaAttention: x = LN(x + dense(attn(x)))
        qkv = P.f32(R, 3 * C)
        P.gemm(a, r[f"{i}.qkv"], B=1, H=R, out=qkv)
        P.free(a)
        o = P.planes(R, C)
        P.ops.append(dict(kind="clap_attn", tag=P.tag, qkv=qkv.ref, mask=mask, out_hi=o.hi, out_lo=o.lo, B=B, L=L, heads=H, C=C,
                          ld_qkv=3 * C, ldo=o.Cp))
        P.free(qkv)
        y = P.f32(R, C)
        P.gemm(o, r[f"{i}.o"], B=1, H=R, out=y, res=x)
        P.free(o, x)
        x2, a2 = layernorm(y, r[f"{i}.ln1"])
        P.free(y)
        # RobertaIntermediate + RobertaOutput: x = LN(x + dense(gelu(dense(x))))
        hm = P.f32(R, Fd)
        P.gemm(a2, r[f"{i}.inter"], B=1, H=R, out=hm)
        P.free(a2)
        g = P.planes(R, Fd)
        P.ops.append(dict(kind="clap_gelu", tag=P.tag, x=hm.ref, out_hi=g.hi, out_lo=g.lo, rows=R, F=Fd, ld_x=Fd, ldo=g.Cp))
        P.free(hm)
        y = P.f32(R, C)
        P.gemm(g, r[f"{i}.out"], B=1, H=R, out=y, res=x2)
        P.free(g, x2)
        x, a = layernorm(y, r[f"{i}.ln2"])
        P.free(y)
    P.tag = 1 + W.n_layer
    P.ops.append(dict(kind="clap_head", tag=P.tag, x=x.ref, wp_t=r["wp_t"], bp=r["bp"], w1_t=r["w1_t"], b1=r["b1"],
                      w2_t=r["w2_t"], b2=r["b2"], out=embed, B=B, L=L, C=C, P=Pj))
    P.free(x, a)
    P.mark("end")
    assert P.arena.size == 0, "encoder plans reference the shared weight arena only"
    pl = P.finish(io, meta=dict(B=B, L=L, n_layer=W.n_layer))
    pl.arena = W.arena
    return pl


# ==============================================================================================
# CLAP audio embedding from the waveform (CLAP.get_audio_embedding, clap/open_clip/model.py:752-777; HTSAT-base,
# clap/open_clip/htsat.py; the resample and truncation of encoders/modules.py:689-716)
# ==============================================================================================
HTSAT_GELU_ROWS = 32768      # rows per clap_gelu launch (its grid's y dimension holds at most 65535)


def htsat_resample_taps(orig_freq: int = 16000, new_freq: int = 48000, lowpass_filter_width: int = 6,
                        rolloff: float = 0.99) -> torch.Tensor:
    """torchaudio.functional.resample's sinc_interp_hann kernel (functional.py _get_sinc_resample_kernel) for a float32
    waveform, computed as torchaudio computes it (in float32): [new / gcd, 2 width + orig / gcd] -- [3, 15] for 16 -> 48 kHz.
    Output sample new * q + j = sum_m taps[j, m] x[orig * q + m - width] (zero padding)."""
    g = math.gcd(orig_freq, new_freq)
    orig, new = orig_freq // g, new_freq // g
    base = min(orig, new) * rolloff
    width = math.ceil(lowpass_filter_width * orig / base)
    dt = torch.float32
    idx = torch.arange(-width, width + orig, dtype=dt)[None, None] / orig
    t = torch.arange(0, -new, -1, dtype=dt)[:, None, None] / new + idx
    t *= base
    t = t.clamp_(-lowpass_filter_width, lowpass_filter_width)
    window = torch.cos(t * math.pi / lowpass_filter_width / 2) ** 2
    t *= math.pi
    k = torch.where(t == 0, torch.tensor(1.0).to(t), t.sin() / t)
    k *= window * (base / orig)
    return k[:, 0].contiguous()


def htsat_bicubic(T: int, out: int = 1024) -> Tuple[torch.Tensor, torch.Tensor]:
    """The time-axis weights of F.interpolate(mode="bicubic", align_corners=True) from T to ``out`` frames, in float32 as
    upsample_bicubic2d computes them (the kernel does the same arithmetic): source x = ((T - 1) / (out - 1)) t, i0 =
    floor(x), t = x - i0, cubic-convolution weights with A = -0.75.  -> (rows [out, 4] clamped to [0, T), weights [out, 4])."""
    scale = torch.tensor((T - 1) / 1.0, dtype=torch.float32) / torch.tensor(out - 1, dtype=torch.float32)
    x = scale * torch.arange(out, dtype=torch.float32)
    i0 = torch.clamp(torch.floor(x).long(), max=T - 1)
    t = torch.clamp(x - i0.float(), 0.0, 1.0)
    A = -0.75

    def c1(v):
        return ((A + 2.0) * v - (A + 3.0)) * v * v + 1.0

    def c2(v):
        return ((A * v - 5.0 * A) * v + 8.0 * A) * v - 4.0 * A

    t2 = 1.0 - t
    w = torch.stack([c2(t + 1.0), c1(t), c1(t2), c2(t2 + 1.0)], 1)
    rows = (i0[:, None] + torch.arange(-1, 3)[None]).clamp(0, T - 1)
    return rows, w


def htsat_relative_position_index(window: int = 8) -> torch.Tensor:
    """WindowAttention.relative_position_index (htsat.py:384-401): [w^2, w^2], the row of the [(2w - 1)^2, heads] bias
    table for query i, key j of a window: (dy + w - 1) (2w - 1) + (dx + w - 1)."""
    yy, xx = torch.meshgrid(torch.arange(window), torch.arange(window), indexing="ij")
    c = torch.stack([yy.reshape(-1), xx.reshape(-1)])
    rel = c[:, :, None] - c[:, None, :] + (window - 1)
    return rel[0] * (2 * window - 1) + rel[1]


def htsat_shift_mask(R: int, window: int = 8, shift: int = 4) -> torch.Tensor:
    """SwinTransformerBlock.attn_mask (htsat.py:545-576) of a shifted block on an R x R grid: [(R / w)^2, w^2, w^2], 0
    where query and key come from the same region of the rolled grid, -100 elsewhere."""
    lab = torch.zeros(R, R)
    cnt = 0
    for hs in (slice(0, -window), slice(-window, -shift), slice(-shift, None)):
        for ws in (slice(0, -window), slice(-window, -shift), slice(-shift, None)):
            lab[hs, ws] = cnt
            cnt += 1
    m = lab.reshape(R // window, window, R // window, window).permute(0, 2, 1, 3).reshape(-1, window * window)
    d = m[:, None, :] - m[:, :, None]
    return torch.where(d != 0, torch.tensor(-100.0), torch.tensor(0.0))


def htsat_block_shift(R: int, j: int) -> int:
    """Shift of block j on an R x R grid: window // 2 on odd blocks, 0 where the grid is no larger than a window."""
    w = arch.CLAP_AUDIO["window"]
    return 0 if R <= w or j % 2 == 0 else w // 2


def htsat_depths(sd: Dict[str, torch.Tensor], prefix: str = "") -> Tuple[int, ...]:
    """Swin blocks per stage of an audio branch whose keys are ``prefix + "audio_branch.layers.<i>.blocks.<j>.*"``.
    Raises KeyError when a stage has none."""
    out = []
    for i in range(len(arch.CLAP_AUDIO["depths"])):
        pre = f"{prefix}audio_branch.layers.{i}.blocks."
        out.append(len({k[len(pre):].split(".")[0] for k in sd if k.startswith(pre)}))
    if 0 in out:
        raise KeyError(f"no HTSAT blocks for some stage under {prefix}audio_branch.layers.<i>.blocks. (found {out})")
    return tuple(out)


@dataclass
class ClapAudioWeights:
    """The audio branch's weight arena, packed once and shared by the plans of every (n, L, sr); ``bounds``: name ->
    the largest magnitude a value entering that operand plane can take (clap_audio_plane_bounds)."""
    arena: torch.Tensor
    depths: Tuple[int, ...]
    refs: Dict[str, object]
    bounds: Dict[str, float]


def clap_audio_plane_bounds(sd: Dict[str, torch.Tensor], depths) -> Dict[str, float]:
    """Bounds, from the weights alone, on every value the encoder writes into fp16 operand planes.  Each is a LayerNorm
    output y = gamma * z + beta with ||z||_2 <= sqrt(C), a linear function of one, or a convex combination / GELU of those:
      LayerNorm output (norm1, norm2, downsample.norm)    |y_c| <= |gamma_c| sqrt(C) + |beta_c|
      v = W_v y + b_v, fc1 pre-activation u = W y + b     |u_n| <= ||w_n * gamma||_2 sqrt(C) + |w_n . beta| + |b_n|
      attention output                                    a mix of rows of v with weights summing to 1: v's bound
      GELU output (fc2's operand)                         |gelu(u)| <= |u|
    name (the reference's module) -> bound, in float64."""
    d = lambda n: sd[n].double()

    def ln(n):
        g, b = d(n + ".weight"), d(n + ".bias")
        return float((g.abs() * math.sqrt(g.numel()) + b.abs()).max())

    def lin(w, b, ln_name):
        g, be = d(ln_name + ".weight"), d(ln_name + ".bias")
        return float(((w * g[None]).norm(dim=1) * math.sqrt(g.numel()) + (w @ be).abs() + b.abs()).max())

    out = {}
    E = arch.CLAP_AUDIO["embed_dim"]
    for i, depth in enumerate(depths):
        C = E * 2 ** i
        for j in range(depth):
            b = f"audio_branch.layers.{i}.blocks.{j}"
            out[f"{b}.norm1"] = ln(f"{b}.norm1")
            out[f"{b}.attn.qkv (v)"] = lin(d(f"{b}.attn.qkv.weight")[2 * C:], d(f"{b}.attn.qkv.bias")[2 * C:], f"{b}.norm1")
            out[f"{b}.norm2"] = ln(f"{b}.norm2")
            out[f"{b}.mlp.fc1"] = lin(d(f"{b}.mlp.fc1.weight"), d(f"{b}.mlp.fc1.bias"), f"{b}.norm2")
        if i < len(depths) - 1:
            out[f"audio_branch.layers.{i}.downsample.norm"] = ln(f"audio_branch.layers.{i}.downsample.norm")
    return out


def pack_clap_audio_weights(sd: Dict[str, torch.Tensor], **pk) -> ClapAudioWeights:
    """Weights of model.split_clap_audio_state_dict / synth.clap_audio_state_dict -> arena: the front end (resample taps,
    melW, bn0), the patch embedding, per block LayerNorm vectors, the qkv / proj / fc1 / fc2 matrices (with biases) as
    two-plane tile images and the relative-position bias gathered to [heads, 64, 64], per shifted stage the window mask,
    per PatchMerging its LayerNorm and reduction, and the final LayerNorm and audio_projection in fp32 ([in, out]) for the
    head kernel.  Raises ValueError, naming the layer, if a value entering an operand plane could exceed the fp16 range
    (clap_audio_plane_bounds)."""
    depths = htsat_depths(sd)
    bounds = clap_audio_plane_bounds(sd, depths)
    for name, v in bounds.items():
        if not v <= FP16_MAX:
            raise ValueError(f"CLAP audio branch: values entering the fp16 operand planes after {name} can reach {v:.6g}, "
                             f"beyond the fp16 range ({FP16_MAX:g}); these weights cannot be encoded without clamping")
    A = arch.CLAP_AUDIO
    P = Planner(**pk)

    def lin(n, bias=True) -> WMat:
        wm, taps, cp = packing.conv_weight_matrix(sd[n + ".weight"].float())
        return P.wmat(wm, sd[n + ".bias"].float() if bias else None, taps, cp, bn=CLAP_BN)

    a = "audio_branch"
    vec2 = lambda n: (P.vec(sd[n + ".weight"]), P.vec(sd[n + ".bias"]))
    rpi = htsat_relative_position_index(A["window"]).reshape(-1)
    r: Dict[str, object] = {
        "taps": P.vec(htsat_resample_taps()),
        "melW": P.vec(sd[f"{a}.logmel_extractor.melW"]),
        "bn": tuple(P.vec(sd[f"{a}.bn0.{k}"]) for k in ("running_mean", "running_var", "weight", "bias")),
        "patch_w": P.vec(sd[f"{a}.patch_embed.proj.weight"].reshape(A["embed_dim"], -1)),
        "patch_b": P.vec(sd[f"{a}.patch_embed.proj.bias"]),
        "patch_ln": vec2(f"{a}.patch_embed.norm"),
        "norm": vec2(f"{a}.norm"),
        "w1_t": P.vec(sd["audio_projection.0.weight"].float().t()), "b1": P.vec(sd["audio_projection.0.bias"]),
        "w2_t": P.vec(sd["audio_projection.2.weight"].float().t()), "b2": P.vec(sd["audio_projection.2.bias"]),
    }
    R = A["spec_size"] // A["patch"]
    for i, depth in enumerate(depths):
        if R > A["window"]:
            r[f"{i}.mask"] = P.vec(htsat_shift_mask(R, A["window"], A["window"] // 2))
        for j in range(depth):
            b = f"{a}.layers.{i}.blocks.{j}"
            tab = sd[f"{b}.attn.relative_position_bias_table"].float()
            r[f"{i}.{j}.bias"] = P.vec(tab[rpi].reshape(A["window"] ** 2, A["window"] ** 2, -1).permute(2, 0, 1))
            r[f"{i}.{j}.ln1"] = vec2(f"{b}.norm1")
            r[f"{i}.{j}.qkv"] = lin(f"{b}.attn.qkv")
            r[f"{i}.{j}.proj"] = lin(f"{b}.attn.proj")
            r[f"{i}.{j}.ln2"] = vec2(f"{b}.norm2")
            r[f"{i}.{j}.fc1"] = lin(f"{b}.mlp.fc1")
            r[f"{i}.{j}.fc2"] = lin(f"{b}.mlp.fc2")
        if i < len(depths) - 1:
            r[f"{i}.merge_ln"] = vec2(f"{a}.layers.{i}.downsample.norm")
            r[f"{i}.reduction"] = lin(f"{a}.layers.{i}.downsample.reduction", bias=False)
        R //= 2
    return ClapAudioWeights(P.arena.build(), depths, r, bounds)


def build_clap_audio(sd: Optional[Dict[str, torch.Tensor]], n: int, length: int, sampling_rate: int,
                     weights: Optional[ClapAudioWeights] = None, **pk) -> Plan:
    """CLAP.get_audio_embedding of n clips of ``length`` samples at ``sampling_rate`` (16 000: resampled to 48 kHz on the
    fly; 48 000), truncated to 480 000 samples at 48 kHz, in fp32.

    io: wav [n, L] fp32 in; embed [n, 512] fp32 out.  Launches: the log-mel front end, the patch embedding, per Swin block
    LN1, the QKV GEMM, window attention, the proj GEMM + residual, LN2, the fc1 GEMM, erf-GELU (one launch per 32768 rows),
    the fc2 GEMM + residual; per PatchMerging its gather + LayerNorm and the reduction GEMM; the head.  Marks "begin",
    "end".  The plan references the arena of ``weights`` (packed from ``sd`` when None)."""
    W = weights if weights is not None else pack_clap_audio_weights(sd, **pk)
    A = arch.CLAP_AUDIO
    n, L, sr = int(n), int(length), int(sampling_rate)
    if sr not in (16000, 48000):
        raise ValueError(f"clap audio: sampling rate {sr} (16000 or 48000)")
    up = 48000 // sr
    L48 = min(up * L, A["max_samples"])
    if n < 1 or L48 <= A["n_fft"] // 2:
        raise ValueError(f"clap audio: {n} clips of {L} samples at {sr} Hz: the 48 kHz signal needs more than "
                         f"{A['n_fft'] // 2} samples (reflect padding)")
    T = L48 // A["hop"] + 1
    P = Planner(**pk)
    r = W.refs
    E, Hd, win, eps = A["embed_dim"], A["head_dim"], A["window"], A["eps"]
    wav = P.raw(n * L * 4)
    embed = P.raw(n * A["joint_dim"] * 4)
    io = dict(wav=("f32", wav, (n, L)), embed=("f32", embed, (n, A["joint_dim"])))

    P.mark("begin")
    P.tag = 0
    mel = P.raw(n * T * A["n_mels"] * 4)
    bm, bv, bw, bb = r["bn"]
    P.ops.append(dict(kind="htsat_logmel", tag=0, wav=wav, taps=r["taps"] if up == 3 else None, melW=r["melW"], bn_mean=bm,
                      bn_var=bv, bn_w=bw, bn_b=bb, out=mel, n=n, L=L, up=up, L48=L48, T=T, eps=A["bn_eps"]))
    R = A["spec_size"] // A["patch"]
    x = P.f32(n * R * R, E)
    P.ops.append(dict(kind="htsat_patch", tag=0, mel=mel, w=r["patch_w"], bias=r["patch_b"], gamma=r["patch_ln"][0],
                      beta=r["patch_ln"][1], out=x.ref, n=n, T=T, eps=eps))
    P.free(mel)
    blk = 0
    for i, depth in enumerate(W.depths):
        C, H = E * 2 ** i, A["heads"][i]
        rows = n * R * R
        for j in range(depth):
            blk += 1
            P.tag = blk
            shift = htsat_block_shift(R, j)
            # x = x + proj(WindowAttention(norm1(x)))
            a = P.prep(_lib.PREP_LN, x, None, *r[f"{i}.{j}.ln1"], eps=eps)
            qkv = P.f32(rows, 3 * C)
            P.gemm(a, r[f"{i}.{j}.qkv"], B=1, H=rows, out=qkv)
            P.free(a)
            o = P.planes(rows, C)
            P.ops.append(dict(kind="htsat_attn", tag=P.tag, qkv=qkv.ref, bias=r[f"{i}.{j}.bias"],
                              mask=r[f"{i}.mask"] if shift else None, out_hi=o.hi, out_lo=o.lo, n=n, R=R, shift=shift,
                              heads=H, head_dim=Hd, C=C, ld_qkv=3 * C, ldo=o.Cp, scale=Hd ** -0.5))
            P.free(qkv)
            y = P.f32(rows, C)
            P.gemm(o, r[f"{i}.{j}.proj"], B=1, H=rows, out=y, res=x)
            P.free(o, x)
            x = y
            # x = x + fc2(gelu(fc1(norm2(x))))
            a = P.prep(_lib.PREP_LN, x, None, *r[f"{i}.{j}.ln2"], eps=eps)
            Fd = A["mlp_ratio"] * C
            hm = P.f32(rows, Fd)
            P.gemm(a, r[f"{i}.{j}.fc1"], B=1, H=rows, out=hm)
            P.free(a)
            g = P.planes(rows, Fd)
            for r0 in range(0, rows, HTSAT_GELU_ROWS):
                nr = min(HTSAT_GELU_ROWS, rows - r0)
                P.ops.append(dict(kind="clap_gelu", tag=P.tag, x=hm.ref + r0 * Fd * 4, out_hi=g.hi + r0 * g.Cp * 2,
                                  out_lo=g.lo + r0 * g.Cp * 2, rows=nr, F=Fd, ld_x=Fd, ldo=g.Cp))
            P.free(hm)
            y = P.f32(rows, C)
            P.gemm(g, r[f"{i}.{j}.fc2"], B=1, H=rows, out=y, res=x)
            P.free(g, x)
            x = y
        if i < len(W.depths) - 1:
            m = P.planes(rows // 4, 4 * C)
            P.ops.append(dict(kind="htsat_merge", tag=P.tag, x=x.ref, gamma=r[f"{i}.merge_ln"][0], beta=r[f"{i}.merge_ln"][1],
                              out_hi=m.hi, out_lo=m.lo, n=n, R=R, C=C, ldo=m.Cp, eps=eps))
            P.free(x)
            x = P.f32(rows // 4, 2 * C)
            P.gemm(m, r[f"{i}.reduction"], B=1, H=rows // 4, out=x)
            P.free(m)
            R //= 2
    P.tag = blk + 1
    Cf = x.C
    P.ops.append(dict(kind="htsat_head", tag=P.tag, x=x.ref, gamma=r["norm"][0], beta=r["norm"][1], w1_t=r["w1_t"],
                      b1=r["b1"], w2_t=r["w2_t"], b2=r["b2"], out=embed, n=n, ntok=R * R, C=Cf, P=A["joint_dim"], eps=eps))
    P.free(x)
    P.mark("end")
    assert P.arena.size == 0, "encoder plans reference the shared weight arena only"
    pl = P.finish(io, meta=dict(n=n, L=L, sr=sr, T=T, depths=W.depths))
    pl.arena = W.arena
    return pl
