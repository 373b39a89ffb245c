"""Weight packing: reference ``state_dict`` tensors -> tensor-core tile images.

Layout consumed by csrc/gemm.cu (and produced on-device by pack_b_kernel for dynamic operands):

    packed[n_tile][k_blk][plane(hi,lo)][row r in 0..bn)[128 bytes]

where a row holds 64 fp16 K-elements of output channel ``n_tile*bn + r`` and its eight 16-byte
chunks are XOR-swizzled with ``r & 7`` (the UMMA SWIZZLE_128B K-major canonical layout), so one
``cp.async.bulk`` per stage drops a ready-to-use B tile into shared memory.  ``hi = fp16(w)``,
``lo = fp16(w - hi)``: 22 significand bits for |w| >= 2^-14 * 2^11, absolute error <= 2^-25 below
(fp16 subnormals), i.e. weights are exact to fp32 round-off at the magnitudes networks hold.

K ordering of a convolution is ``k = tap * Cp + c`` (Cp = Cin rounded up to 8, zero padded), taps
in the order of the (dy, dx) list the planner emits.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch

BK = 64


def round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def choose_bn(N: int) -> int:
    if N % 128 == 0:
        return 128
    if N % 64 == 0:
        return 64
    if N % 32 == 0 or N < 32:
        return 32
    return 64 if N < 128 else 128


def conv_weight_matrix(w: torch.Tensor) -> Tuple[torch.Tensor, int, int]:
    """Conv2d [Cout, Cin, kh, kw] or Conv1d [Cout, Cin, k] or Linear [Cout, Cin] -> ([Cout, taps*Cp], taps, Cp)
    with k = tap*Cp + c and taps enumerated row-major over (kh, kw)."""
    if w.dim() == 2:
        w = w[:, :, None]
    cout, cin = w.shape[0], w.shape[1]
    taps = 1
    for d in w.shape[2:]:
        taps *= d
    cp = round_up(cin, 8)
    m = torch.zeros(cout, taps, cp, dtype=torch.float32)
    m[:, :, :cin] = w.reshape(cout, cin, taps).permute(0, 2, 1).float()
    return m.reshape(cout, taps * cp), taps, cp


def conv1d_weight_matrix(w: torch.Tensor) -> Tuple[torch.Tensor, int, int]:
    """HF ``Conv1D`` weight [in, out] (y = x W + b, the GPT-2 linear layers) -> ([out, Cp], 1 tap, Cp): the transpose of
    a Linear weight, then the usual [N, K] matrix."""
    return conv_weight_matrix(w.t().contiguous())


def geglu_row_order(n_inner: int, bn: int) -> torch.Tensor:
    """Row permutation of GEGLU.proj ([2*n_inner, C]: values then gates, attention.py:42-44) so that every
    bn-row tile holds bn/2 value rows followed by their bn/2 gate rows."""
    half = bn // 2
    assert n_inner % half == 0
    idx = []
    for t in range(n_inner // half):
        idx.append(torch.arange(t * half, (t + 1) * half))
        idx.append(n_inner + torch.arange(t * half, (t + 1) * half))
    return torch.cat(idx)


F16_MAX = 65504.0


def split_f16(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """x ~= hi + lo with fp16 planes, saturating at +-65504 exactly like the device-side split (csrc/common.cuh)."""
    w = w.float().clamp(-F16_MAX, F16_MAX)
    hi = w.to(torch.float16)
    lo = (w - hi.float()).to(torch.float16)
    return hi, lo


def pack_tiles(wm: torch.Tensor, bn: int) -> Tuple[torch.Tensor, torch.Tensor, int, int]:
    """[N, K] fp32 -> (packed uint8 1-D, plain fp32 [Npad, Kpad], Npad, Kpad)."""
    N, K = wm.shape
    Npad, Kpad = round_up(N, bn), round_up(K, BK)
    plain = torch.zeros(Npad, Kpad, dtype=torch.float32)
    plain[:N, :K] = wm
    hi, lo = split_f16(plain)
    nt, kb = Npad // bn, Kpad // BK

    def tiles(p: torch.Tensor) -> torch.Tensor:
        # [Npad, Kpad] -> [nt, bn, kb, 8 chunks, 8 elems] -> [nt, kb, bn, 8, 8]
        t = p.reshape(nt, bn, kb, 8, 8).permute(0, 2, 1, 3, 4).contiguous()
        r = torch.arange(bn) & 7
        j = torch.arange(8)
        src = (j[None, :] ^ r[:, None])            # stored chunk position p holds logical chunk p ^ (r&7)
        idx = src[None, None, :, :, None].expand(nt, kb, bn, 8, 8)
        return torch.gather(t, 3, idx)

    both = torch.stack([tiles(hi), tiles(lo)], dim=2)          # [nt, kb, 2, bn, 8, 8]
    packed = both.contiguous().view(torch.uint8).reshape(-1)
    return packed, plain, Npad, Kpad


def unpack_tiles(packed: torch.Tensor, N: int, K: int, bn: int) -> torch.Tensor:
    """Inverse of pack_tiles (hi + lo as fp32) -- used by tests."""
    Npad, Kpad = round_up(N, bn), round_up(K, BK)
    nt, kb = Npad // bn, Kpad // BK
    both = packed.view(torch.float16).reshape(nt, kb, 2, bn, 8, 8).float()
    r = torch.arange(bn) & 7
    j = torch.arange(8)
    src = (j[None, :] ^ r[:, None])
    idx = src[None, None, None, :, :, None].expand(nt, kb, 2, bn, 8, 8)
    un = torch.gather(both, 4, idx)                            # XOR swizzle is an involution
    w = un[:, :, 0] + un[:, :, 1]                              # [nt, kb, bn, 8, 8]
    w = w.permute(0, 2, 1, 3, 4).reshape(Npad, Kpad)
    return w[:N, :K]


def conv_transpose_phases(w: torch.Tensor, u: int) -> List[dict]:
    """ConvTranspose1d weight [Cin, Cout, k], stride u, padding (k-u)//2 (hifigan/models.py:127-133) ->
    one stride-1 convolution per output phase r (t = q*u + r):

        y[b, q*u + r, n] = sum_m sum_c x[b, q + d_m, c] * w[c, n, j_m],   j_m = (r+p) % u + m*u,
                                                                          d_m = (r+p) // u - m

    Returns [{r, taps: [d_m], weight: [Cout, ntaps*Cp]}]."""
    cin, cout, k = w.shape
    p = (k - u) // 2
    cp = round_up(cin, 8)
    out = []
    for r in range(u):
        j0 = (r + p) % u
        js = list(range(j0, k, u))
        d0 = (r + p) // u
        taps = [d0 - m for m in range(len(js))]
        m = torch.zeros(cout, len(js), cp, dtype=torch.float32)
        for mi, j in enumerate(js):
            m[:, mi, :cin] = w[:, :, j].t().float()
        out.append(dict(r=r, taps=taps, weight=m.reshape(cout, len(js) * cp), cp=cp))
    return out
