"""The halo A path of the persistent GEMM (aldm_gemm_a_mode == AMODE_HALO): a 3x3, stride-1 convolution loads each
64-channel block of an 8 x 16 (W % 16 == 0) or 16 x 8 (W == 8) pixel tile once (upsampled or not), with its one-pixel border, and issues
the nine taps from that copy through shifted shared-memory descriptors.

The GPU cases run through test_gpu_kernel_matrix.test_gemm_matrix: the same float64 reference, error bounds and guard
bands as every other GEMM variant.  They cover both tile shapes, with and without the nearest x2 upsample, one and two
A planes, Cp of 64, 128, 256 and 640, batch 1
and 16 with the batch modulo (x shared by the cond and uncond halves), every epilogue body and store the halo path can
take with one and with two A planes (FAST with a strided row vector and residual, compact fp32, compact and pair plane
stores, and generic with NCHW, SiLU or alpha / accumulate), ragged N tiles, and images of one tile row or column (every
tile touches the zero border) up to several tiles per persistent CTA.  The CPU tests pin which descriptors take the halo path and that every other shape keeps the gather."""
import pytest

from audioldm2_b200 import _lib, plan
from tests import test_gpu_kernel_matrix as KM

T3, T3A = plan.TAPS_3x3, plan.TAPS_3x3_ASYM

HALO_CASES = {
    # tw = 16 (8 x 16 tiles)
    "halo_w16_a2_c128_res": dict(B=2, H=16, W=16, Cin=128, N=128, taps=T3, bn=128, res=True),
    "halo_w32_a1_c64_pln": dict(H=8, W=32, Cin=64, N=128, taps=T3, bn=128, out="planes", planes_out=1, a_planes=1),
    "halo_w16_a2_c640_nchw": dict(H=8, W=16, Cin=640, N=128, taps=T3, bn=128, out="nchw"),
    "halo_w48_a1_c64_fast": dict(B=2, H=24, W=48, Cin=64, N=256, taps=T3, bn=128, rowvec=True, res=True, a_planes=1),
    "halo_w16_a2_c64_b16_bmod": dict(B=16, H=8, W=16, Cin=64, N=128, taps=T3, bn=128, bmod=8, res=True),
    "halo_w16_a2_c64_many": dict(B=8, H=128, W=16, Cin=64, N=256, taps=T3, bn=128, res=True),
    # tw = 8 (16 x 8 tiles)
    "halo_w8_a2_c256_b16_bmod": dict(B=16, H=16, W=8, Cin=256, N=256, taps=T3, bn=128, bmod=8, res=True),
    "halo_w8_a1_c128_n192": dict(H=32, W=8, Cin=128, N=192, taps=T3, bn=128, out="planes", a_planes=1),
    "halo_w8_a2_c128_dual": dict(B=2, H=48, W=8, Cin=128, N=128, taps=T3, bn=128, dual=2, pad_cols=8),
    # nearest x2 upsample folded into the halo
    "halo_up_w16_a2_c128": dict(B=2, H=16, W=32, Cin=128, N=128, taps=T3, up=1, bn=128, res=True),
    "halo_up_w8_a2_c64_bmod": dict(B=4, H=32, W=8, Cin=64, N=64, taps=T3, up=1, bmod=2, bn=64, out="planes"),
    # weights packed in 64-row tiles
    "halo_w16_a2_c64_bn64": dict(B=2, H=16, W=32, Cin=64, N=192, taps=T3, bn=64, res=True),
    # FAST body with two A planes: the ResBlock's first convolution adds the timestep embedding, a row vector read at a
    # column offset inside a row of every ResBlock's embeddings
    "halo_w16_a2_c128_fast_emb": dict(B=4, H=8, W=32, Cin=128, N=128, taps=T3, bn=128, rowvec=True, ld_rowvec=1000,
                                      rowvec_col=256, res=True, res_pad=4),
    "halo_w8_a2_c64_fast_emb": dict(B=3, H=32, W=8, Cin=64, N=192, taps=T3, bn=128, rowvec=True, ld_rowvec=600,
                                    rowvec_col=400, pad_cols=8),
    "halo_up_w16_a2_c64_fast_emb": dict(B=2, H=16, W=32, Cin=64, N=128, taps=T3, up=1, bn=128, rowvec=True,
                                        ld_rowvec=260, rowvec_col=132, res=True),
    # GENERIC body: an activation; alpha / accumulate with a leading dimension the compact bodies cannot store
    "halo_w16_a1_c64_silu": dict(B=2, H=8, W=16, Cin=64, N=128, taps=T3, bn=128, act=_lib.ACT_SILU, a_planes=1),
    "halo_w8_a2_c128_alpha_acc": dict(B=2, H=16, W=8, Cin=128, N=128, taps=T3, bn=64, res=True, alpha=1 / 3,
                                      accumulate=True, pad_cols=2),
    # compact fp32 body with one A plane; pair plane stores with two
    "halo_w16_a1_c128_f32n": dict(B=2, H=16, W=16, Cin=128, N=128, taps=T3, bn=128, a_planes=1),
    "halo_w32_a2_c64_pair": dict(H=8, W=32, Cin=64, N=128, taps=T3, bn=128, out="planes", planes_out=1),
}

# shapes that must keep the gather: one property away from a halo case each
GATHER_CASES = {
    "gather_stride2": dict(B=2, H=16, W=16, Cin=64, N=128, taps=T3, OH=8, OW=8, sy=2, sx=2, bn=128),
    "gather_up_w8_h8": dict(B=2, H=8, W=8, Cin=64, N=128, taps=T3, up=1, bn=128),
    "gather_asym": dict(B=2, H=16, W=16, Cin=64, N=128, taps=T3A, bn=128),
    "gather_cp40": dict(B=2, H=16, W=16, Cin=40, N=128, taps=T3, bn=128),
    "gather_w4": dict(B=2, H=16, W=4, Cin=64, N=128, taps=T3, bn=128),
    "gather_w24": dict(B=2, H=16, W=24, Cin=64, N=128, taps=T3, bn=128),
    "gather_w8_h8": dict(B=2, H=8, W=8, Cin=64, N=128, taps=T3, bn=128),
    "gather_w16_h12": dict(B=2, H=12, W=16, Cin=64, N=128, taps=T3, bn=128),
    "gather_bn32": dict(B=2, H=16, W=16, Cin=64, N=128, taps=T3, bn=32),
    "gather_geglu": dict(B=2, H=16, W=16, Cin=64, N=256, taps=T3, bn=128, act=_lib.ACT_GEGLU),
    "gather_splitk": dict(B=2, H=16, W=16, Cin=640, N=128, taps=T3, bn=128, splitk=4),
    "gather_1d": dict(B=2, H=64, Cin=64, N=128, taps=plan.taps_1d(3), bn=128),
    "gather_1x1": dict(B=2, H=16, W=16, Cin=64, N=128, bn=128),
}


def _desc(name: str, spec: dict, monkeypatch):
    monkeypatch.setitem(KM.GEMM_MATRIX, name, spec)
    c = KM.plan_gemm(name, plan.H100_SMS)
    d = KM._gemm_desc(c)
    if spec.get("splitk", 1) > 1:
        d.splitk = spec["splitk"]
    return d


@pytest.mark.parametrize("name", sorted(HALO_CASES))
def test_halo_selected(name, monkeypatch):
    _lib.build()
    d = _desc(name, HALO_CASES[name], monkeypatch)
    assert _lib.gemm_a_mode(d) == _lib.AMODE_HALO
    v = _lib.gemm_variant(d)
    assert v[0] == 64 and v[2] == HALO_CASES[name].get("a_planes", 2), v      # 64-wide N tiles of the 128-wide packing


@pytest.mark.parametrize("name", sorted(GATHER_CASES))
def test_other_shapes_keep_the_gather(name, monkeypatch):
    _lib.build()
    d = _desc(name, GATHER_CASES[name], monkeypatch)
    assert _lib.gemm_a_mode(d) == _lib.AMODE_GATHER


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(HALO_CASES))
def test_halo_conv(name, monkeypatch):
    monkeypatch.setitem(KM.GEMM_MATRIX, name, HALO_CASES[name])
    assert _lib.gemm_a_mode(KM._gemm_desc(KM.plan_gemm(name, KM._n_sm()))) == _lib.AMODE_HALO
    KM.test_gemm_matrix(name)
