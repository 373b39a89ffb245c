"""CPU checks of the C-ABI: the library builds/loads, exports every symbol the header declares,
and the ctypes mirrors agree with the C layout.  No compute calls (no GPU here)."""
import ctypes as C
import os
import re

import pytest

from audioldm2_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def L():
    _lib.build()
    return _lib.lib()


def test_header_symbols_exported(L):
    hdr = open(os.path.join(ROOT, "include", "aldm_b200.h")).read()
    declared = set(re.findall(r"\b(aldm_[a-z0-9_]+)\s*\(", hdr))
    declared -= {"aldm_program_run("}
    assert declared, "no declarations parsed"
    for name in sorted(declared):
        assert hasattr(L, name), f"{name} declared in include/aldm_b200.h but not exported"
    assert declared == set(_lib.EXPORTED)


def test_struct_mirrors(L):
    assert L.aldm_abi_version() == _lib.ABI_VERSION
    assert L.aldm_sizeof_op() == C.sizeof(_lib.Op)
    assert L.aldm_sizeof_gemm_desc() == C.sizeof(_lib.GemmDesc)
    for i, f in enumerate(["B", "ntaps", "dy", "N", "ldo", "act", "alpha"]):
        assert L.aldm_offsetof_gemm(i) == getattr(_lib.GemmDesc, f).offset, f


def test_enum_values_match_header():
    hdr = open(os.path.join(ROOT, "include", "aldm_b200.h")).read()
    def val(name):
        m = re.search(r"\b" + name + r"\s*=\s*(-?\d+)", hdr)
        assert m, name
        return int(m.group(1))
    assert val("ALDM_GEMM_TC") == _lib.GEMM_TC and val("ALDM_GEMM_SIMT") == _lib.GEMM_SIMT and val("ALDM_GEMM_TC_V1") == _lib.GEMM_TC_V1
    assert [val("ALDM_ACT_NONE"), val("ALDM_ACT_GEGLU"), val("ALDM_ACT_TANH"), val("ALDM_ACT_SILU")] == [0, 1, 2, 3]
    assert [val("ALDM_OUT_F32"), val("ALDM_OUT_PLANES"), val("ALDM_OUT_NCHW")] == [0, 1, 2]
    assert [val("ALDM_EPI_" + n) for n in ("FAST", "GEGLU", "GENERIC", "F32N", "PLN")] == \
        [_lib.EPI_FAST, _lib.EPI_GEGLU, _lib.EPI_GENERIC, _lib.EPI_F32N, _lib.EPI_PLN]
    assert [val("ALDM_RED_" + n) for n in ("NONE", "REDUCE4", "GENERIC")] == [_lib.RED_NONE, _lib.RED_REDUCE4, _lib.RED_GENERIC]
    assert [val("ALDM_STORE_" + n) for n in ("ROW", "COMPACT", "PAIR_PLN", "PAIR_GEGLU", "PAIR_QK")] == \
        [_lib.STORE_ROW, _lib.STORE_COMPACT, _lib.STORE_PAIR_PLN, _lib.STORE_PAIR_GEGLU, _lib.STORE_PAIR_QK]
    assert [val("ALDM_PREP_" + n) for n in ("COPY", "SILU", "LRELU", "GN", "GN_SILU", "LN")] == [0, 1, 2, 3, 4, 5]
    assert [val("ALDM_OP_" + n) for n in ("GEMM", "PREP", "ATTN", "SOFTMAX", "TEMB", "TRANSPOSE", "PACKB", "COPY")] == \
        [1, 2, 3, 4, 5, 6, 7, 8]
    assert val("ALDM_ABI_VERSION") if False else True
    assert int(re.search(r"#define ALDM_MAX_TAPS (\d+)", hdr).group(1)) == _lib.MAX_TAPS
    assert int(re.search(r"#define ALDM_ABI_VERSION (\d+)", hdr).group(1)) == _lib.ABI_VERSION


def test_errors_are_codes_not_crashes(L):
    # argument validation happens before any CUDA call, so this is safe without a GPU
    assert L.aldm_gemm(None, None) == -1
    assert b"null" in L.aldm_last_error()
    d = _lib.GemmDesc()
    d.B, d.OH, d.OW, d.bn = 1, 1, 1, 48
    assert L.aldm_gemm(C.byref(d), None) == -6          # ALDM_E_UNSUPPORTED: no silent fallback
    assert b"bn=48" in L.aldm_last_error()


def test_engine_abi_validates_without_gpu(L):
    """aldm_engine_* (SURVEY 8b seams): descriptor mirror + argument checks return codes, never crash."""
    assert L.aldm_sizeof_engine_desc() == C.sizeof(_lib.EngineDesc)
    h = C.c_void_p()
    assert L.aldm_engine_create(None, C.byref(h)) == -1
    d = _lib.EngineDesc()
    assert L.aldm_engine_create(C.byref(d), C.byref(h)) == -1          # n_lanes = 0
    assert b"n_lanes" in L.aldm_last_error()
    d.n_lanes = 2
    assert L.aldm_engine_create(C.byref(d), C.byref(h)) == -2          # ALDM_E_SHAPE: B = 0
    d.B, d.latent_elems, d.n_ctx = 3, 64, 1
    assert L.aldm_engine_create(C.byref(d), C.byref(h)) == -2          # B % n_lanes != 0
    d.B = 2
    assert L.aldm_engine_create(C.byref(d), C.byref(h)) == -1          # lane 0: no UNet program / slots
    assert b"UNet" in L.aldm_last_error()
    for l in range(2):                                                   # dummy non-null handles
        d.lane[l].step, d.lane[l].x_slot, d.lane[l].t_slot, d.lane[l].eps_slot = 1, 16, 16, 16
    assert L.aldm_engine_create(C.byref(d), C.byref(h)) == -1          # context 0 slots missing
    d.n_ctx = 0
    assert L.aldm_engine_create(C.byref(d), C.byref(h)) == 0 and h.value
    assert L.aldm_engine_vae_decode(h, None, None, None) == -1           # no decoder program
    assert L.aldm_engine_set_conditioning(h, 2, None, None, 0, None, None, 0, None, None) == -1
    L.aldm_engine_destroy(h)


def test_product_path_does_not_import_oracle():
    pkg = os.path.join(ROOT, "audioldm2_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py"):
            src = open(os.path.join(pkg, fn)).read()
            assert "import oracle" not in src and "from oracle" not in src, fn
