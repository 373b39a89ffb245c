"""ctypes binding of the C-ABI in include/aldm_b200.h (+ the in-tree nvcc build).

The shared library is built IN-TREE (audioldm2_b200/libaldm_b200.so) so it travels with the
package.  There is no fallback: if the library is missing or the device
is not sm_90 (H100), every entry point raises.
"""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB_PATH = os.path.join(HERE, "libaldm_b200.so")
SOURCES = ["gemm.cu", "prep.cu", "attention.cu", "elementwise.cu", "stft.cu", "program.cu", "engine_abi.cu", "microbench.cu",
           "cond/seqgen.cu", "text/t5.cu", "clap/clap_text.cu", "audio/htsat.cu", "sampler/plms.cu",
           "sampler/style.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "--use_fast_math=false"]

# nvcc from PATH, else from the CUDA toolkit (CUDA_HOME, default /usr/local/cuda)
NVCC = shutil.which("nvcc") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")

MAX_TAPS = 16
ABI_VERSION = 14

# enums (keep in sync with the header; checked by tests/test_abi.py against the header text)
GEMM_TC, GEMM_SIMT, GEMM_TC_V1 = 0, 1, 2
GEMM_STATIC_B = 1 << 16
ACT_NONE, ACT_GEGLU, ACT_TANH, ACT_SILU, ACT_GELU_TANH = 0, 1, 2, 3, 4
OUT_F32, OUT_PLANES, OUT_NCHW, OUT_QKV = 0, 1, 2, 3
EPI_FAST, EPI_GEGLU, EPI_GENERIC, EPI_F32N, EPI_PLN = 0, 1, 2, 3, 4              # aldm_gemm_variant out[1]
RED_NONE, RED_REDUCE4, RED_GENERIC = 0, 1, 2                                     # out[3]
STORE_ROW, STORE_COMPACT, STORE_PAIR_PLN, STORE_PAIR_GEGLU, STORE_PAIR_QK = 0, 1, 2, 3, 4   # out[4]
AMODE_GATHER, AMODE_HALO = 0, 1                                                   # aldm_gemm_a_mode
PREP_COPY, PREP_SILU, PREP_LRELU, PREP_GN, PREP_GN_SILU, PREP_LN = 0, 1, 2, 3, 4, 5
OP_GEMM, OP_PREP, OP_ATTN, OP_SOFTMAX, OP_TEMB, OP_TRANSPOSE, OP_PACKB, OP_COPY = 1, 2, 3, 4, 5, 6, 7, 8
OP_SEQ_ASSEMBLE, OP_KV_ATTN, OP_SEQ_FEEDBACK = 9, 10, 11
OP_T5_EMBED, OP_T5_RMSNORM, OP_T5_ATTN, OP_T5_GATE = 12, 13, 14, 15
OP_CLAP_EMBED, OP_CLAP_LN, OP_CLAP_ATTN, OP_CLAP_GELU, OP_CLAP_HEAD = 16, 17, 18, 19, 20
OP_HTSAT_LOGMEL, OP_HTSAT_PATCH, OP_HTSAT_ATTN, OP_HTSAT_MERGE, OP_HTSAT_HEAD = 21, 22, 23, 24, 25
PLMS_AVERAGE = 0                                                                  # aldm_plms_step order of the first step's average


class GemmDesc(C.Structure):
    _fields_ = [
        ("a_hi", C.c_void_p), ("a_lo", C.c_void_p), ("w_packed", C.c_void_p), ("w_plain", C.c_void_p),
        ("bias", C.c_void_p), ("rowvec", C.c_void_p), ("res", C.c_void_p), ("out", C.c_void_p),
        ("out_hi", C.c_void_p), ("out_lo", C.c_void_p), ("out2_hi", C.c_void_p), ("out2_lo", C.c_void_p),
        ("ws", C.c_void_p),
        ("B", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("Cp", C.c_int32),
        ("up", C.c_int32), ("bmod", C.c_int32),
        ("OH", C.c_int32), ("OW", C.c_int32), ("sy", C.c_int32), ("sx", C.c_int32),
        ("ntaps", C.c_int32),
        ("dy", C.c_int16 * MAX_TAPS), ("dx", C.c_int16 * MAX_TAPS),
        ("N", C.c_int32), ("K", C.c_int32), ("Kpad", C.c_int32), ("bn", C.c_int32),
        ("ldo", C.c_int32), ("ld_res", C.c_int32), ("ld_rowvec", C.c_int32),
        ("OHF", C.c_int32), ("OWF", C.c_int32), ("osy", C.c_int32), ("ooy", C.c_int32),
        ("act", C.c_int32), ("out_mode", C.c_int32), ("accumulate", C.c_int32), ("splitk", C.c_int32),
        ("impl", C.c_int32), ("n_split", C.c_int32), ("tok_per_batch", C.c_int32), ("ld_t", C.c_int32),
        ("alpha", C.c_float),
    ]


class PrepDesc(C.Structure):
    _fields_ = [
        ("src0", C.c_void_p), ("src1", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p),
        ("out_hi", C.c_void_p), ("out_lo", C.c_void_p), ("scratch", C.c_void_p),
        ("rows", C.c_int32), ("c0", C.c_int32), ("c1", C.c_int32), ("Cp", C.c_int32),
        ("B", C.c_int32), ("HW", C.c_int32), ("groups", C.c_int32), ("mode", C.c_int32),
        ("eps", C.c_float), ("slope", C.c_float), ("src_nchw", C.c_int32),
    ]


class AttnDesc(C.Structure):
    _fields_ = [
        ("q_hi", C.c_void_p), ("q_lo", C.c_void_p), ("k_hi", C.c_void_p), ("k_lo", C.c_void_p),
        ("vt_hi", C.c_void_p), ("vt_lo", C.c_void_p), ("mask", C.c_void_p),
        ("out_hi", C.c_void_p), ("out_lo", C.c_void_p),
        ("B", C.c_int32), ("heads", C.c_int32), ("Nq", C.c_int32), ("Nk", C.c_int32),
        ("ldq", C.c_int32), ("ldk", C.c_int32), ("ld_t", C.c_int32), ("ldo", C.c_int32),
        ("q_col", C.c_int32), ("k_col", C.c_int32), ("kv_bmod", C.c_int32), ("impl", C.c_int32),
        ("scale", C.c_float),
    ]


class _Softmax(C.Structure):
    _fields_ = [("x", C.c_void_p), ("out_hi", C.c_void_p), ("out_lo", C.c_void_p),
                ("rows", C.c_int32), ("n", C.c_int32), ("scale", C.c_float)]


class _Temb(C.Structure):
    _fields_ = [("t", C.c_void_p), ("freqs", C.c_void_p), ("out_hi", C.c_void_p), ("out_lo", C.c_void_p),
                ("B", C.c_int32), ("dim", C.c_int32)]


class _Transpose(C.Structure):
    _fields_ = [("src", C.c_void_p), ("dst", C.c_void_p), ("B", C.c_int32), ("C", C.c_int32),
                ("HW", C.c_int32), ("to_nhwc", C.c_int32)]


class _PackB(C.Structure):
    _fields_ = [("src", C.c_void_p), ("dst_packed", C.c_void_p), ("dst_plain", C.c_void_p),
                ("lds", C.c_int32), ("transpose", C.c_int32), ("N", C.c_int32), ("K", C.c_int32), ("bn", C.c_int32)]


class _Copy(C.Structure):
    _fields_ = [("src", C.c_void_p), ("dst", C.c_void_p), ("bytes", C.c_int64)]


class KvAttnDesc(C.Structure):
    _fields_ = [("seq", C.c_void_p), ("mask", C.c_void_p), ("out_hi", C.c_void_p), ("out_lo", C.c_void_p),
                ("B", C.c_int32), ("heads", C.c_int32), ("lmax", C.c_int32), ("ld_seq", C.c_int32), ("p0", C.c_int32),
                ("nq", C.c_int32), ("ldo", C.c_int32), ("scale", C.c_float)]


class SeqAssembleDesc(C.Structure):
    _fields_ = [("x", C.c_void_p), ("sos", C.c_void_p), ("eos", C.c_void_p), ("wpe", C.c_void_p), ("t5_mask", C.c_void_p),
                ("mask", C.c_void_p), ("B", C.c_int32), ("L", C.c_int32), ("lmax", C.c_int32), ("C", C.c_int32)]


class SeqFeedbackDesc(C.Structure):
    _fields_ = [("x", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p), ("wpe", C.c_void_p), ("out", C.c_void_p),
                ("next", C.c_void_p), ("B", C.c_int32), ("nq", C.c_int32), ("C", C.c_int32), ("pos", C.c_int32),
                ("k", C.c_int32), ("gen_len", C.c_int32), ("eps", C.c_float)]


class T5EmbedDesc(C.Structure):
    _fields_ = [("ids", C.c_void_p), ("table", C.c_void_p), ("out", C.c_void_p), ("rows", C.c_int32), ("vocab", C.c_int32),
                ("C", C.c_int32)]


class T5RmsnormDesc(C.Structure):
    _fields_ = [("x", C.c_void_p), ("gamma", C.c_void_p), ("out_hi", C.c_void_p), ("out_lo", C.c_void_p),
                ("out_f32", C.c_void_p), ("rows", C.c_int32), ("C", C.c_int32), ("ldo", C.c_int32), ("eps", C.c_float)]


class T5AttnDesc(C.Structure):
    _fields_ = [("qkv", C.c_void_p), ("bias", C.c_void_p), ("mask", C.c_void_p), ("out_hi", C.c_void_p), ("out_lo", C.c_void_p),
                ("B", C.c_int32), ("L", C.c_int32), ("heads", C.c_int32), ("d_kv", C.c_int32), ("C", C.c_int32),
                ("ld_qkv", C.c_int32), ("ldo", C.c_int32)]


class T5GateDesc(C.Structure):
    _fields_ = [("x", C.c_void_p), ("out_hi", C.c_void_p), ("out_lo", C.c_void_p), ("sat", C.c_void_p),
                ("rows", C.c_int32), ("F", C.c_int32), ("ld_x", C.c_int32), ("ldo", C.c_int32)]


class ClapEmbedDesc(C.Structure):
    _fields_ = [("ids", C.c_void_p), ("word", C.c_void_p), ("pos", C.c_void_p), ("type", C.c_void_p), ("out", C.c_void_p),
                ("B", C.c_int32), ("L", C.c_int32), ("vocab", C.c_int32), ("n_pos", C.c_int32), ("C", C.c_int32),
                ("pad", C.c_int32)]


class ClapLnDesc(C.Structure):
    _fields_ = [("x", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p), ("out_f32", C.c_void_p),
                ("out_hi", C.c_void_p), ("out_lo", C.c_void_p), ("rows", C.c_int32), ("C", C.c_int32), ("ldo", C.c_int32),
                ("eps", C.c_float)]


class ClapAttnDesc(C.Structure):
    _fields_ = [("qkv", C.c_void_p), ("mask", C.c_void_p), ("out_hi", C.c_void_p), ("out_lo", C.c_void_p),
                ("B", C.c_int32), ("L", C.c_int32), ("heads", C.c_int32), ("C", C.c_int32), ("ld_qkv", C.c_int32),
                ("ldo", C.c_int32)]


class ClapGeluDesc(C.Structure):
    _fields_ = [("x", C.c_void_p), ("out_hi", C.c_void_p), ("out_lo", C.c_void_p),
                ("rows", C.c_int32), ("F", C.c_int32), ("ld_x", C.c_int32), ("ldo", C.c_int32)]


class ClapHeadDesc(C.Structure):
    _fields_ = [("x", C.c_void_p), ("wp_t", C.c_void_p), ("bp", C.c_void_p), ("w1_t", C.c_void_p), ("b1", C.c_void_p),
                ("w2_t", C.c_void_p), ("b2", C.c_void_p), ("out", C.c_void_p),
                ("B", C.c_int32), ("L", C.c_int32), ("C", C.c_int32), ("P", C.c_int32)]


class HtsatLogmelDesc(C.Structure):
    _fields_ = [("wav", C.c_void_p), ("taps", C.c_void_p), ("melW", C.c_void_p), ("bn_mean", C.c_void_p),
                ("bn_var", C.c_void_p), ("bn_w", C.c_void_p), ("bn_b", C.c_void_p), ("out", C.c_void_p),
                ("n", C.c_int32), ("L", C.c_int32), ("up", C.c_int32), ("L48", C.c_int32), ("T", C.c_int32),
                ("eps", C.c_float)]


class HtsatPatchDesc(C.Structure):
    _fields_ = [("mel", C.c_void_p), ("w", C.c_void_p), ("bias", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p),
                ("out", C.c_void_p), ("n", C.c_int32), ("T", C.c_int32), ("eps", C.c_float)]


class HtsatAttnDesc(C.Structure):
    _fields_ = [("qkv", C.c_void_p), ("bias", C.c_void_p), ("mask", C.c_void_p), ("out_hi", C.c_void_p),
                ("out_lo", C.c_void_p), ("n", C.c_int32), ("R", C.c_int32), ("shift", C.c_int32), ("heads", C.c_int32),
                ("head_dim", C.c_int32), ("C", C.c_int32), ("ld_qkv", C.c_int32), ("ldo", C.c_int32), ("scale", C.c_float)]


class HtsatMergeDesc(C.Structure):
    _fields_ = [("x", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p), ("out_hi", C.c_void_p), ("out_lo", C.c_void_p),
                ("n", C.c_int32), ("R", C.c_int32), ("C", C.c_int32), ("ldo", C.c_int32), ("eps", C.c_float)]


class HtsatHeadDesc(C.Structure):
    _fields_ = [("x", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p), ("w1_t", C.c_void_p), ("b1", C.c_void_p),
                ("w2_t", C.c_void_p), ("b2", C.c_void_p), ("out", C.c_void_p),
                ("n", C.c_int32), ("ntok", C.c_int32), ("C", C.c_int32), ("P", C.c_int32), ("eps", C.c_float)]


class _OpU(C.Union):
    _fields_ = [("gemm", GemmDesc), ("prep", PrepDesc), ("attn", AttnDesc), ("softmax", _Softmax),
                ("temb", _Temb), ("transpose", _Transpose), ("packb", _PackB), ("copy", _Copy),
                ("seq_assemble", SeqAssembleDesc), ("kv_attn", KvAttnDesc), ("seq_feedback", SeqFeedbackDesc),
                ("t5_embed", T5EmbedDesc), ("t5_rmsnorm", T5RmsnormDesc), ("t5_attn", T5AttnDesc), ("t5_gate", T5GateDesc),
                ("clap_embed", ClapEmbedDesc), ("clap_ln", ClapLnDesc), ("clap_attn", ClapAttnDesc), ("clap_gelu", ClapGeluDesc),
                ("clap_head", ClapHeadDesc), ("htsat_logmel", HtsatLogmelDesc), ("htsat_patch", HtsatPatchDesc),
                ("htsat_attn", HtsatAttnDesc), ("htsat_merge", HtsatMergeDesc), ("htsat_head", HtsatHeadDesc)]


class Op(C.Structure):
    _fields_ = [("kind", C.c_int32), ("tag", C.c_int32), ("u", _OpU)]


MAX_LANES = 8


class UnetLane(C.Structure):
    """aldm_unet_lane: one independent sub-batch of the UNet (own programs + workspace slots)."""
    _fields_ = [("cond", C.c_void_p), ("step", C.c_void_p), ("x_slot", C.c_void_p), ("t_slot", C.c_void_p),
                ("eps_slot", C.c_void_p), ("ctx_slot", C.c_void_p * 2), ("mask_slot", C.c_void_p * 2),
                ("film_slot", C.c_void_p)]


class EngineDesc(C.Structure):
    """aldm_engine_desc (include/aldm_b200.h): programs + their fixed I/O slots."""
    _fields_ = [("lane", UnetLane * MAX_LANES), ("n_lanes", C.c_int32),
                ("vae_dec", C.c_void_p), ("vocoder", C.c_void_p), ("vae_enc", C.c_void_p),
                ("z_slot", C.c_void_p), ("mel_slot", C.c_void_p), ("voc_mel_slot", C.c_void_p), ("wave_slot", C.c_void_p),
                ("enc_mel_slot", C.c_void_p), ("moments_slot", C.c_void_p), ("B", C.c_int32), ("latent_elems", C.c_int32),
                ("mel_elems", C.c_int32), ("wave_len", C.c_int32), ("n_ctx", C.c_int32), ("ctx_len", C.c_int32 * 2),
                ("ctx_dim", C.c_int32 * 2), ("film_dim", C.c_int32), ("use_graph", C.c_int32)]


def build(verbose: bool = False, force: bool = False) -> str:
    """Compile every CUDA source for sm_90a into audioldm2_b200/libaldm_b200.so (nvcc cross-compiles
    without a GPU).  Rebuilds only when a source is newer than the library."""
    srcs = [os.path.join(CSRC, s) for s in SOURCES]
    deps = srcs + [os.path.join(CSRC, "common.cuh"), os.path.join(ROOT, "include", "aldm_b200.h")]
    if not force and os.path.exists(LIB_PATH) and all(os.path.getmtime(LIB_PATH) >= os.path.getmtime(d) for d in deps):
        return LIB_PATH
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for s in srcs:
        o = os.path.join(HERE, "build", os.path.basename(s) + ".o")
        objs.append(o)
        cmd = [NVCC] + [f for f in NVCC_FLAGS if not f.startswith("--use_fast_math")] + ["-c", s, "-o", o]
        if verbose:
            print(" ".join(cmd))
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for cmd, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError("nvcc failed: %s\n%s" % (" ".join(cmd), out.decode()))
        if verbose and out:
            print(out.decode())
    cmd = [NVCC, "-shared", "-o", LIB_PATH] + objs + ["-lcudart"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    if r.returncode != 0:
        raise RuntimeError("link failed: %s\n%s" % (" ".join(cmd), r.stdout.decode()))
    return LIB_PATH


_lib = None


def lib() -> C.CDLL:
    """Load the shared library (raises if it has not been built -- no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'`. "
                           "There is no CPU/PyTorch fallback for the native path.")
    L = C.CDLL(LIB_PATH)
    vp, i32, i64, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
    sig = {
        "aldm_gemm": (i32, [C.POINTER(GemmDesc), vp]),
        "aldm_gemm_variant": (i32, [C.POINTER(GemmDesc), C.POINTER(i32)]),
        "aldm_gemm_a_mode": (i32, [C.POINTER(GemmDesc), C.POINTER(i32)]),
        "aldm_prep": (i32, [C.POINTER(PrepDesc), vp]),
        "aldm_pack_b": (i32, [vp, i32, i32, i32, i32, i32, vp, vp, vp]),
        "aldm_attention": (i32, [C.POINTER(AttnDesc), vp]),
        "aldm_kv_attention": (i32, [C.POINTER(KvAttnDesc), vp]),
        "aldm_seq_assemble": (i32, [C.POINTER(SeqAssembleDesc), vp]),
        "aldm_seq_feedback": (i32, [C.POINTER(SeqFeedbackDesc), vp]),
        "aldm_t5_embed": (i32, [C.POINTER(T5EmbedDesc), vp]),
        "aldm_t5_rmsnorm": (i32, [C.POINTER(T5RmsnormDesc), vp]),
        "aldm_t5_attention": (i32, [C.POINTER(T5AttnDesc), vp]),
        "aldm_t5_gate": (i32, [C.POINTER(T5GateDesc), vp]),
        "aldm_clap_embed": (i32, [C.POINTER(ClapEmbedDesc), vp]),
        "aldm_clap_layernorm": (i32, [C.POINTER(ClapLnDesc), vp]),
        "aldm_clap_attention": (i32, [C.POINTER(ClapAttnDesc), vp]),
        "aldm_clap_gelu": (i32, [C.POINTER(ClapGeluDesc), vp]),
        "aldm_clap_head": (i32, [C.POINTER(ClapHeadDesc), vp]),
        "aldm_htsat_logmel": (i32, [C.POINTER(HtsatLogmelDesc), vp]),
        "aldm_htsat_patch": (i32, [C.POINTER(HtsatPatchDesc), vp]),
        "aldm_htsat_window_attention": (i32, [C.POINTER(HtsatAttnDesc), vp]),
        "aldm_htsat_merge": (i32, [C.POINTER(HtsatMergeDesc), vp]),
        "aldm_htsat_head": (i32, [C.POINTER(HtsatHeadDesc), vp]),
        "aldm_softmax_rows": (i32, [vp, i32, i32, f32, vp, vp, vp]),
        "aldm_timestep_embedding": (i32, [vp, i32, i32, vp, vp, vp, vp]),
        "aldm_ddim_step": (i32, [vp, vp, vp, vp, vp, vp, i64, f32, f32, f32, f32, f32, vp]),
        "aldm_plms_step": (i32, [vp, vp, vp, vp, vp, vp, i32, vp, vp, vp, i64, f32, f32, f32, f32, vp]),
        "aldm_stochastic_encode": (i32, [vp, vp, vp, i64, f32, f32, vp, vp]),
        "aldm_masked_blend": (i32, [vp, vp, vp, vp, i32, i32, i32, f32, f32, vp]),
        "aldm_transpose_chw": (i32, [vp, vp, i32, i32, i32, i32, vp]),
        "aldm_posterior_sample": (i32, [vp, vp, vp, i32, i32, i32, f32, vp]),
        "aldm_stft_mel": (i32, [vp, i32, i32, i32, i32, vp, i32, vp, i32, vp]),
        "aldm_program_create": (i32, [C.POINTER(Op), i32, C.POINTER(vp)]),
        "aldm_program_run": (i32, [vp, vp]),
        "aldm_program_run_range": (i32, [vp, i32, i32, vp]),
        "aldm_program_capture": (i32, [vp, vp]),
        "aldm_program_replay": (i32, [vp, vp]),
        "aldm_program_num_launches": (i32, [vp]),
        "aldm_program_is_captured": (i32, [vp]),
        "aldm_program_destroy": (None, [vp]),
        "aldm_engine_create": (i32, [C.POINTER(EngineDesc), C.POINTER(vp)]),
        "aldm_engine_destroy": (None, [vp]),
        "aldm_engine_set_conditioning": (i32, [vp, i32, vp, vp, i32, vp, vp, i32, vp, vp]),
        "aldm_engine_precompute": (i32, [vp, vp]),
        "aldm_engine_unet_eps": (i32, [vp, vp, i64, vp, vp, vp]),
        "aldm_engine_ddim_step": (i32, [vp, vp, i64, vp, f32, f32, f32, f32, f32, vp, vp, vp]),
        "aldm_engine_plms_step": (i32, [vp, vp, i64, vp, vp, vp, vp, i32, vp, f32, f32, f32, f32, vp, vp, vp]),
        "aldm_engine_vae_decode": (i32, [vp, vp, vp, vp]),
        "aldm_engine_vocoder": (i32, [vp, vp, vp, vp]),
        "aldm_engine_vae_encode": (i32, [vp, vp, vp, vp]),
        "aldm_sizeof_engine_desc": (C.c_size_t, []),
        "aldm_abi_version": (i32, []),
        "aldm_sizeof_op": (C.c_size_t, []),
        "aldm_sizeof_gemm_desc": (C.c_size_t, []),
        "aldm_offsetof_gemm": (C.c_size_t, [i32]),
        "aldm_last_error": (C.c_char_p, []),
        "aldm_device_check": (i32, [i32]),
        "aldm_debug_timeline": (i32, [vp, i32]),
        "aldm_debug_store_rate": (i32, [i32, i32, i32, i64, vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)          # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if L.aldm_abi_version() != ABI_VERSION:
        raise RuntimeError("libaldm_b200.so ABI version mismatch: rebuild")
    if L.aldm_sizeof_engine_desc() != C.sizeof(EngineDesc):
        raise RuntimeError("ctypes mirror of aldm_engine_desc does not match the C layout")
    if L.aldm_sizeof_op() != C.sizeof(Op) or L.aldm_sizeof_gemm_desc() != C.sizeof(GemmDesc):
        raise RuntimeError("ctypes mirror of aldm_op / aldm_gemm_desc does not match the C layout")
    _lib = L
    return L


EXPORTED = ["aldm_gemm", "aldm_gemm_variant", "aldm_gemm_a_mode", "aldm_prep", "aldm_pack_b", "aldm_attention", "aldm_softmax_rows",
            "aldm_kv_attention", "aldm_seq_assemble", "aldm_seq_feedback",
            "aldm_t5_embed", "aldm_t5_rmsnorm", "aldm_t5_attention", "aldm_t5_gate",
            "aldm_clap_embed", "aldm_clap_layernorm", "aldm_clap_attention", "aldm_clap_gelu", "aldm_clap_head",
            "aldm_htsat_logmel", "aldm_htsat_patch", "aldm_htsat_window_attention", "aldm_htsat_merge", "aldm_htsat_head",
            "aldm_timestep_embedding", "aldm_ddim_step", "aldm_plms_step", "aldm_stochastic_encode", "aldm_masked_blend", "aldm_transpose_chw",
            "aldm_posterior_sample", "aldm_stft_mel", "aldm_program_create", "aldm_program_run",
            "aldm_program_run_range", "aldm_program_capture", "aldm_program_replay",
            "aldm_program_num_launches", "aldm_program_is_captured", "aldm_program_destroy", "aldm_engine_create",
            "aldm_engine_destroy", "aldm_engine_set_conditioning", "aldm_engine_precompute", "aldm_engine_unet_eps",
            "aldm_engine_ddim_step", "aldm_engine_plms_step", "aldm_engine_vae_decode", "aldm_engine_vocoder", "aldm_engine_vae_encode",
            "aldm_sizeof_engine_desc", "aldm_abi_version", "aldm_sizeof_op",
            "aldm_sizeof_gemm_desc", "aldm_offsetof_gemm", "aldm_last_error", "aldm_device_check", "aldm_debug_timeline",
            "aldm_debug_store_rate"]


def gemm_variant(d: GemmDesc) -> tuple:
    """aldm_gemm_variant: (bn, epi, a_planes, reduction, store) of the kernel aldm_gemm runs for `d` (no GPU needed)."""
    out = (C.c_int32 * 5)()
    check(lib().aldm_gemm_variant(C.byref(d), out), "gemm_variant")
    return tuple(out)


def gemm_a_mode(d: GemmDesc) -> int:
    """aldm_gemm_a_mode: AMODE_GATHER or AMODE_HALO, how the kernel aldm_gemm runs for `d` loads A (no GPU needed)."""
    out = C.c_int32()
    check(lib().aldm_gemm_a_mode(C.byref(d), C.byref(out)), "gemm_a_mode")
    return out.value


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = lib().aldm_last_error().decode(errors="replace")
        raise RuntimeError(f"aldm error {rc} {what}: {msg}")


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
