"""The CLAP audio encoder and the native re-ranker on the GPU: the kernels of csrc/audio/*.cu against float64 inside 4 KB
guard bands at production shapes, every GEMM signature of the plan through tests/test_gpu_kernel_matrix.py's checker, the
whole encoder against the reference fixtures and the float64 oracle, bit-exact properties and text_to_audio end to end.

Bounds (relative L2 AND per element, as tests/test_gpu_kernel_matrix.py, unless stated):
  * htsat_logmel_kernel: the fp32 resample (15 fmaf in order, ~15 x 2^-24 of sum |tap x|), a radix-2 FFT of 10 stages
    (~10 x 2^-24 x sqrt(sum x^2) absolute per bin) and the 513-term mel sum (~16 x 2^-24 of the sum: a fixed lane-strided
    order) move the mel energy by ~1e-6 relative where it is well above the FFT's absolute error, i.e. 10 log10 by
    ~5e-6 dB, then / 15 dB (bn0): ~1e-6 absolute on O(1) outputs.  Bins near the 1e-10 floor are not reached by the test
    signals.  Bound: relative L2 < 1e-5, |err| <= 1e-4 max |ref|.
  * htsat_patch_kernel: four-term bicubic sums (source indices and weights computed in fp32 as the reference computes
    them, plan.htsat_bicubic; the float64 reference applies the same fp32 weights), a 16-term conv dot product and
    LayerNorm(128): a few 2^-24 relative, amplified by the LayerNorm's 1 / std: relative L2 < 1e-5, |err| <= 1e-4 max
    |ref|.
  * htsat_window_attention_kernel: fp32 q, k, v; 32-term dot products (<= 32 x 2^-24 of sum |q k|), the bias and mask
    adds, expf (2 ulp) and a 64-term P V sum, then the two-plane split: the two-plane budget of the matrix.
  * htsat_merge_kernel: LayerNorm over 4C <= 2048 with fixed-order sums (as clap_layernorm_kernel) and the split: the
    two-plane budget.
  * htsat_head_kernel: 64 LayerNorms of 1024 and the mean (64 x 2^-24), then two fp32 dot products of <= 1024 terms and
    the normalisation: relative L2 < 1e-5 per clip.
The encoder: relative L2 per clip below TOL = 1e-4 against the reference fixtures (fp32 torch on the CPU) and against the
float64 oracle at n = 24.  CPU emulation of the planned program (fp16 two-plane GEMM operands, fp32 elsewhere,
tests/test_clap_audio_cpu.py) bounds the cost of the operand planes on the small-depth cases; the tensor cores'
truncating accumulation adds at most ~1e-6 per GEMM (tests/test_gpu_kernel_matrix.py) over 18 x 4 + 3 GEMMs.
"""
import glob
import os
import re
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:            # also run as a script (the ALDM_PDL=0 child of test_encoder_pdl_matches_serialized_run)
    sys.path.insert(0, ROOT)

from audioldm2_b200 import _lib, arch, plan, synth
from oracle import clap as OC
from oracle import clap_audio as OA
from tests.conftest import rel_l2
from tests.golden import clap_audio_cases as CA
from tests.test_gpu_kernel_matrix import GUARD, Win, _assert_unchanged, _check
from tests.test_gpu_seqgen import Ws

DEV = "cuda:0"
TOL = 1e-4          # relative L2 per clip (docstring)

KERNEL_TESTS = {
    "htsat_logmel_kernel": "test_htsat_logmel",
    "htsat_patch_kernel": "test_htsat_patch",
    "htsat_window_attention_kernel": "test_htsat_window_attention",
    "htsat_merge_kernel": "test_htsat_merge",
    "htsat_head_kernel": "test_htsat_head",
}


def test_every_audio_kernel_has_a_test():
    """Inventory of csrc/audio/*.cu: every __global__ kernel is mapped to a test of this file, and no entry is stale."""
    found = set()
    for path in glob.glob(os.path.join(ROOT, "audioldm2_b200", "csrc", "audio", "*.cu")):
        found |= set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s+)?(\w+)", open(path).read()))
    assert found == set(KERNEL_TESTS), (sorted(found - set(KERNEL_TESTS)), sorted(set(KERNEL_TESTS) - found))
    mod = sys.modules[__name__]
    assert all(callable(getattr(mod, t, None)) for t in KERNEL_TESTS.values())


def _st():
    return torch.cuda.current_stream().cuda_stream


def _bounded(name, got, ref, rl2, rel_max):
    e = rel_l2(got, ref)
    m = float((got.double().cpu() - ref.double().cpu()).abs().max() / ref.double().abs().max())
    print(f"{name}: rel L2 {e:.3g}, max {m:.3g}")
    assert e < rl2 and m <= rel_max, (name, e, m)


# ----------------------------------------------------------------------------------------------
# kernels
# ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("sr,L", [(16000, 5120), (16000, 40000), (16000, 163840), (48000, 15360), (48000, 491520)])
def test_htsat_logmel(sr, L):
    """T = 33 (the shortest latent at 16 kHz) .. 1001 (10.24 s, truncated), both rates."""
    sd = CA.weights((2, 2, 2, 2))
    n = 2
    wav = CA.waveform(n, L, seed=L + sr)
    up = 48000 // sr
    L48 = min(up * L, 480000)
    T = L48 // 480 + 1
    a = "audio_branch"
    ts = [wav, plan.htsat_resample_taps(), sd[f"{a}.logmel_extractor.melW"]] + \
        [sd[f"{a}.bn0.{k}"] for k in ("running_mean", "running_var", "weight", "bias")]
    ws = Ws(sum(4 * t.numel() for t in ts) + 4 * n * T * 64 + 64 * GUARD)
    offs = [ws.put(t.float()) for t in ts]
    o_off = ws.alloc(4 * n * T * 64)
    before = ws.buf.clone()
    d = _lib.HtsatLogmelDesc(*[ws.ptr(o) for o in offs], out=ws.ptr(o_off), n=n, L=L, up=up, L48=L48, T=T, eps=1e-5)
    _lib.check(_lib.lib().aldm_htsat_logmel(d, _st()), "htsat_logmel")
    torch.cuda.synchronize()
    _assert_unchanged(ws.buf, before, [Win(o_off, n * T, 64, 64, 4)])
    got = ws.f32(o_off, n * T * 64).reshape(n, T, 64).cpu()
    x = wav.double()
    if sr != 48000:
        x = OA.resample_16k_to_48k(x)
    ref = OA.logmel({k: v.double() for k, v in sd.items()}, x[:, :480000])
    assert ref.shape == got.shape
    _bounded(f"logmel sr={sr} L={L}", got, ref, 1e-5, 1e-4)


@pytest.mark.gpu
def test_htsat_logmel_rejects_bad_shapes():
    d = _lib.HtsatLogmelDesc(wav=16, taps=16, melW=16, bn_mean=16, bn_var=16, bn_w=16, bn_b=16, out=16, n=1, L=170, up=3,
                             L48=510, T=2, eps=1e-5)
    assert _lib.lib().aldm_htsat_logmel(d, None) == -2           # ALDM_E_SHAPE: 510 samples cannot be reflect-padded
    d.L, d.L48, d.up = 600, 600, 2
    assert _lib.lib().aldm_htsat_logmel(d, None) != 0


@pytest.mark.gpu
@pytest.mark.parametrize("n,T", [(1, 33), (3, 501), (2, 1001)])
def test_htsat_patch(n, T):
    g = torch.Generator().manual_seed(n * 1000 + T)
    mel = torch.randn(n, T, 64, generator=g)
    w, b = torch.randn(128, 16, generator=g) / 4, 0.1 * torch.randn(128, generator=g)
    gamma, beta = 1 + 0.1 * torch.randn(128, generator=g), 0.1 * torch.randn(128, generator=g)
    ws = Ws(4 * (mel.numel() + w.numel() + 3 * 128) + 4 * n * 4096 * 128 + 64 * GUARD)
    offs = [ws.put(t) for t in (mel, w, b, gamma, beta)]
    o_off = ws.alloc(4 * n * 4096 * 128)
    before = ws.buf.clone()
    d = _lib.HtsatPatchDesc(*[ws.ptr(o) for o in offs], out=ws.ptr(o_off), n=n, T=T, eps=1e-5)
    _lib.check(_lib.lib().aldm_htsat_patch(d, _st()), "htsat_patch")
    torch.cuda.synchronize()
    _assert_unchanged(ws.buf, before, [Win(o_off, n * 4096, 128, 128, 4)])
    got = ws.f32(o_off, n * 4096 * 128).reshape(n, 4096, 128).cpu()
    rows, wt = plan.htsat_bicubic(T)                 # the fp32 source indices and weights the fp32 reference computes
    xt = (mel.double()[:, rows] * wt.double()[None, :, :, None]).sum(2)
    img = xt.permute(0, 2, 1).reshape(n, 64, 4, 256).permute(0, 2, 1, 3).reshape(n, 1, 256, 256)
    h = F.conv2d(img, w.double().reshape(128, 1, 4, 4), b.double(), stride=4).flatten(2).transpose(1, 2)
    ref = F.layer_norm(h, (128,), gamma.double(), beta.double(), 1e-5)
    _bounded(f"patch n={n} T={T}", got, ref, 1e-5, 1e-4)


ATT_CASES = [(R, shift, n) for R, n in ((64, 2), (32, 3), (16, 3), (8, 5)) for shift in ((0, 4) if R > 8 else (0,))]


@pytest.mark.gpu
@pytest.mark.parametrize("R,shift,n", ATT_CASES)
def test_htsat_window_attention(R, shift, n):
    """Every stage (R = 64, 32, 16, 8 with its heads), unshifted and shifted blocks."""
    stage = {64: 0, 32: 1, 16: 2, 8: 3}[R]
    H = arch.CLAP_AUDIO["heads"][stage]
    C = 32 * H
    g = torch.Generator().manual_seed(R * 10 + shift + n)
    rows = n * R * R
    qkv = torch.randn(rows, 3 * C, generator=g)
    qkv[:, :C] *= 2.0
    table = 0.5 * torch.randn(225, H, generator=g)
    bias = table[plan.htsat_relative_position_index().reshape(-1)].reshape(64, 64, H).permute(2, 0, 1).contiguous()
    mask = plan.htsat_shift_mask(R) if shift else None
    ldo = C + 8
    ws = Ws(4 * (qkv.numel() + bias.numel() + (mask.numel() if shift else 0)) + 4 * rows * ldo + 64 * GUARD)
    q_off, b_off = ws.put(qkv), ws.put(bias)
    m_off = ws.put(mask) if shift else None
    hi, lo = ws.alloc(2 * rows * ldo), ws.alloc(2 * rows * ldo)
    before = ws.buf.clone()
    d = _lib.HtsatAttnDesc(qkv=ws.ptr(q_off), bias=ws.ptr(b_off), mask=ws.ptr(m_off) if shift else None, out_hi=ws.ptr(hi),
                           out_lo=ws.ptr(lo), n=n, R=R, shift=shift, heads=H, head_dim=32, C=C, ld_qkv=3 * C, ldo=ldo,
                           scale=32 ** -0.5)
    _lib.check(_lib.lib().aldm_htsat_window_attention(d, _st()), "htsat_window_attention")
    torch.cuda.synchronize()
    _assert_unchanged(ws.buf, before, [Win(hi, rows, ldo, C, 2), Win(lo, rows, ldo, C, 2)])
    got = (ws.f16(hi, rows * ldo).float() + ws.f16(lo, rows * ldo).float()).reshape(rows, ldo)[:, :C]
    # float64 reference through the module's own roll / partition (oracle.clap_audio)
    x = qkv.double().view(n, R, R, 3 * C)
    if shift:
        x = torch.roll(x, (-shift, -shift), (1, 2))
    xw = OA.partition(x, 8).reshape(-1, 64, 3, H, 32).permute(2, 0, 3, 1, 4)
    q, k, v = xw[0] * torch.tensor(32 ** -0.5, dtype=torch.float32).double(), xw[1], xw[2]
    att = q @ k.transpose(-1, -2) + bias.double()[None]
    if shift:
        att = (att.view(n, -1, H, 64, 64) + mask.double()[None, :, None]).view(-1, H, 64, 64)
    o = (torch.softmax(att, -1) @ v).transpose(1, 2).reshape(-1, 8, 8, C)
    o = OA.unpartition(o, 8, R, R)
    if shift:
        o = torch.roll(o, (shift, shift), (1, 2))
    _check(f"htsat_attention R={R} shift={shift}", got, o.reshape(rows, C), planes=2)


@pytest.mark.gpu
def test_htsat_window_attention_rejects_bad_shapes():
    d = _lib.HtsatAttnDesc(qkv=16, bias=16, mask=16, out_hi=16, n=1, R=64, shift=4, heads=2, head_dim=64, C=128,
                           ld_qkv=384, ldo=128, scale=0.125)
    assert _lib.lib().aldm_htsat_window_attention(d, None) == -6     # ALDM_E_UNSUPPORTED: head_dim 64
    d.head_dim, d.heads, d.R = 32, 4, 60
    assert _lib.lib().aldm_htsat_window_attention(d, None) == -2     # ALDM_E_SHAPE: R not a multiple of 8


@pytest.mark.gpu
@pytest.mark.parametrize("R,C,n", [(64, 128, 2), (32, 256, 3), (16, 512, 5)])
def test_htsat_merge(R, C, n):
    """All three merge widths (4C = 512, 1024, 2048) at their production resolutions."""
    g = torch.Generator().manual_seed(R + C + n)
    x = torch.randn(n * R * R, C, generator=g) * 3 + torch.randn(n * R * R, 1, generator=g)
    gamma, beta = 1 + 0.1 * torch.randn(4 * C, generator=g), 0.1 * torch.randn(4 * C, generator=g)
    rows, ldo = n * R * R // 4, 4 * C + 8
    ws = Ws(4 * (x.numel() + 8 * C) + 4 * rows * ldo + 64 * GUARD)
    x_off, g_off, b_off = ws.put(x), ws.put(gamma), ws.put(beta)
    hi, lo = ws.alloc(2 * rows * ldo), ws.alloc(2 * rows * ldo)
    before = ws.buf.clone()
    d = _lib.HtsatMergeDesc(x=ws.ptr(x_off), gamma=ws.ptr(g_off), beta=ws.ptr(b_off), out_hi=ws.ptr(hi), out_lo=ws.ptr(lo),
                            n=n, R=R, C=C, ldo=ldo, eps=1e-5)
    _lib.check(_lib.lib().aldm_htsat_merge(d, _st()), "htsat_merge")
    torch.cuda.synchronize()
    _assert_unchanged(ws.buf, before, [Win(hi, rows, ldo, 4 * C, 2), Win(lo, rows, ldo, 4 * C, 2)])
    got = (ws.f16(hi, rows * ldo).float() + ws.f16(lo, rows * ldo).float()).reshape(rows, ldo)[:, :4 * C]
    xv = x.double().view(n, R, R, C)
    cat = torch.cat([xv[:, 0::2, 0::2], xv[:, 1::2, 0::2], xv[:, 0::2, 1::2], xv[:, 1::2, 1::2]], -1).reshape(rows, 4 * C)
    ref = F.layer_norm(cat, (4 * C,), gamma.double(), beta.double(), 1e-5)
    _check(f"htsat_merge C={C}", got, ref, planes=2)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 24])
def test_htsat_head(n):
    g = torch.Generator().manual_seed(n)
    C, Pj = 1024, 512
    x = torch.randn(n * 64, C, generator=g) * 2 + 0.5
    gamma, beta = 1 + 0.1 * torch.randn(C, generator=g), 0.1 * torch.randn(C, generator=g)
    w1, w2 = torch.randn(Pj, C, generator=g) / C ** 0.5, torch.randn(Pj, Pj, generator=g) / Pj ** 0.5
    b1, b2 = 0.1 * torch.randn(Pj, generator=g), 0.1 * torch.randn(Pj, generator=g)
    ts = [x, gamma, beta, w1.t().contiguous(), b1, w2.t().contiguous(), b2]
    ws = Ws(sum(4 * t.numel() for t in ts) + 4 * n * Pj + 64 * GUARD)
    offs = [ws.put(t) for t in ts]
    o_off = ws.alloc(4 * n * Pj)
    before = ws.buf.clone()
    d = _lib.HtsatHeadDesc(*[ws.ptr(o) for o in offs], out=ws.ptr(o_off), n=n, ntok=64, C=C, P=Pj, eps=1e-5)
    _lib.check(_lib.lib().aldm_htsat_head(d, _st()), "htsat_head")
    torch.cuda.synchronize()
    _assert_unchanged(ws.buf, before, [Win(o_off, n, Pj, Pj, 4)])
    m = F.layer_norm(x.double().view(n, 64, C), (C,), gamma.double(), beta.double(), 1e-5).mean(1)
    ref = F.normalize(torch.relu(m @ w1.double().t() + b1.double()) @ w2.double().t() + b2.double(), dim=-1)
    got = ws.f32(o_off, n * Pj).reshape(n, Pj).double().cpu()
    assert max(rel_l2(got[b], ref[b]) for b in range(n)) < 1e-5


# ----------------------------------------------------------------------------------------------
# the plan's GEMMs through the float64 checker of the kernel matrix
# ----------------------------------------------------------------------------------------------
GEMM_CLIPS = (3, 6, 12, 24)     # the clip counts the re-ranker (batchsize 1, 2, 4, 8 x 3 candidates) and the timing plan


@pytest.mark.gpu
@pytest.mark.parametrize("n", GEMM_CLIPS)
def test_plan_gemms(n, monkeypatch):
    """Every distinct GEMM descriptor of the full-depth plan of n clips of 10.24 s (tile width and split-K follow the row
    count) through the kernel matrix's float64 checker.  Planned here, not at collection."""
    from tests import test_gpu_kernel_matrix as KM
    from tests.test_gpu_production_shapes import _spec
    w = _enc(CA.BASE, 16000).weights
    specs = {}
    for o in plan.build_clap_audio(None, n, 163840, 16000, weights=w).ops:
        if o["kind"] == "gemm":
            s = _spec(dict(op=o))
            specs.setdefault(repr(sorted(s.items())), s)
    assert len(specs) >= 10
    for k, (_, spec) in enumerate(sorted(specs.items())):
        name = f"htsat_n{n}_{k}"
        monkeypatch.setitem(KM.GEMM_MATRIX, name, spec)
        KM.test_gemm_matrix(name)
        torch.cuda.empty_cache()


# ----------------------------------------------------------------------------------------------
# the encoder
# ----------------------------------------------------------------------------------------------
_ENCS = {}


def _enc(depths, sr, use_graph=True):
    from audioldm2_b200.clap import NativeCLAPAudioEncoder
    key = (depths, sr, use_graph)
    if key not in _ENCS:
        w = next((e.weights for k, e in _ENCS.items() if k[0] == depths), None)
        _ENCS[key] = NativeCLAPAudioEncoder(CA.weights(depths) if w is None else None, DEV, sampling_rate=sr,
                                            use_graph=use_graph, weights=w)
    return _ENCS[key]


def _per_clip(got, ref):
    return max(rel_l2(got[b], ref[b]) for b in range(ref.shape[0]))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CA.CASES))
def test_encoder_matches_reference(name):
    depths, sr, L, n, _ = CA.CASES[name]
    got = _enc(depths, sr).embed(CA.inputs(name).to(DEV)).cpu()
    assert torch.isfinite(got).all()
    e = _per_clip(got, CA.load()[name])
    print(f"{name}: rel L2 {e:.3g}")
    assert e < TOL


@pytest.mark.gpu
@pytest.mark.parametrize("sr", [16000, 48000])
def test_encoder_matches_float64_oracle_n24(sr):
    L = 163840 if sr == 16000 else 491520
    wav = CA.waveform(24, L, seed=sr + 3)
    got = _enc(CA.BASE, sr).embed(wav.to(DEV)).cpu()
    ref = OA.clap_audio_embed(CA.weights(CA.BASE), wav.to(DEV), sr, depths=CA.BASE, device=DEV).cpu()
    e = _per_clip(got, ref)
    print(f"n=24 sr={sr}: rel L2 {e:.3g}")
    assert e < TOL


@pytest.mark.gpu
def test_encoder_validates_input():
    enc = _enc(CA.SMALL, 16000)
    for bad in (torch.zeros(2, 1000, dtype=torch.float64), torch.zeros(1000), torch.zeros(1, 170)):
        with pytest.raises(ValueError):
            enc.embed(bad.to(DEV))
    with pytest.raises(ValueError):
        _enc(CA.SMALL, 48000).embed(torch.zeros(1, 512, device=DEV))


@pytest.mark.gpu
def test_encoder_bit_exact_properties():
    """Graph replay equals the eager run and a repeated replay; a clip permutation permutes the result exactly."""
    wav = CA.waveform(3, 40000, seed=11).to(DEV)
    enc = _enc(CA.BASE, 16000)
    base = enc.embed(wav)
    assert torch.equal(enc.embed(wav), base)
    assert torch.equal(_enc(CA.BASE, 16000, use_graph=False).embed(wav), base), "graph replay differs from the eager run"
    perm = torch.tensor([2, 0, 1], device=DEV)
    assert torch.equal(enc.embed(wav[perm]), base[perm])


def _pdl_embeds():
    wav = CA.waveform(2, 40000, seed=12).to(DEV)
    return _enc(CA.BASE, 16000, use_graph=False).embed(wav).cpu()


@pytest.mark.gpu
def test_encoder_pdl_matches_serialized_run(tmp_path):
    got = _pdl_embeds()
    path = str(tmp_path / "serial.pt")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), path]
    r = subprocess.run(cmd, env=dict(os.environ, ALDM_PDL="0"), cwd=ROOT, timeout=900,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    assert r.returncode == 0, r.stdout.decode(errors="replace")[-4000:]
    assert torch.equal(got, torch.load(path))


# ----------------------------------------------------------------------------------------------
# ranking
# ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_ranker_matches_reference_cos_similarity():
    """The seeded cos_similarity call of the fixtures: same similarity (within the encoders' bounds), same chosen
    indices, same replaced rows and the same CPU generator state afterwards."""
    from audioldm2_b200.clap import NativeCLAPRanker, NativeCLAPTextEncoder
    golden = CA.load()
    wav, texts, B = CA.rank_inputs()
    text = NativeCLAPTextEncoder(CA.text_weights(), DEV)
    rk = NativeCLAPRanker(_enc(CA.SMALL, 16000), text, synth.clap_tokenize)
    torch.manual_seed(int(golden["rank_seed"]))
    sim = rk(wav.to(DEV), texts).cpu()
    assert torch.equal(torch.get_rng_state(), golden["rank_rng_state"])
    assert (sim - golden["rank_similarity"]).abs().max() < 1e-4
    assert OA.select(sim, B) == golden["rank_best"].tolist()


# ----------------------------------------------------------------------------------------------
# end to end
# ----------------------------------------------------------------------------------------------
class _OracleRanker:
    """A callable ranker that runs oracle/clap_audio.py in float64 on the egressed waveform, with forward's draws."""

    def __init__(self, sd_a, sd_t, sr):
        self.sd_a, self.sd_t, self.sr = sd_a, sd_t, sr
        self.uncond = OC.clap_text_embed(sd_t, *synth.clap_tokenize([""]), 12, device=DEV).cpu()
        self.calls = []

    def __call__(self, waveform, texts):
        ids, mask = synth.clap_tokenize(list(texts))
        sim, ra, rt = OA.cos_similarity(
            lambda: OA.clap_audio_embed(self.sd_a, waveform.to(DEV), self.sr, device=DEV).cpu(),
            lambda: OC.clap_text_embed(self.sd_t, ids, mask, 12, device=DEV).cpu(), self.uncond)
        self.calls.append(sim)
        return sim


@pytest.mark.gpu
@pytest.mark.parametrize("model_name", ["audioldm_48k", "audioldm2-full"])
def test_text_to_audio_native_ranking(model_name):
    """batchsize 2, 3 candidates per prompt, synthetic weights: the native ranker returns the same waveform bytes and
    leaves the same CPU generator state as a callable ranker running the float64 oracle on the host copy; the top-two
    margin of every prompt exceeds the encoders' error bound, so the choice is determined."""
    from audioldm2_b200 import pipeline
    kw = dict(ddim_steps=4, batchsize=2, n_candidate_gen_per_text=3, duration=2.5, seed=5)
    ld = pipeline.build_model(model_name=model_name, clap_tokenize=synth.clap_tokenize)
    out = pipeline.text_to_audio(ld, "a dog barks", **kw)
    st = torch.get_rng_state()
    sr = ld.cfg["sampling_rate"]
    orc = _OracleRanker(synth.clap_audio_state_dict(), synth.clap_text_state_dict(), sr)
    ld2 = pipeline.build_model(model_name=model_name, ranker=orc)
    ref = pipeline.text_to_audio(ld2, "a dog barks", **kw)
    assert torch.equal(torch.get_rng_state(), st)
    sim = orc.calls[-1].reshape(3, 2)
    top = sim.sort(0, descending=True).values
    print(model_name, "similarity", sim.tolist())
    assert bool(((top[0] - top[1]) > 1e-3).all()), "seed the case so that the choice is determined"
    assert out.shape == ref.shape and out.tobytes() == ref.tobytes()


@pytest.mark.gpu
def test_rank_shards_with_native_ranking():
    """A sharded call (one rank per prompt, no process group) with 3 candidates per prompt: every rank makes the 2 x 6
    replacement draws of the whole call in global row order and ranks its own 3 candidates.  Each rank chooses the
    single-process call's candidate, its similarities are the single-process ones at its rows, the CPU generator state
    after the call is the single-process state, and its waveform equals the single-process row within the sharding
    tests' 1e-3 (the ranks run batch-3 engines instead of batch 6)."""
    from audioldm2_b200 import pipeline
    from audioldm2_b200.utils import seed_everything
    ld = pipeline.build_model(model_name="audioldm_48k", clap_tokenize=synth.clap_tokenize)
    ld.latent_t_size = 64
    batch = pipeline.make_batch_for_text_to_audio(["a dog barks", "rain on a tin roof"], batchsize=2)
    rk = ld.native_ranker()
    calls = []
    orig = rk.__call__

    class Recording:
        def __call__(self, waveform, texts, rows=None, n_total=None):
            sim = orig(waveform, texts, rows=rows, n_total=n_total)
            calls.append((rows, n_total, list(texts), sim.cpu()))
            return sim

    ld._native_ranker = Recording()
    seed_everything(7)
    full = ld._generate_local(batch, 4, 1.0, 3, 3.5, None, None, None, None)
    st_full = torch.get_rng_state()
    rows_f, n_f, texts_f, sim_f = calls[-1]
    assert rows_f is None and n_f == 6 and len(texts_f) == 6
    best_f = OA.select(sim_f, 2)
    print("single process: similarity", sim_f.tolist(), "best", best_f)
    for r in range(2):
        seed_everything(7)
        part = ld._generate_sharded((r, 2, r, r + 1), batch, 4, 1.0, 3, 3.5, None, None, None)
        assert torch.equal(torch.get_rng_state(), st_full), r
        rows, n_total, texts, sim = calls[-1]
        assert rows == [r, r + 2, r + 4] and n_total == 6 and texts == [texts_f[g] for g in rows]
        assert (sim - sim_f[rows]).abs().max() < 1e-3, (r, sim.tolist(), sim_f[rows].tolist())
        k = int(torch.argmax(sim))
        assert rows[k] == best_f[r], (r, rows[k], best_f)
        assert part.shape == (1,) + full.shape[1:]
        assert rel_l2(torch.from_numpy(part), torch.from_numpy(full[r:r + 1])) < 1e-3, r


if __name__ == "__main__":            # ALDM_PDL=0 child of test_encoder_pdl_matches_serialized_run
    torch.save(_pdl_embeds(), sys.argv[1])
