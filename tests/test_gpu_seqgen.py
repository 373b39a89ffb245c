"""The AudioMAE token generator on the GPU: its kernels (csrc/cond/*.cu) and the GELU-tanh GEMM epilogue against float64,
inside 4 KB guard bands; the whole stage against the reference fixtures and the float64 oracle; bit-exact properties.

Bounds (relative L2 AND per element, as tests/test_gpu_kernel_matrix.py):
  * kv_attention_kernel: q, k, v are fp32 (the c_attn GEMM's fp32 output), the reference uses the same fp32 values in
    float64.  Scores carry the fp32 dot-product error (64 terms, <= 2^-21 sum |q_i k_i| / 8, ~1e-6 for O(1) inputs), the
    exponentials expf's 2 ulp, the P V sum ~nk 2^-24 sum p |v|; the output is split into two fp16 planes (2^-22).  So the
    two-plane budget holds: relative L2 < 2e-5 and |err| <= 1e-4 rms(ref), a 10x margin at 1024 keys.
  * seq_feedback_kernel: two-pass fp32 LayerNorm.  The rows have |mean| / std = 30, so every centred value carries the
    rounding of the fp32 mean: a few units of 2^-24 |mean| = 30 x 2^-24 std ~ 2e-6 std (times rstd |g|), the same shift
    for the whole row; rstd and the affine step add a few ulp of |ref|.  Bounds: relative L2 < 8e-6 (2^-17, twice the
    worst mean error of 4 units), |err| <= 1e-5 rms(ref) + 2^-19 |ref| per element.
  * seq_assemble_kernel: one fp32 addition per element, compared bit for bit with the same addition in torch.
  * GELU-tanh GEMM: the GEMM bound of the matrix test (2e-5 / 1e-4 rms for fp32 and two-plane outputs); gelu_new has slope
    <= 1.13, and tanhf is accurate to 2 ulp, so the activation adds < 2^-21 |ref|.
The stage: the relative L2 per generated token is below 2e-5 against the reference fixtures (fp32 torch on the CPU) and
against the float64 oracle: two-plane GEMM operands cost ~2e-6 (measured by CPU emulation), the remaining fp32 rounding
below that.
"""
import glob
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:            # also run as a script (the ALDM_PDL=0 child of test_stage_pdl_matches_serialized_run)
    sys.path.insert(0, ROOT)

from audioldm2_b200 import _lib, arch, engine, plan, pipeline, synth
from audioldm2_b200.packing import round_up
from audioldm2_b200.plan import F32, Planner, Ref
from oracle import seqgen as OS
from tests.conftest import rel_l2
from tests.golden import seqgen_cases as SC
from tests.test_gpu_kernel_matrix import GUARD, Win, _assert_unchanged, _check, _guarded, _guarded_planes, _run_guarded

DEV = "cuda:0"
TOL = 2e-5

# kernel -> the test of this file that runs it against a float64 reference
KERNEL_TESTS = {
    "kv_attention_kernel": "test_kv_attention",
    "seq_assemble_kernel": "test_seq_assemble",
    "seq_feedback_kernel": "test_seq_feedback",
}


def test_every_cond_kernel_has_a_test():
    """Inventory of csrc/cond/*.cu: every __global__ kernel is mapped to a test of this file, and no entry is stale."""
    found = set()
    for path in glob.glob(os.path.join(ROOT, "audioldm2_b200", "csrc", "cond", "*.cu")):
        found |= set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s+)?(\w+)", open(path).read()))
    assert found == set(KERNEL_TESTS), (sorted(found - set(KERNEL_TESTS)), sorted(set(KERNEL_TESTS) - found))
    mod = sys.modules[__name__]
    assert all(callable(getattr(mod, t, None)) for t in KERNEL_TESTS.values())


class Ws:
    """A 0xFF-filled device workspace with guarded regions (GUARD bytes before and after each)."""

    def __init__(self, nbytes):
        self.buf = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device=DEV)
        self.top = 0

    def alloc(self, nbytes):
        off = self.top + GUARD
        self.top = off + round_up(nbytes, 256) + GUARD
        assert self.top <= self.buf.numel()
        return off

    def put(self, t):
        b = t.contiguous().view(torch.uint8).reshape(-1)
        off = self.alloc(b.numel())
        self.buf[off:off + b.numel()].copy_(b.to(DEV))
        return off

    def ptr(self, off):
        return self.buf.data_ptr() + off

    def f32(self, off, n):
        return self.buf[off:off + 4 * n].view(torch.float32)

    def f16(self, off, n):
        return self.buf[off:off + 2 * n].view(torch.float16)


def _st():
    return torch.cuda.current_stream().cuda_stream


# ----------------------------------------------------------------------------------------------
# kv_attention_kernel
# ----------------------------------------------------------------------------------------------
KV_CASES = [(1, 6), (3, 37), (8, 133), (3, 1024), (8, 1024)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["prefill", "decode"])
@pytest.mark.parametrize("B,P", KV_CASES)
def test_kv_attention(B, P, mode):
    g = torch.Generator().manual_seed(B * 7919 + P)
    H, C = 12, 768
    lmax = min(P + 8, 1024)
    p0, nq = (0, P) if mode == "prefill" else (P - 1, 1)
    seq = torch.full((B, lmax, 3 * C), float("nan"))                # positions >= p0 + nq are never read
    seq[:, :P] = torch.randn(B, P, 3 * C, generator=g)
    seq[:, :P, :C] *= 2.0                                           # scores of a few units: a peaked softmax
    mask = (torch.rand(B, lmax, generator=g) < 0.8).float()
    mask[:, 0] = 1
    for b in range(B):                                              # a padded tail per row, like ragged T5 inputs
        mask[b, max(1, P - 1 - 5 * b):max(1, P - 1)] = 0
    mask[:, P:] = 1
    ws = Ws(2 * 4 * B * lmax * 3 * C + 4 * B * nq * C + 64 * GUARD)
    s_off, m_off = ws.put(seq), ws.put(mask)
    o_hi, o_lo = ws.alloc(2 * B * nq * C), ws.alloc(2 * B * nq * C)
    before = ws.buf.clone()
    d = _lib.KvAttnDesc(seq=ws.ptr(s_off), mask=ws.ptr(m_off), out_hi=ws.ptr(o_hi), out_lo=ws.ptr(o_lo), B=B, heads=H,
                        lmax=lmax, ld_seq=3 * C, p0=p0, nq=nq, ldo=C, scale=0.125)
    _lib.check(_lib.lib().aldm_kv_attention(d, _st()), "kv_attention")
    torch.cuda.synchronize()
    wins = [Win(o_hi, B * nq, C, C, 2), Win(o_lo, B * nq, C, C, 2)]
    _assert_unchanged(ws.buf, before, wins)
    got = ws.f16(o_hi, B * nq * C).float() + ws.f16(o_lo, B * nq * C).float()
    s64 = seq.double()
    nk = p0 + nq
    q = s64[:, p0:nk, :C].reshape(B, nq, H, 64).transpose(1, 2)
    k = s64[:, :nk, C:2 * C].reshape(B, nk, H, 64).transpose(1, 2)
    v = s64[:, :nk, 2 * C:].reshape(B, nk, H, 64).transpose(1, 2)
    keep = (torch.arange(nk)[None, :] <= (p0 + torch.arange(nq))[:, None])[None, None] & (mask[:, None, None, :nk] == 1)
    w = (q @ k.transpose(-1, -2) / 8.0).masked_fill(~keep, float("-inf"))
    ref = (torch.softmax(w, -1) @ v).transpose(1, 2).reshape(B * nq, C)
    _check(f"kv_attention B={B} P={P} {mode}", got, ref, planes=2)


@pytest.mark.gpu
def test_kv_attention_rejects_bad_shapes():
    d = _lib.KvAttnDesc(seq=16, mask=16, out_hi=16, B=1, heads=12, lmax=1025, ld_seq=2304, p0=0, nq=1, ldo=768, scale=0.125)
    assert _lib.lib().aldm_kv_attention(d, None) == -2
    d.lmax, d.p0, d.nq = 64, 60, 8
    assert _lib.lib().aldm_kv_attention(d, None) == -2


# ----------------------------------------------------------------------------------------------
# seq_assemble_kernel / seq_feedback_kernel
# ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("B,L", [(1, 1), (3, 32), (8, 128)])
def test_seq_assemble(B, L):
    g = torch.Generator().manual_seed(B + L)
    C, Pn = 768, L + 5
    lmax = Pn + 8
    x = torch.full((B, Pn, C), float("nan"))
    x[:, 1] = torch.randn(B, C, generator=g)
    x[:, 4:4 + L] = torch.randn(B, L, C, generator=g)
    sos, eos, wpe = torch.randn(2, C, generator=g), torch.randn(2, C, generator=g), 0.02 * torch.randn(1024, C, generator=g)
    t5m = (torch.rand(B, L, generator=g) < 0.7).float()
    ws = Ws(4 * (2 * B * Pn * C + 1024 * C + 8 * C + B * (L + lmax)) + 64 * GUARD)
    x_off, s_off, e_off, w_off, t_off = ws.put(x), ws.put(sos), ws.put(eos), ws.put(wpe), ws.put(t5m)
    m_off = ws.alloc(4 * B * lmax)
    before = ws.buf.clone()
    d = _lib.SeqAssembleDesc(x=ws.ptr(x_off), sos=ws.ptr(s_off), eos=ws.ptr(e_off), wpe=ws.ptr(w_off), t5_mask=ws.ptr(t_off),
                             mask=ws.ptr(m_off), B=B, L=L, lmax=lmax, C=C)
    _lib.check(_lib.lib().aldm_seq_assemble(d, _st()), "seq_assemble")
    torch.cuda.synchronize()
    _assert_unchanged(ws.buf, before, [Win(x_off, B * Pn, C, C, 4), Win(m_off, B, lmax, lmax, 4)])
    want = x.clone()
    want[:, 0], want[:, 2], want[:, 3], want[:, Pn - 1] = sos[0], eos[0], sos[1], eos[1]
    want = want + wpe[:Pn]
    assert torch.equal(ws.f32(x_off, B * Pn * C).cpu().reshape(B, Pn, C), want)
    wm = torch.ones(B, lmax)
    wm[:, 4:4 + L] = t5m
    assert torch.equal(ws.f32(m_off, B * lmax).cpu().reshape(B, lmax), wm)


@pytest.mark.gpu
@pytest.mark.parametrize("B,nq,last", [(1, 6, False), (3, 37, False), (8, 1, False), (8, 1, True)])
def test_seq_feedback(B, nq, last):
    g = torch.Generator().manual_seed(B * 31 + nq)
    C, gen, k, pos = 768, 8, 3, 500
    x = torch.randn(B * nq, C, generator=g) + 30.0 * torch.randn(B * nq, 1, generator=g).sign()     # |mean| / std = 30
    gamma, beta = 1 + 0.1 * torch.randn(C, generator=g), 0.02 * torch.randn(C, generator=g)
    wpe = 0.02 * torch.randn(1024, C, generator=g)
    ws = Ws(4 * (B * nq * C + 1030 * C + B * gen * C + B * C) + 64 * GUARD)
    x_off, g_off, b_off, w_off = ws.put(x), ws.put(gamma), ws.put(beta), ws.put(wpe)
    o_off, n_off = ws.alloc(4 * B * gen * C), ws.alloc(4 * B * C)
    before = ws.buf.clone()
    d = _lib.SeqFeedbackDesc(x=ws.ptr(x_off), gamma=ws.ptr(g_off), beta=ws.ptr(b_off), wpe=ws.ptr(w_off), out=ws.ptr(o_off),
                             next=None if last else ws.ptr(n_off), B=B, nq=nq, C=C, pos=pos, k=k, gen_len=gen, eps=1e-5)
    _lib.check(_lib.lib().aldm_seq_feedback(d, _st()), "seq_feedback")
    torch.cuda.synchronize()
    wins = [Win(o_off, B * gen, C, C, 4, rows=torch.arange(B) * gen + k)] + ([] if last else [Win(n_off, B, C, C, 4)])
    _assert_unchanged(ws.buf, before, wins)
    xl = x.double().reshape(B, nq, C)[:, -1]
    ref = torch.nn.functional.layer_norm(xl, (C,), gamma.double(), beta.double(), 1e-5)
    for name, off, want in [("token", o_off, ref)] + ([] if last else [("next", n_off, ref + wpe[pos + 1].double())]):
        got = ws.f32(off, B * gen * C).reshape(B, gen, C)[:, k] if name == "token" else ws.f32(off, B * C).reshape(B, C)
        got = got.double().cpu()
        assert rel_l2(got, want) < 8e-6, name
        bound = 1e-5 * float(want.pow(2).mean().sqrt()) + 2.0 ** -19 * want.abs()
        assert ((got - want).abs() <= bound).all(), name


# ----------------------------------------------------------------------------------------------
# GEMM with ALDM_ACT_GELU_TANH: the generic epilogue body, with and without split-K
# ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("bn,splitk,planes_out", [(32, 1, True), (64, 1, False), (128, 1, True), (32, 3, True), (128, 4, False)])
def test_gemm_gelu_tanh(bn, splitk, planes_out):
    g = torch.Generator().manual_seed(bn * 10 + splitk)
    M, K, N = 333, 768, 384
    P = Planner()
    a = _guarded_planes(P, M, K, 2)
    w = torch.randn(N, K, generator=g) / K ** 0.5
    bias = 0.02 * torch.randn(N, generator=g)
    wm = P.wmat(w, bias, 1, K, bn=bn)
    out = _guarded_planes(P, M, N, 2) if planes_out else None
    out_f = None if planes_out else F32(_guarded(P, M * N * 4), M, N)
    o = P.gemm(a, wm, B=1, H=M, act=_lib.ACT_GELU_TANH, out_planes=out, out=out_f)
    scratch, zero = [], []
    if splitk > 1:
        nbytes = splitk * round_up(M, 128) * round_up(N, bn) * 4
        o["splitk"], o["ws"] = splitk, _guarded(P, nbytes + GUARD)
        scratch, zero = [(o["ws"].off, nbytes)], [(o["ws"].off, nbytes + GUARD)]
    pl = P.finish({})
    d = pl.resolve(1 << 20, 1 << 30)[0].u.gemm              # addresses only need to be non-null and aligned
    bn_, epi, ap, red, store = _lib.gemm_variant(d)
    assert (bn_, epi, ap, red) == (bn, _lib.EPI_GENERIC, 2, _lib.RED_GENERIC if splitk > 1 else _lib.RED_NONE)
    x = torch.randn(M, K, generator=g)
    from audioldm2_b200.packing import split_f16
    hi, lo = split_f16(x)
    writes = [(a.hi.off, hi), (a.lo.off, lo)]
    wins = [Win(out.hi.off, M, N, N, 2), Win(out.lo.off, M, N, N, 2)] if planes_out else [Win(out_f.ref.off, M, N, N, 4)]
    prog = _run_guarded(pl, writes, wins, zero=zero, scratch=scratch)
    ws = prog.ws
    if planes_out:
        got = ws[out.hi.off:out.hi.off + 2 * M * N].view(torch.float16).float() + ws[out.lo.off:out.lo.off + 2 * M * N].view(torch.float16).float()
    else:
        got = ws[out_f.ref.off:out_f.ref.off + 4 * M * N].view(torch.float32)
    ref = OS.gelu_new((hi.double() + lo.double()) @ w.double().t() + bias.double())
    _check(f"gelu_tanh bn={bn} splitk={splitk}", got.reshape(M, N), ref, planes=2 if planes_out else 0)


# ----------------------------------------------------------------------------------------------
# the stage
# ----------------------------------------------------------------------------------------------
_GENS = {}


def _gen(n_layer, use_graph=True):
    from audioldm2_b200.seqgen import NativeAudioMAEGenerator
    key = (n_layer, use_graph)
    if key not in _GENS:
        _GENS[key] = NativeAudioMAEGenerator(SC.weights(n_layer), DEV, use_graph=use_graph)
    return _GENS[key]


def _per_token(got, ref):
    return max(rel_l2(got[:, k], ref[:, k]) for k in range(ref.shape[1]))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SC.CASES))
def test_stage_matches_reference(name):
    golden = SC.load()
    n_layer = SC.CASES[name][0]
    got = _gen(n_layer).generate(*[t.to(DEV) for t in SC.inputs(name)]).cpu()
    assert torch.isfinite(got).all()
    assert _per_token(got, golden[name]) < TOL


@pytest.mark.gpu
def test_stage_matches_float64_oracle_b8_l128():
    lens = [128, 100, 77, 64, 31, 12, 5, 1]
    clap, t5, mask = synth.encoder_outputs(8, lens, seed=99)
    got = _gen(12).generate(clap.to(DEV), t5.to(DEV), mask.to(DEV)).cpu()
    ref = OS.audiomae_generate(SC.weights(12), clap.double(), t5.double(), mask.double(), 12)
    assert _per_token(got, ref) < TOL


@pytest.mark.gpu
def test_stage_bit_exact_properties():
    lens = [32, 9, 20]
    clap, t5, mask = (t.to(DEV) for t in synth.encoder_outputs(3, lens, seed=5))
    gen = _gen(12)
    base = gen.generate(clap, t5, mask)
    perm = torch.tensor([2, 0, 1], device=DEV)
    assert torch.equal(gen.generate(clap[perm], t5[perm], mask[perm]), base[perm]), "row permutation"
    t5b = torch.where(mask[..., None] == 1, t5, 1e3 * torch.randn_like(t5))
    assert torch.equal(gen.generate(clap, t5b, mask), base), "masked T5 values changed the output"
    assert torch.equal(_gen(12, use_graph=False).generate(clap, t5, mask), base), "graph replay differs from the eager run"


def _pdl_tokens():
    clap, t5, mask = (t.to(DEV) for t in synth.encoder_outputs(2, [40, 13], seed=6))
    return _gen(12, use_graph=False).generate(clap, t5, mask).cpu()


@pytest.mark.gpu
def test_stage_pdl_matches_serialized_run(tmp_path):
    got = _pdl_tokens()
    path = str(tmp_path / "serial.pt")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), path]
    r = subprocess.run(cmd, env=dict(os.environ, ALDM_PDL="0"), cwd=ROOT, timeout=900, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT)
    assert r.returncode == 0, r.stdout.decode(errors="replace")[-4000:]
    assert torch.equal(got, torch.load(path))


# ----------------------------------------------------------------------------------------------
# end to end
# ----------------------------------------------------------------------------------------------
class _Boundary:
    """UNet-boundary provider carrying given AudioMAE tokens next to the encoder provider's T5 states."""

    def __init__(self, enc, tokens):
        self.enc, self.tokens = enc, tokens

    def cond(self, batch):
        c = self.enc.cond(batch)
        return {"crossattn_audiomae_generated": [self.tokens, torch.ones(self.tokens.shape[:2], device=self.tokens.device)],
                "crossattn_flan_t5": c["crossattn_flan_t5"]}

    def uncond(self, n):
        return self.enc.uncond(n)


@pytest.mark.gpu
def test_text_to_audio_with_encoder_outputs():
    """audioldm2-full, B = 2, 10 DDIM steps, 3 candidates per prompt.  (1) Encoder outputs give the same waveform bits as
    a UNet-boundary provider carrying the native tokens, and that provider never builds the generator.  (2) Against the
    same call with the float64 oracle's tokens, the waveform is within 1e-3 relative L2: the token error does not grow
    through the sampler past the path's budget.  (The UNet / VAE / vocoder path itself is checked against its oracle by
    tests/test_gpu_nets.py.)"""
    cfg = arch.model_config("audioldm2-full")
    enc = pipeline.SyntheticEncoderOutputs(cfg, t5_lens=(32, 19), device=DEV)
    ld = pipeline.build_model(model_name="audioldm2-full", cond_provider=enc)
    kw = dict(batchsize=2, ddim_steps=10, n_candidate_gen_per_text=3, duration=2.5)
    with pytest.warns(UserWarning):
        wave = pipeline.text_to_audio(ld, "a dog barks", **kw)
    batch = {"text": ["a", "b"]}
    c = enc.cond(batch)
    native = ld.seqgen().generate(c["film_clap_cond1"], *c["crossattn_flan_t5"])
    oracle = OS.audiomae_generate(synth.seqgen_state_dict(), *[t.double().cpu() for t in (c["film_clap_cond1"],) + tuple(c["crossattn_flan_t5"])])
    for tokens, exact in ((native, True), (oracle.float().to(DEV), False)):
        ld2 = pipeline.build_model(model_name="audioldm2-full", cond_provider=_Boundary(enc, tokens))
        with pytest.warns(UserWarning):
            w2 = pipeline.text_to_audio(ld2, "a dog barks", **kw)
        assert ld2._seqgen is None, "a UNet-boundary provider built the generator"
        if exact:
            assert np.array_equal(w2, wave), "encoder outputs and native tokens at the UNet boundary differ"
        else:
            assert rel_l2(torch.from_numpy(wave), torch.from_numpy(w2)) < 1e-3
        del ld2
        torch.cuda.empty_cache()


@pytest.mark.gpu
def test_rank_shards_with_encoder_outputs():
    """A sharded call (one rank per prompt; no process group, so each rank's rows come back as they are) generates the
    AudioMAE tokens for the whole call on every rank -- the same (B, L) plan and bits as one process -- and keeps its
    rows.  Its waveform equals the single-process call's rows within the sharding test's 1e-3 (tests/test_gpu_nets.py:
    the UNet's split-K choices depend on the batch)."""
    from audioldm2_b200.utils import seed_everything
    cfg = arch.model_config("audioldm2-full")
    enc = pipeline.SyntheticEncoderOutputs(cfg, t5_lens=(32, 11), device=DEV)
    ld = pipeline.build_model(model_name="audioldm2-full", cond_provider=enc)
    ld.latent_t_size = 64
    batch = pipeline.make_batch_for_text_to_audio(["a", "b"], batchsize=2)
    gen = ld.seqgen()
    seen = []
    orig = gen.generate

    def recording(clap, t5, mask):
        out = orig(clap, t5, mask)
        seen.append((tuple(t5.shape), out.clone()))
        return out

    gen.generate = recording
    seed_everything(42)
    full = ld._generate_local(batch, 5, 1.0, 1, 3.5, None, None, None, None)
    for r in range(2):
        seed_everything(42)
        part = ld._generate_sharded((r, 2, r, r + 1), batch, 5, 1.0, 1, 3.5, None, None, None)
        assert part.shape == (1,) + full.shape[1:]
        assert rel_l2(torch.from_numpy(part), torch.from_numpy(full[r:r + 1])) < 1e-3, r
    assert [sh for sh, _ in seen] == [(2, 32, 1024)] * 3, "a rank generated for its own rows only"
    assert all(torch.equal(t, seen[0][1]) for _, t in seen), "the ranks' tokens differ from the single-process tokens"


if __name__ == "__main__":          # child of test_stage_pdl_matches_serialized_run
    assert os.environ.get("ALDM_PDL") == "0"
    torch.save(_pdl_tokens(), sys.argv[1])
