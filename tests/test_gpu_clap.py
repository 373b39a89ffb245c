"""The CLAP text encoder on the GPU: its kernels (csrc/clap/*.cu) against float64 inside 4 KB guard bands, the whole stage
against the reference fixtures and the float64 oracle, bit-exact properties and the pipeline end to end.

Bounds (relative L2 AND per element, as tests/test_gpu_kernel_matrix.py):
  * clap_embed_kernel: a gather and two fp32 adds in HF's order, compared bit for bit with torch's fp32 sum, HF position
    ids included.
  * clap_layernorm_kernel: two fixed-order fp32 sums of C = 768 terms (24 sequential per lane, then a 5-level tree):
    the mean carries ~30 x 2^-24 of sum |x| / C, the variance of the centred values ~30 x 2^-24 relative, half of that
    in 1/sqrt, then two roundings in (x - mean) * r * gamma + beta: a few 1e-6 of max |y|.  fp32 output: relative L2
    < 2e-6 and |err| <= 4e-6 max |ref|.  Plane output: the two-plane split adds 2^-22, inside the matrix's two-plane
    budget (2e-5 / 1e-4 rms).
  * clap_attention_kernel: q, k, v are fp32 (the QKV GEMM's fp32 output), the reference uses the same values in float64.
    The scores carry the fp32 error of a 64-term dot product (<= 64 x 2^-24 sum |q_i k_i|, scaled by the exact 1/8),
    which moves each probability by that relative amount; expf adds 2 ulp, the P V sum over <= 512 keys
    ~512 x 2^-24 sum p |v|, the split 2^-22: the two-plane budget.
  * clap_gelu_kernel: erff (2 ulp) times fp32 products, then the split: the two-plane budget.
  * clap_head_kernel: three fp32 dot products of <= 768 terms in order (<= 768 x 2^-24 of sum |w x| each), tanh
    (2 ulp) and the normalisation: relative L2 < 1e-5 per row against float64.
The stage: relative L2 per batch row below 3e-5 against the reference fixtures (fp32 torch on the CPU, all 512
positions) and against the float64 oracle at B = 8 with ragged rows and one 512-token row, 12 blocks.  CPU emulation of
the planned program (fp16 two-plane GEMM operands, fp32 arithmetic, tests/test_clap_cpu.py's emulator) measures the cost
of the two-plane operands and of the trim at 1.1e-6 to 1.4e-6 per row against float64 on the 2-block cases and 2.3e-6
to 2.9e-6 on the 12-block ones; the tensor cores' truncating accumulation (tests/test_gpu_kernel_matrix.py) adds at
most ~1e-6 per GEMM, so 3e-5 leaves a margin of about 5x.
"""
import glob
import os
import re
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:            # also run as a script (the ALDM_PDL=0 child of test_stage_pdl_matches_serialized_run)
    sys.path.insert(0, ROOT)

from audioldm2_b200 import _lib, arch, pipeline, synth
from oracle import clap as OC
from tests.conftest import rel_l2
from tests.golden import clap_cases as CC
from tests.test_gpu_kernel_matrix import GUARD, Win, _assert_unchanged, _check
from tests.test_gpu_seqgen import Ws

DEV = "cuda:0"
TOL = 3e-5          # relative L2 per batch row (docstring)

# kernel -> the test of this file that runs it against a float64 reference
KERNEL_TESTS = {
    "clap_embed_kernel": "test_clap_embed",
    "clap_layernorm_kernel": "test_clap_layernorm",
    "clap_attention_kernel": "test_clap_attention",
    "clap_gelu_kernel": "test_clap_gelu",
    "clap_head_kernel": "test_clap_head",
}


def test_every_clap_kernel_has_a_test():
    """Inventory of csrc/clap/*.cu: every __global__ kernel is mapped to a test of this file, and no entry is stale."""
    found = set()
    for path in glob.glob(os.path.join(ROOT, "audioldm2_b200", "csrc", "clap", "*.cu")):
        found |= set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s+)?(\w+)", open(path).read()))
    assert found == set(KERNEL_TESTS), (sorted(found - set(KERNEL_TESTS)), sorted(set(KERNEL_TESTS) - found))
    mod = sys.modules[__name__]
    assert all(callable(getattr(mod, t, None)) for t in KERNEL_TESTS.values())


def _st():
    return torch.cuda.current_stream().cuda_stream


# ----------------------------------------------------------------------------------------------
# kernels
# ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("B,L", [(1, 1), (3, 37), (2, 512)])
def test_clap_embed(B, L):
    g = torch.Generator().manual_seed(B * 7 + L)
    V, NP, C = 1000, 514, 768
    word, pos, typ = torch.randn(V, C, generator=g), torch.randn(NP, C, generator=g), torch.randn(C, generator=g)
    ids = torch.randint(0, V, (B, L), generator=g)
    ids[:, 0] = 0
    if L > 4:                                          # interior pad ids, and a padded tail
        ids[0, 2] = 1
        ids[-1, L // 2:] = 1
        ids[-1, L - 3] = 7
    ws = Ws(4 * (V * C + NP * C + C + 2 * B * L * C) + 8 * B * L + 64 * GUARD)
    w_off, p_off, t_off, i_off = ws.put(word), ws.put(pos), ws.put(typ), ws.put(ids)
    o_off = ws.alloc(4 * B * L * C)
    before = ws.buf.clone()
    d = _lib.ClapEmbedDesc(ids=ws.ptr(i_off), word=ws.ptr(w_off), pos=ws.ptr(p_off), type=ws.ptr(t_off), out=ws.ptr(o_off),
                           B=B, L=L, vocab=V, n_pos=NP, C=C, pad=1)
    _lib.check(_lib.lib().aldm_clap_embed(d, _st()), "clap_embed")
    torch.cuda.synchronize()
    _assert_unchanged(ws.buf, before, [Win(o_off, B * L, C, C, 4)])
    want = (word[ids] + typ) + pos[OC.position_ids(ids)]
    assert torch.equal(ws.f32(o_off, B * L * C).cpu().reshape(B, L, C), want)
    # an id the host failed to reject gives a NaN row, never a read outside the table
    ws.buf[i_off:i_off + 8].copy_(torch.tensor([V], dtype=torch.int64).view(torch.uint8).to(DEV))
    _lib.check(_lib.lib().aldm_clap_embed(d, _st()), "clap_embed")
    torch.cuda.synchronize()
    assert torch.isnan(ws.f32(o_off, C)).all()


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [1, 333, 4096])
def test_clap_layernorm(rows):
    g = torch.Generator().manual_seed(rows)
    C, eps = 768, 1e-5
    x = torch.randn(rows, C, generator=g) * (1 + 10 * torch.rand(rows, 1, generator=g)) + 3 * torch.randn(rows, 1, generator=g)
    gamma, beta = 1 + 0.1 * torch.randn(C, generator=g), 0.1 * torch.randn(C, generator=g)
    ldo = C + 8
    ws = Ws(4 * (rows * C + 2 * C) + 4 * rows * C + 4 * rows * ldo + 64 * GUARD)
    x_off, g_off, b_off = ws.put(x), ws.put(gamma), ws.put(beta)
    of, hi, lo = ws.alloc(4 * rows * C), ws.alloc(2 * rows * ldo), ws.alloc(2 * rows * ldo)
    before = ws.buf.clone()
    d = _lib.ClapLnDesc(x=ws.ptr(x_off), gamma=ws.ptr(g_off), beta=ws.ptr(b_off), out_f32=ws.ptr(of), out_hi=ws.ptr(hi),
                        out_lo=ws.ptr(lo), rows=rows, C=C, ldo=ldo, eps=eps)
    _lib.check(_lib.lib().aldm_clap_layernorm(d, _st()), "clap_layernorm")
    torch.cuda.synchronize()
    _assert_unchanged(ws.buf, before, [Win(of, rows, C, C, 4), Win(hi, rows, ldo, C, 2), Win(lo, rows, ldo, C, 2)])
    ref = torch.nn.functional.layer_norm(x.double(), (C,), gamma.double(), beta.double(), eps)
    got = ws.f32(of, rows * C).reshape(rows, C).double().cpu()
    assert rel_l2(got, ref) < 2e-6
    assert ((got - ref).abs() <= 4e-6 * ref.abs().amax(1, keepdim=True)).all()
    pl = (ws.f16(hi, rows * ldo).float() + ws.f16(lo, rows * ldo).float()).reshape(rows, ldo)[:, :C]
    _check(f"clap_layernorm rows={rows}", pl, ref, planes=2)


ATT_CASES = [(1, 1), (3, 37), (2, 130), (8, 512)]


@pytest.mark.gpu
@pytest.mark.parametrize("B,L", ATT_CASES)
def test_clap_attention(B, L):
    g = torch.Generator().manual_seed(B * 131 + L)
    H, C = 12, 768
    qkv = torch.randn(B * L, 3 * C, generator=g)
    qkv[:, :C] *= 2.0                                               # logits q.k / 8 of a few units: a peaked softmax
    mask = torch.ones(B, L)
    for b in range(B):                                              # ragged rows, and scattered padding
        mask[b, max(1, L - 37 * b):] = 0
    mask[:, 1:] *= (torch.rand(B, L - 1, generator=g) < 0.9).float()
    ws = Ws(4 * (B * L * 3 * C + B * L) + 4 * B * L * C + 64 * GUARD)
    q_off, m_off = ws.put(qkv), ws.put(mask)
    hi, lo = ws.alloc(2 * B * L * C), ws.alloc(2 * B * L * C)
    before = ws.buf.clone()
    d = _lib.ClapAttnDesc(qkv=ws.ptr(q_off), mask=ws.ptr(m_off), out_hi=ws.ptr(hi), out_lo=ws.ptr(lo), B=B, L=L, heads=H, C=C,
                          ld_qkv=3 * C, ldo=C)
    _lib.check(_lib.lib().aldm_clap_attention(d, _st()), "clap_attention")
    torch.cuda.synchronize()
    _assert_unchanged(ws.buf, before, [Win(hi, B * L, C, C, 2), Win(lo, B * L, C, C, 2)])
    got = ws.f16(hi, B * L * C).float() + ws.f16(lo, B * L * C).float()
    x = qkv.double().reshape(B, L, 3, H, 64)
    q, k, v = (x[:, :, j].transpose(1, 2) for j in range(3))
    s = (q @ k.transpose(-1, -2)) / 8
    s = s.masked_fill(mask[:, None, None, :] != 1, float("-inf"))
    ref = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B * L, C)
    _check(f"clap_attention B={B} L={L}", got, ref, planes=2)


@pytest.mark.gpu
def test_clap_attention_rejects_bad_shapes():
    d = _lib.ClapAttnDesc(qkv=16, mask=16, out_hi=16, B=1, L=513, heads=12, C=768, ld_qkv=2304, ldo=768)
    assert _lib.lib().aldm_clap_attention(d, None) == -2           # ALDM_E_SHAPE: more than 512 tokens
    d.L, d.heads = 512, 16
    assert _lib.lib().aldm_clap_attention(d, None) == -2           # heads x 64 != C


@pytest.mark.gpu
@pytest.mark.parametrize("rows,F", [(1, 64), (77, 3072), (4096, 3072)])
def test_clap_gelu(rows, F):
    g = torch.Generator().manual_seed(rows + F)
    ld_x, ldo = F + 4, F + 8
    x = 3.0 * torch.randn(rows, ld_x, generator=g)
    ws = Ws(4 * rows * ld_x + 4 * rows * ldo + 64 * GUARD)
    x_off = ws.put(x)
    hi, lo = ws.alloc(2 * rows * ldo), ws.alloc(2 * rows * ldo)
    before = ws.buf.clone()
    d = _lib.ClapGeluDesc(x=ws.ptr(x_off), out_hi=ws.ptr(hi), out_lo=ws.ptr(lo), rows=rows, F=F, ld_x=ld_x, ldo=ldo)
    _lib.check(_lib.lib().aldm_clap_gelu(d, _st()), "clap_gelu")
    torch.cuda.synchronize()
    _assert_unchanged(ws.buf, before, [Win(hi, rows, ldo, F, 2), Win(lo, rows, ldo, F, 2)])
    got = (ws.f16(hi, rows * ldo).float() + ws.f16(lo, rows * ldo).float()).reshape(rows, ldo)[:, :F]
    _check(f"clap_gelu rows={rows} F={F}", got, OC.gelu(x.double()[:, :F]), planes=2)


@pytest.mark.gpu
@pytest.mark.parametrize("B,L", [(1, 1), (8, 77)])
def test_clap_head(B, L):
    g = torch.Generator().manual_seed(B + L)
    C, Pj = 768, 512
    x = torch.randn(B * L, C, generator=g)
    wp, w1, w2 = (torch.randn(n, k, generator=g) / k ** 0.5 for n, k in ((C, C), (Pj, C), (Pj, Pj)))
    bp, b1, b2 = 0.1 * torch.randn(C, generator=g), 0.1 * torch.randn(Pj, generator=g), 0.1 * torch.randn(Pj, generator=g)
    ts = [x, wp.t().contiguous(), bp, w1.t().contiguous(), b1, w2.t().contiguous(), b2]
    ws = Ws(sum(4 * t.numel() for t in ts) + 4 * B * Pj + 64 * GUARD)
    offs = [ws.put(t) for t in ts]
    o_off = ws.alloc(4 * B * Pj)
    before = ws.buf.clone()
    d = _lib.ClapHeadDesc(*[ws.ptr(o) for o in offs], out=ws.ptr(o_off), B=B, L=L, C=C, P=Pj)
    _lib.check(_lib.lib().aldm_clap_head(d, _st()), "clap_head")
    torch.cuda.synchronize()
    _assert_unchanged(ws.buf, before, [Win(o_off, B, Pj, Pj, 4)])
    xd = x.double().reshape(B, L, C)[:, 0]
    p = torch.tanh(xd @ wp.double().t() + bp.double())
    y = torch.relu(p @ w1.double().t() + b1.double()) @ w2.double().t() + b2.double()
    ref = torch.nn.functional.normalize(y, dim=-1)
    got = ws.f32(o_off, B * Pj).reshape(B, Pj).double().cpu()
    assert max(rel_l2(got[b], ref[b]) for b in range(B)) < 1e-5


# ----------------------------------------------------------------------------------------------
# the stage
# ----------------------------------------------------------------------------------------------
_ENCS = {}


def _enc(n_layer, use_graph=True):
    from audioldm2_b200.clap import NativeCLAPTextEncoder
    key = (n_layer, use_graph)
    if key not in _ENCS:
        _ENCS[key] = NativeCLAPTextEncoder(CC.weights(n_layer), DEV, use_graph=use_graph)
    return _ENCS[key]


def _per_row(got, ref):
    return max(rel_l2(got[b], ref[b]) for b in range(ref.shape[0]))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CC.CASES))
def test_stage_matches_reference(name):
    golden = CC.load()
    ids, mask = (t.to(DEV) for t in CC.inputs(name))
    got = _enc(CC.CASES[name][0]).embed(ids, mask).cpu()
    assert torch.isfinite(got).all()
    assert _per_row(got, golden[name]) < TOL


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CC.UNCOND))
def test_unconditional_matches_reference(name):
    enc = _enc(CC.UNCOND[name])
    u = enc.unconditional().cpu()
    assert u.shape == (1, 512) and enc.unconditional() is enc._uncond
    assert rel_l2(u, CC.load()[name]) < TOL


@pytest.mark.gpu
def test_stage_matches_float64_oracle_b8():
    ids, mask = synth.clap_token_ids(CC.RAGGED8, seed=99)
    got = _enc(12).embed(ids.to(DEV), mask.to(DEV)).cpu()
    ref = OC.clap_text_embed(CC.weights(12), ids, mask, 12)
    assert _per_row(got, ref) < TOL


@pytest.mark.gpu
def test_stage_validates_tokens():
    enc = _enc(2)
    ids, mask = (t.to(DEV) for t in CC.inputs("tiny_b3"))
    for bad in ((ids.float(), mask), (ids + arch.CLAP_TEXT["vocab"], mask), (ids, mask * 2), (ids, mask * 0)):
        with pytest.raises(ValueError):
            enc.embed(*bad)


@pytest.mark.gpu
def test_stage_bit_exact_properties():
    """512-padded input equals the same ids cut at L_eff bit for bit (the host plans on L_eff either way); graph replay
    equals the eager run; a row permutation permutes the result exactly."""
    ids, mask = (t.to(DEV) for t in synth.clap_token_ids([32, 9, 20], seed=5))
    enc = _enc(12)
    base = enc.embed(ids, mask)
    assert torch.equal(enc.embed(ids[:, :32], mask[:, :32]), base), "padded and trimmed input differ"
    assert torch.equal(enc.embed(ids[:, :100], mask[:, :100]), base)
    assert list(enc._progs)[-1] == (3, 32)
    assert torch.equal(_enc(12, use_graph=False).embed(ids, mask), base), "graph replay differs from the eager run"
    perm = torch.tensor([2, 0, 1], device=DEV)
    assert torch.equal(enc.embed(ids[perm], mask[perm]), base[perm]), "row permutation"


def _pdl_embeds():
    ids, mask = (t.to(DEV) for t in synth.clap_token_ids([40, 13], seed=6))
    return _enc(12, use_graph=False).embed(ids, mask).cpu()


@pytest.mark.gpu
def test_stage_pdl_matches_serialized_run(tmp_path):
    got = _pdl_embeds()
    path = str(tmp_path / "serial.pt")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), path]
    r = subprocess.run(cmd, env=dict(os.environ, ALDM_PDL="0"), cwd=ROOT, timeout=900, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT)
    assert r.returncode == 0, r.stdout.decode(errors="replace")[-4000:]
    assert torch.equal(got, torch.load(path))


# ----------------------------------------------------------------------------------------------
# end to end
# ----------------------------------------------------------------------------------------------
class _Embeddings:
    """Embedding-level provider: given CLAP embeddings of a token provider's prompts and CLAP(""), it makes the
    reference's replacement draws itself (as the token path does, at the same point of the call) and returns
    ``film_clap_cond1`` [B, 1, 512]; ``extra`` holds states for the other entries of the conditional / unconditional
    dicts."""

    def __init__(self, emb, uemb, cond_extra=None, uncond_fn=None):
        self.emb, self.uemb, self.cond_extra, self.uncond_fn = emb, uemb, cond_extra or {}, uncond_fn
        self.calls = 0

    def cond(self, batch):
        e = self.emb.clone()
        for i, r in enumerate(pipeline.clap_replacement_draws(e.shape[0], self.calls > 0)):
            if r:
                e[i] = self.uemb[0]
        self.calls += 1
        return {"film_clap_cond1": e[:, None], **self.cond_extra}

    def uncond(self, n):
        if self.uncond_fn is not None:
            return self.uncond_fn(n)
        return {"film_clap_cond1": self.uemb[:, None].expand(n, 1, 512).contiguous()}


@pytest.mark.gpu
def test_48k_text_to_audio_with_token_ids():
    """audioldm_48k, B = 3, 10 DDIM steps, guidance 3.5, two calls (the second makes the extra draw): token ids (native
    CLAP, with CLAP("") in the unconditional branch) give the same waveform bits as an embedding-level provider carrying
    the native embeddings, and agree within 1e-3 relative L2 with the same calls fed the float64 oracle's embeddings."""
    cfg = arch.model_config("audioldm_48k")
    tok = pipeline.SyntheticPromptTokens(cfg, lens=(24, 11, 5), device=DEV)
    kw = dict(batchsize=3, ddim_steps=10, n_candidate_gen_per_text=1, duration=2.5)
    ld = pipeline.build_model(model_name="audioldm_48k", cond_provider=tok)
    waves = [pipeline.text_to_audio(ld, "a dog barks", seed=s, **kw) for s in (42, 43)]
    enc = ld.clap_encoder()
    ids, mask = tok.cond({"text": ["x"] * 3})["film_clap_cond1"]
    emb, uemb = enc.embed(ids, mask), enc.unconditional().clone()
    ld.cond_provider = _Embeddings(emb, uemb)
    ld.conditional_dry_run_finished = False
    for s, w in zip((42, 43), waves):
        assert (pipeline.text_to_audio(ld, "a dog barks", seed=s, **kw) == w).all(), "token ids and embeddings differ"
    sd = synth.clap_text_state_dict()
    oemb = OC.clap_text_embed(sd, ids.cpu(), mask.cpu(), 12).float().to(DEV)
    ouemb = OC.clap_text_embed(sd, *(t[:, :2].cpu() for t in tok.uncond(1)["film_clap_cond1"]), 12).float().to(DEV)
    ld.cond_provider = _Embeddings(oemb, ouemb)
    ld.conditional_dry_run_finished = False
    for s, w in zip((42, 43), waves):
        w2 = pipeline.text_to_audio(ld, "a dog barks", seed=s, **kw)
        assert rel_l2(torch.from_numpy(w), torch.from_numpy(w2)) < 1e-3


@pytest.mark.gpu
def test_full_text_to_audio_with_clap_and_t5_ids():
    """audioldm2-full, B = 2, 10 DDIM steps, guidance 3.5: CLAP + T5 token ids give the same waveform bits as the call
    given encoder outputs built from the native CLAP and T5 results (GPT-2 then runs on both alike).  The encoder-level
    provider never builds the CLAP encoder."""
    cfg = arch.model_config("audioldm2-full")
    tok = pipeline.SyntheticPromptTokens(cfg, lens=(24, 11), t5_lens=(19, 7), device=DEV)
    kw = dict(batchsize=2, ddim_steps=10, n_candidate_gen_per_text=1, duration=2.5)
    ld = pipeline.build_model(model_name="audioldm2-full", cond_provider=tok)
    wave = pipeline.text_to_audio(ld, "a dog barks", **kw)
    c = tok.cond({"text": ["x"] * 2})
    emb, uemb = ld.clap_encoder().embed(*c["film_clap_cond1"]), ld.clap_encoder().unconditional().clone()
    t5c, t5u = ld.t5_encoders()
    t5_ids, t5_mask = c["crossattn_flan_t5"]
    h = t5c.encode(t5_ids, t5_mask)
    hu = t5u.unconditional(2)
    ld.cond_provider = _Embeddings(emb, uemb, {"crossattn_flan_t5": [h, t5_mask.float()]},
                                   lambda n: {"crossattn_audiomae_generated": [torch.zeros(n, 8, 768, device=DEV),
                                                                               torch.ones(n, 8, device=DEV)],
                                              "crossattn_flan_t5": [hu[:1].expand(n, 1, 1024).contiguous(),
                                                                    torch.ones(n, 1, device=DEV)]})
    ld.conditional_dry_run_finished = False
    clap_enc, ld._clap = ld._clap, None
    w2 = pipeline.text_to_audio(ld, "a dog barks", **kw)
    assert ld._clap is None, "an embedding-level provider built the CLAP encoder"
    ld._clap = clap_enc
    assert (w2 == wave).all()


if __name__ == "__main__":          # child of test_stage_pdl_matches_serialized_run
    assert os.environ.get("ALDM_PDL") == "0"
    torch.save(_pdl_embeds(), sys.argv[1])
