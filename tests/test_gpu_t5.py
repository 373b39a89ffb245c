"""The Flan-T5 encoder on the GPU: its kernels (csrc/text/*.cu) against float64 inside 4 KB guard bands, the saturation
counter, the whole stage against the reference fixtures and the float64 oracle, bit-exact properties and the pipeline
end to end.

Bounds (relative L2 AND per element, as tests/test_gpu_kernel_matrix.py):
  * t5_embed_kernel: a gather, compared bit for bit.
  * t5_rmsnorm_kernel: one fp32 sum of C = 1024 squares (32 sequential terms per lane, then a 5-level tree): relative
    error <= ~37 x 2^-24 ~ 2.2e-6 of the sum, half of that in 1/sqrt, plus two roundings in gamma * (x * r): at most
    ~2e-6 |ref|.  fp32 output: |err| <= 2^-18 |ref| per element (3.8e-6, a 2x margin) and relative L2 < 2e-6.  Plane
    output: the two-plane split adds 2^-22, so the matrix's two-plane budget (2e-5 / 1e-4 rms) holds with a wide margin.
  * t5_attention_kernel: q, k, v are fp32 (the QKV GEMM's fp32 output), the reference uses the same values in float64.
    The logits are unscaled, so the scores carry the fp32 error of a 64-term dot product, <= 64 x 2^-24 sum |q_i k_i|
    (~2e-5 absolute for the inputs here, whose logits reach |s| ~ 10), which moves each probability by the same
    relative amount; expf adds 2 ulp, the P V sum over <= 128 keys ~ 128 x 2^-24 sum p |v|, the split 2^-22.  Two-plane
    budget: relative L2 < 2e-5 and |err| <= 1e-4 rms(ref).
  * t5_gate_kernel: gelu_new with the accurate tanhf (2 ulp; slope <= 1.13) times one fp32 product, then the two-plane
    split: the two-plane budget.  The counter is exact: it counts |y| > 65504.
The stage: relative L2 per batch row below 3e-5 against the reference fixtures (fp32 torch on the CPU) and against the
float64 oracle at B = 8, L = 128, 24 blocks.  CPU emulation of the planned program (fp16 two-plane operands, fp32
arithmetic, tests/test_t5_cpu.py's emulator) measures the cost of the two-plane GEMM operands on that case at 3.1e-6
to 3.7e-6 per row against float64; fp32 torch itself is at 4.3e-7; the tensor cores' truncating accumulation
(tests/test_gpu_kernel_matrix.py) adds at most ~1e-6 per GEMM, so 3e-5 leaves a margin of about 5x.
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

from audioldm2_b200 import _lib, arch, pipeline, synth
from oracle import t5 as OT
from tests.conftest import rel_l2
from tests.golden import t5_cases as TC
from tests.test_gpu_kernel_matrix import GUARD, Win, _assert_unchanged, _check
from tests.test_gpu_seqgen import Ws

DEV = "cuda:0"
TOL = 3e-5          # relative L2 per batch row (docstring)

# kernel -> the test of this file that runs it against a float64 reference
KERNEL_TESTS = {
    "t5_embed_kernel": "test_t5_embed",
    "t5_rmsnorm_kernel": "test_t5_rmsnorm",
    "t5_attention_kernel": "test_t5_attention",
    "t5_gate_kernel": "test_t5_gate",
}


def test_every_text_kernel_has_a_test():
    """Inventory of csrc/text/*.cu: every __global__ kernel is mapped to a test of this file, and no entry is stale."""
    found = set()
    for path in glob.glob(os.path.join(ROOT, "audioldm2_b200", "csrc", "text", "*.cu")):
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
@pytest.mark.parametrize("rows", [1, 37, 1024])
def test_t5_embed(rows):
    g = torch.Generator().manual_seed(rows)
    V, C = 1000, 1024
    table = torch.randn(V, C, generator=g)
    ids = torch.randint(0, V, (rows,), generator=g)
    ids[0], ids[-1] = 0, V - 1
    ws = Ws(4 * (V * C + 2 * rows * C) + 8 * rows + 64 * GUARD)
    t_off, i_off = ws.put(table), ws.put(ids)
    o_off = ws.alloc(4 * rows * C)
    before = ws.buf.clone()
    d = _lib.T5EmbedDesc(ids=ws.ptr(i_off), table=ws.ptr(t_off), out=ws.ptr(o_off), rows=rows, vocab=V, C=C)
    _lib.check(_lib.lib().aldm_t5_embed(d, _st()), "t5_embed")
    torch.cuda.synchronize()
    _assert_unchanged(ws.buf, before, [Win(o_off, rows, C, C, 4)])
    assert torch.equal(ws.f32(o_off, rows * C).cpu().reshape(rows, C), table[ids])
    # an id the host failed to reject gives a NaN row, never a read outside the table
    ws.buf[i_off:i_off + 8].copy_(torch.tensor([V], dtype=torch.int64).view(torch.uint8).to(DEV))
    _lib.check(_lib.lib().aldm_t5_embed(d, _st()), "t5_embed")
    torch.cuda.synchronize()
    assert torch.isnan(ws.f32(o_off, C)).all()


@pytest.mark.gpu
@pytest.mark.parametrize("rows,mode", [(1, "planes"), (333, "planes"), (1024, "planes"), (5, "f32"), (1024, "f32")])
def test_t5_rmsnorm(rows, mode):
    g = torch.Generator().manual_seed(rows * 3 + len(mode))
    C, eps = 1024, 1e-6
    x = torch.randn(rows, C, generator=g) * (1 + 10 * torch.rand(rows, 1, generator=g)) + 0.5
    gamma = 1 + 0.1 * torch.randn(C, generator=g)
    ldo = C + 8 if mode == "planes" else C
    ws = Ws(4 * (rows * C + C) + 4 * rows * ldo + 64 * GUARD)
    x_off, g_off = ws.put(x), ws.put(gamma)
    if mode == "planes":
        hi, lo = ws.alloc(2 * rows * ldo), ws.alloc(2 * rows * ldo)
        d = _lib.T5RmsnormDesc(x=ws.ptr(x_off), gamma=ws.ptr(g_off), out_hi=ws.ptr(hi), out_lo=ws.ptr(lo), rows=rows, C=C,
                               ldo=ldo, eps=eps)
        wins = [Win(hi, rows, ldo, C, 2), Win(lo, rows, ldo, C, 2)]
    else:
        of = ws.alloc(4 * rows * C)
        d = _lib.T5RmsnormDesc(x=ws.ptr(x_off), gamma=ws.ptr(g_off), out_f32=ws.ptr(of), rows=rows, C=C, ldo=C, eps=eps)
        wins = [Win(of, rows, C, C, 4)]
    before = ws.buf.clone()
    _lib.check(_lib.lib().aldm_t5_rmsnorm(d, _st()), "t5_rmsnorm")
    torch.cuda.synchronize()
    _assert_unchanged(ws.buf, before, wins)
    ref = OT.rms_norm(x.double(), gamma.double(), eps)
    if mode == "planes":
        got = (ws.f16(hi, rows * ldo).float() + ws.f16(lo, rows * ldo).float()).reshape(rows, ldo)[:, :C]
        _check(f"t5_rmsnorm rows={rows}", got, ref, planes=2)
    else:
        got = ws.f32(of, rows * C).reshape(rows, C).double().cpu()
        assert rel_l2(got, ref) < 2e-6
        assert ((got - ref).abs() <= 2.0 ** -18 * ref.abs()).all()


ATT_CASES = [(1, 1), (3, 37), (2, 64), (8, 128)]


@pytest.mark.gpu
@pytest.mark.parametrize("B,L", ATT_CASES)
def test_t5_attention(B, L):
    g = torch.Generator().manual_seed(B * 131 + L)
    H, C = 16, 1024
    qkv = torch.randn(B * L, 3 * C, generator=g)
    qkv[:, :C] *= 0.35                                              # unscaled logits of a few units: a peaked softmax
    bias = torch.randn(H, 255, generator=g)
    mask = torch.ones(B, L)
    for b in range(B):                                              # ragged rows, and scattered padding
        mask[b, max(1, L - 11 * b):] = 0
    mask[:, 1:] *= (torch.rand(B, L - 1, generator=g) < 0.9).float()
    ws = Ws(4 * (B * L * 3 * C + H * 255 + B * L) + 4 * B * L * C + 64 * GUARD)
    q_off, b_off, m_off = ws.put(qkv), ws.put(bias), ws.put(mask)
    hi, lo = ws.alloc(2 * B * L * C), ws.alloc(2 * B * L * C)
    before = ws.buf.clone()
    d = _lib.T5AttnDesc(qkv=ws.ptr(q_off), bias=ws.ptr(b_off), mask=ws.ptr(m_off), out_hi=ws.ptr(hi), out_lo=ws.ptr(lo), B=B, L=L,
                        heads=H, d_kv=64, C=C, ld_qkv=3 * C, ldo=C)
    _lib.check(_lib.lib().aldm_t5_attention(d, _st()), "t5_attention")
    torch.cuda.synchronize()
    _assert_unchanged(ws.buf, before, [Win(hi, B * L, C, C, 2), Win(lo, B * L, C, C, 2)])
    got = ws.f16(hi, B * L * C).float() + ws.f16(lo, B * L * C).float()
    x = qkv.double().reshape(B, L, 3, H, 64)
    q, k, v = (x[:, :, j].transpose(1, 2) for j in range(3))
    pos = torch.arange(L)
    s = q @ k.transpose(-1, -2) + bias.double()[:, pos[None, :] - pos[:, None] + 127][None]
    s = s.masked_fill(mask[:, None, None, :] != 1, float("-inf"))
    ref = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B * L, C)
    _check(f"t5_attention B={B} L={L}", got, ref, planes=2)


@pytest.mark.gpu
def test_t5_attention_rejects_bad_shapes():
    d = _lib.T5AttnDesc(qkv=16, bias=16, mask=16, out_hi=16, B=1, L=129, heads=16, d_kv=64, C=1024, ld_qkv=3072, ldo=1024)
    assert _lib.lib().aldm_t5_attention(d, None) == -2             # ALDM_E_SHAPE: more than 128 tokens
    d.L, d.d_kv = 128, 32
    assert _lib.lib().aldm_t5_attention(d, None) == -6             # ALDM_E_UNSUPPORTED: d_kv != 64
    d.d_kv, d.heads = 64, 12
    assert _lib.lib().aldm_t5_attention(d, None) == -2             # heads x 64 != C


@pytest.mark.gpu
@pytest.mark.parametrize("rows,F", [(1, 64), (77, 2816), (1024, 2816)])
def test_t5_gate(rows, F):
    g = torch.Generator().manual_seed(rows + F)
    ld_x, ldo = 2 * F + 4, F + 8
    x = 2.0 * torch.randn(rows, ld_x, generator=g)
    ws = Ws(4 * rows * ld_x + 4 * rows * ldo + 4 + 64 * GUARD)
    x_off = ws.put(x)
    hi, lo = ws.alloc(2 * rows * ldo), ws.alloc(2 * rows * ldo)
    s_off = ws.put(torch.zeros(1, dtype=torch.int32))
    before = ws.buf.clone()
    d = _lib.T5GateDesc(x=ws.ptr(x_off), out_hi=ws.ptr(hi), out_lo=ws.ptr(lo), sat=ws.ptr(s_off), rows=rows, F=F, ld_x=ld_x, ldo=ldo)
    _lib.check(_lib.lib().aldm_t5_gate(d, _st()), "t5_gate")
    torch.cuda.synchronize()
    _assert_unchanged(ws.buf, before, [Win(hi, rows, ldo, F, 2), Win(lo, rows, ldo, F, 2)])
    assert int(ws.buf[s_off:s_off + 4].view(torch.int32)) == 0
    got = (ws.f16(hi, rows * ldo).float() + ws.f16(lo, rows * ldo).float()).reshape(rows, ldo)[:, :F]
    xd = x.double()
    _check(f"t5_gate rows={rows} F={F}", got, OT.gelu_new(xd[:, :F]) * xd[:, F:2 * F], planes=2)


@pytest.mark.gpu
def test_t5_gate_counts_saturation():
    """gelu_new(100) = 100 exactly in fp32, so y = 100 b: b = 655.05 gives |y| > 65504 and is counted (once per element,
    in every row), b = 655.03 does not."""
    rows, F = 3, 64
    x = torch.zeros(rows, 2 * F)
    x[:, :F] = 100.0
    x[:, F:] = 1.0
    x[:, F + 5] = 655.03
    ws = Ws(4 * rows * 2 * F + 4 * rows * F + 4 + 64 * GUARD)
    x_off = ws.put(x)
    hi, lo = ws.alloc(2 * rows * F), ws.alloc(2 * rows * F)
    s_off = ws.put(torch.zeros(1, dtype=torch.int32))
    d = _lib.T5GateDesc(x=ws.ptr(x_off), out_hi=ws.ptr(hi), out_lo=ws.ptr(lo), sat=ws.ptr(s_off), rows=rows, F=F, ld_x=2 * F, ldo=F)
    _lib.check(_lib.lib().aldm_t5_gate(d, _st()), "t5_gate")
    torch.cuda.synchronize()
    assert int(ws.buf[s_off:s_off + 4].view(torch.int32)) == 0, "a value just below 65504 was counted"
    x[:, F + 9] = 655.05
    x[1, F + 20] = -700.0
    ws.buf[x_off:x_off + x.numel() * 4].copy_(x.view(torch.uint8).reshape(-1).to(DEV))
    _lib.check(_lib.lib().aldm_t5_gate(d, _st()), "t5_gate")
    torch.cuda.synchronize()
    assert int(ws.buf[s_off:s_off + 4].view(torch.int32)) == rows + 1


# ----------------------------------------------------------------------------------------------
# the stage
# ----------------------------------------------------------------------------------------------
_ENCS = {}


def _enc(n_layer, use_graph=True):
    from audioldm2_b200.t5 import NativeFlanT5Encoder
    key = (n_layer, use_graph)
    if key not in _ENCS:
        _ENCS[key] = NativeFlanT5Encoder(TC.weights(n_layer), DEV, use_graph=use_graph)
    return _ENCS[key]


def _per_row(got, ref):
    return max(rel_l2(got[b], ref[b]) for b in range(ref.shape[0]))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(TC.CASES))
def test_stage_matches_reference(name):
    golden = TC.load()
    ids, mask = (t.to(DEV) for t in TC.inputs(name))
    got = _enc(TC.CASES[name][0]).encode(ids, mask).cpu()
    assert torch.isfinite(got).all()
    assert _per_row(got, golden[name]) < TOL


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(TC.UNCOND))
def test_unconditional_matches_reference(name):
    enc = _enc(TC.UNCOND[name])
    u = enc.unconditional(3).cpu()
    assert u.shape == (3, 1, 1024) and torch.equal(u[0], u[2])
    assert rel_l2(u[:1], TC.load()[name]) < TOL
    assert enc.unconditional(5).data_ptr() != enc._uncond.data_ptr() and enc._uncond.shape == (1, 1, 1024)


@pytest.mark.gpu
def test_stage_matches_float64_oracle_b8_l128():
    lens = [128, 100, 77, 64, 31, 12, 5, 1]
    ids, mask = synth.token_ids(lens, seed=99)
    got = _enc(24).encode(ids.to(DEV), mask.to(DEV)).cpu()
    ref = OT.t5_encode(TC.weights(24), ids, mask, 24)
    assert _per_row(got, ref) < TOL


@pytest.mark.gpu
def test_stage_raises_on_saturation():
    """A block whose gated product leaves the fp16 range raises and names the block; the counter is cleared, so the
    next call on unsaturated weights is clean."""
    from audioldm2_b200.t5 import NativeFlanT5Encoder
    sd = dict(TC.weights(2))
    k = "encoder.block.1.layer.1.DenseReluDense.wi_1.weight"
    sd[k] = sd[k] * 1e5
    enc = NativeFlanT5Encoder(sd, DEV)
    ids, mask = (t.to(DEV) for t in TC.inputs("tiny_b3_l32"))
    with pytest.raises(RuntimeError, match=r"block\(s\) 1 \("):
        enc.encode(ids, mask)
    assert not enc.program(3, 32).view("sat").any()
    ok = _enc(2).encode(ids, mask)
    assert torch.isfinite(ok).all()


@pytest.mark.gpu
def test_stage_validates_tokens():
    enc = _enc(2)
    ids, mask = (t.to(DEV) for t in TC.inputs("tiny_b3_l32"))
    for bad in ((ids.float(), mask), (ids + arch.T5["vocab"], mask), (ids, mask * 2), (ids, mask * 0)):
        with pytest.raises(ValueError):
            enc.encode(*bad)


@pytest.mark.gpu
def test_stage_bit_exact_properties():
    ids, mask = (t.to(DEV) for t in synth.token_ids([32, 9, 20], seed=5))
    enc = _enc(24)
    base = enc.encode(ids, mask)
    assert torch.equal(_enc(24, use_graph=False).encode(ids, mask), base), "graph replay differs from the eager run"
    perm = torch.tensor([2, 0, 1], device=DEV)
    assert torch.equal(enc.encode(ids[perm], mask[perm]), base[perm]), "row permutation"


def _pdl_states():
    ids, mask = (t.to(DEV) for t in synth.token_ids([40, 13], seed=6))
    return _enc(24, use_graph=False).encode(ids, mask).cpu()


@pytest.mark.gpu
def test_stage_pdl_matches_serialized_run(tmp_path):
    got = _pdl_states()
    path = str(tmp_path / "serial.pt")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), path]
    r = subprocess.run(cmd, env=dict(os.environ, ALDM_PDL="0"), cwd=ROOT, timeout=900, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT)
    assert r.returncode == 0, r.stdout.decode(errors="replace")[-4000:]
    assert torch.equal(got, torch.load(path))


# ----------------------------------------------------------------------------------------------
# end to end
# ----------------------------------------------------------------------------------------------
class _OracleStates:
    """Encoder-level provider holding the float64 oracle's T5 states of a token provider's ids (and its CLAP vector);
    the unconditional branch holds the oracle's T5("")."""

    def __init__(self, tok, n):
        self.tok = tok
        c = tok.cond({"text": ["x"] * n})
        ids, mask = c["crossattn_flan_t5"]
        sd = synth.t5_state_dict()
        self.h = OT.t5_encode(sd, ids.cpu(), mask.cpu(), 24).float().to(DEV)
        self.mask, self.clap = mask.to(DEV), c["film_clap_cond1"].to(DEV)
        self.u = OT.t5_encode(sd, torch.tensor([[1]]), torch.ones(1, 1), 24).float().to(DEV)

    def cond(self, batch):
        return {"film_clap_cond1": self.clap, "crossattn_flan_t5": [self.h, self.mask]}

    def uncond(self, n):
        return {"crossattn_audiomae_generated": [torch.zeros(n, 8, 768, device=DEV), torch.ones(n, 8, device=DEV)],
                "crossattn_flan_t5": [self.u.expand(n, 1, 1024).contiguous(), torch.ones(n, 1, device=DEV)]}


@pytest.mark.gpu
def test_text_to_audio_with_token_ids():
    """audioldm2-full, B = 2, 10 DDIM steps, 3 candidates per prompt, guidance 3.5: token ids (native T5, then GPT-2, then
    the UNet, with T5("") in the unconditional branch) against the same call with an encoder-level provider fed the
    float64 oracle's T5 states for the same ids: the waveforms agree within 1e-3 relative L2.  A provider at the
    encoder level never builds the T5 encoder."""
    cfg = arch.model_config("audioldm2-full")
    tok = pipeline.SyntheticTokenIds(cfg, lens=(32, 19), device=DEV)
    kw = dict(batchsize=2, ddim_steps=10, n_candidate_gen_per_text=3, duration=2.5)
    ld = pipeline.build_model(model_name="audioldm2-full", cond_provider=tok)
    with pytest.warns(UserWarning):
        wave = pipeline.text_to_audio(ld, "a dog barks", **kw)
    assert ld._t5 is not None and ld._t5[0] is ld._t5[1], "one encoder for equal cond / uncond weights"
    del ld
    torch.cuda.empty_cache()
    ld2 = pipeline.build_model(model_name="audioldm2-full", cond_provider=_OracleStates(tok, 2))
    with pytest.warns(UserWarning):
        w2 = pipeline.text_to_audio(ld2, "a dog barks", **kw)
    assert ld2._t5 is None, "an encoder-level provider built the T5 encoder"
    assert rel_l2(torch.from_numpy(wave), torch.from_numpy(w2)) < 1e-3


@pytest.mark.gpu
def test_rank_shards_with_token_ids():
    """A sharded call (one rank per prompt; no process group) encodes the token ids of the whole call on every rank -- the
    same (B, L) plan and bits as one process -- and keeps its rows.  Its waveform equals the single-process call's rows
    within the sharding test's 1e-3."""
    from audioldm2_b200.utils import seed_everything
    cfg = arch.model_config("audioldm2-full")
    tok = pipeline.SyntheticTokenIds(cfg, lens=(32, 11), device=DEV)
    ld = pipeline.build_model(model_name="audioldm2-full", cond_provider=tok)
    ld.latent_t_size = 64
    batch = pipeline.make_batch_for_text_to_audio(["a", "b"], batchsize=2)
    enc = ld.t5_encoders()[0]
    seen = []
    orig = enc.encode

    def recording(ids, mask):
        out = orig(ids, mask)
        seen.append((tuple(ids.shape), out.clone()))
        return out

    enc.encode = recording
    seed_everything(42)
    full = ld._generate_local(batch, 5, 1.0, 1, 3.5, None, None, None, None)
    for r in range(2):
        seed_everything(42)
        part = ld._generate_sharded((r, 2, r, r + 1), batch, 5, 1.0, 1, 3.5, None, None, None)
        assert part.shape == (1,) + full.shape[1:]
        assert rel_l2(torch.from_numpy(part), torch.from_numpy(full[r:r + 1])) < 1e-3, r
    uncond = [sh for sh, _ in seen if sh == (1, 1)]
    seen = [(sh, t) for sh, t in seen if sh != (1, 1)]
    assert uncond == [(1, 1)], "T5(\"\") is encoded once and cached"
    assert [sh for sh, _ in seen] == [(2, 32)] * 3, "a rank encoded its own rows only"
    assert all(torch.equal(t, seen[0][1]) for _, t in seen), "the ranks' states differ from the single-process states"


if __name__ == "__main__":          # child of test_stage_pdl_matches_serialized_run
    assert os.environ.get("ALDM_PDL") == "0"
    torch.save(_pdl_states(), sys.argv[1])
