"""CPU checks of the AudioMAE token generator: the float64 oracle against the reference fixtures, the planned program
(run op by op by an emulator that knows the generator's op kinds and the GELU-tanh epilogue) against them, the synthetic
checkpoint's key list, the checkpoint split and the conditioning routing of the pipeline."""
import math

import pytest
import torch

from audioldm2_b200 import _lib, arch, model, packing, pipeline, plan, synth
from audioldm2_b200.plan import Ref
from oracle import seqgen as OS
from tests.conftest import rel_l2
from tests.emulator import Emulator
from tests.golden import seqgen_cases as SC

TOL = 2e-5         # relative L2 per generated token


@pytest.fixture(scope="module")
def golden():
    return SC.load()


def _per_token(got, ref):
    return max(rel_l2(got[:, k], ref[:, k]) for k in range(ref.shape[1]))


def _case(name, full):
    return pytest.param(name, marks=pytest.mark.slow) if full else name


CASE_PARAMS = [_case(n, c[0] == 12) for n, c in SC.CASES.items()]


@pytest.mark.parametrize("name", CASE_PARAMS)
def test_oracle_matches_reference(golden, name):
    n_layer = SC.CASES[name][0]
    clap, t5, mask = SC.inputs(name)
    got = OS.audiomae_generate(SC.weights(n_layer), clap.double(), t5.double(), mask.double(), n_layer)
    assert got.dtype == torch.float64 and got.shape == golden[name].shape
    assert _per_token(got, golden[name]) < TOL


class SeqgenEmulator(Emulator):
    """tests/emulator.py plus the generator's op kinds (include/aldm_b200.h) and ALDM_ACT_GELU_TANH."""

    def op_gemm(self, o):
        if o["act"] != _lib.ACT_GELU_TANH:
            return super().op_gemm(o)
        assert o.get("res") is None and o["alpha"] == 1.0 and not o["accumulate"]
        M = o["B"] * o["OH"] * o["OW"]
        self.mem["tmp"] = torch.zeros(M * o["N"] * 4, dtype=torch.uint8)
        super().op_gemm(dict(o, act=_lib.ACT_NONE, out_mode=_lib.OUT_F32, out=Ref("tmp", 0), ldo=o["N"], out_hi=None, out_lo=None,
                             OHF=o["OH"], osy=1, ooy=0))
        v = OS.gelu_new(self.f32(Ref("tmp", 0), M * o["N"]).reshape(M, o["N"]))
        b = torch.arange(M) // (o["OH"] * o["OW"])
        orow = (b * o["OHF"] + (torch.arange(M) // o["OW"]) % o["OH"] * o["osy"] + o["ooy"]) * o["OWF"] + torch.arange(M) % o["OW"]
        nrows = o["B"] * o["OHF"] * o["OWF"]
        if o["out_mode"] == _lib.OUT_PLANES:
            self.put_planes(o["out_hi"], o.get("out_lo"), nrows, o["N"], o["ldo"], orow, v)
        else:
            assert o["out_mode"] == _lib.OUT_F32
            torch.as_strided(self.f32(o["out"], (nrows - 1) * o["ldo"] + o["N"]), (nrows, o["N"]), (o["ldo"], 1))[orow] = v

    def op_seq_assemble(self, o):
        B, L, C, lmax = o["B"], o["L"], o["C"], o["lmax"]
        P = L + 5
        x = self.f32(o["x"], B * P * C).reshape(B, P, C)
        sos, eos = self.f32(o["sos"], 2 * C).reshape(2, C), self.f32(o["eos"], 2 * C).reshape(2, C)
        proj = x.clone()
        assert torch.isfinite(proj[:, 1]).all() and torch.isfinite(proj[:, 4:4 + L]).all(), "projections not written"
        proj[:, 0], proj[:, 2], proj[:, 3], proj[:, P - 1] = sos[0], eos[0], sos[1], eos[1]
        x[:] = proj + self.f32(o["wpe"], P * C).reshape(P, C)
        m = torch.ones(B, lmax)
        m[:, 4:4 + L] = self.f32(o["t5_mask"], B * L).reshape(B, L)
        self.f32(o["mask"], B * lmax)[:] = m.reshape(-1)

    def op_kv_attn(self, o):
        B, H, lmax, ld, p0, nq = o["B"], o["heads"], o["lmax"], o["ld_seq"], o["p0"], o["nq"]
        C = H * 64
        seq = self.f32(o["seq"], B * lmax * ld).reshape(B, lmax, ld)
        nk = p0 + nq
        q = seq[:, p0:nk, :C].reshape(B, nq, H, 64).transpose(1, 2)
        k = seq[:, :nk, C:2 * C].reshape(B, nk, H, 64).transpose(1, 2)
        v = seq[:, :nk, 2 * C:3 * C].reshape(B, nk, H, 64).transpose(1, 2)
        assert torch.isfinite(q).all() and torch.isfinite(k).all() and torch.isfinite(v).all(), "KV cache reads garbage"
        s = (q @ k.transpose(-1, -2)) * o["scale"]
        keep = (torch.arange(nk)[None, :] <= (p0 + torch.arange(nq))[:, None])[None, None]
        keep = keep & (self.f32(o["mask"], B * lmax).reshape(B, lmax)[:, None, None, :nk] == 1)
        s = s.masked_fill(~keep, float("-inf"))
        out = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B * nq, C)
        self.write_planes(o["out_hi"], o.get("out_lo"), out, o["ldo"], B * nq)

    def op_seq_feedback(self, o):
        B, nq, C = o["B"], o["nq"], o["C"]
        x = self.f32(o["x"], B * nq * C).reshape(B, nq, C)[:, -1]
        y = torch.nn.functional.layer_norm(x, (C,), self.f32(o["gamma"], C), self.f32(o["beta"], C), o["eps"])
        self.f32(o["out"], B * o["gen_len"] * C).reshape(B, o["gen_len"], C)[:, o["k"]] = y
        if o.get("next") is not None:
            self.f32(o["next"], B * C)[:] = (y + self.f32(o["wpe"], (o["pos"] + 2) * C).reshape(-1, C)[o["pos"] + 1]).reshape(-1)


def _emulate(name):
    n_layer, lens, _ = SC.CASES[name]
    clap, t5, mask = SC.inputs(name)
    pl = plan.build_seqgen(SC.weights(n_layer), len(lens), max(lens))
    em = SeqgenEmulator(pl)
    em.write_io("clap", clap); em.write_io("t5", t5); em.write_io("t5_mask", mask)
    em.run()
    return em.read_io("tokens"), pl


@pytest.mark.parametrize("name", [_case(n, c[0] == 12) for n, c in SC.CASES.items() if n.endswith(("l32", "l128")) or c[0] == 2])
def test_planned_program_matches_reference(golden, name):
    got, pl = _emulate(name)
    assert _per_token(got, golden[name]) < TOL


def test_plan_structure():
    pl = plan.build_seqgen(SC.weights(2), 3, 32)
    kinds = [o["kind"] for o in pl.ops]
    per_pass = 2 * (7 + 0) + 1            # per layer: LN, c_attn, kv_attn, c_proj, LN, c_fc, c_proj; then the feedback
    assert kinds[:5] == ["prep", "gemm", "prep", "gemm", "seq_assemble"]
    assert len(kinds) == 5 + 8 * (2 * 7 + 1) and per_pass == 15
    assert [pl.marks[f"decode{k}_end"] - pl.marks[f"decode{k - 1}_end" if k > 1 else "prefill_end"] for k in range(1, 8)] == [15] * 7
    fc = [o for o in pl.ops if o["kind"] == "gemm" and o["act"] == _lib.ACT_GELU_TANH]
    assert len(fc) == 16 and all(o["a_lo"] is not None for o in pl.ops if o["kind"] == "gemm")     # two planes everywhere
    attn = [o for o in pl.ops if o["kind"] == "kv_attn"]
    assert [(o["p0"], o["nq"]) for o in attn[::2]] == [(0, 37)] + [(36 + k, 1) for k in range(1, 8)]
    # the c_attn GEMMs write their rows in place in the sequence buffer: positions [p0, p0 + nq) of each batch row
    ca = [o for o in pl.ops if o["kind"] == "gemm" and o["N"] == 2304]
    assert all(o["OHF"] == 45 and o["ooy"] == a["p0"] and o["H"] == a["nq"] for o, a in zip(ca, attn))
    with pytest.raises(ValueError):
        plan.build_seqgen(SC.weights(2), 1, 1012)


def test_shared_weight_arena():
    w = plan.pack_seqgen_weights(SC.weights(2))
    a, b = plan.build_seqgen(None, 1, 5, weights=w), plan.build_seqgen(None, 8, 128, weights=w)
    assert a.arena is w.arena and b.arena is w.arena
    full = arch.seqgen_param_shapes(12, with_wte=False)
    n = sum(math.prod(s) for k, s in full.items() if ".h." in k and k.endswith("weight") and len(s) == 2)
    assert 330e6 < 4 * n < 350e6           # two fp16 planes of the 48 GPT-2 matrices: about 340 MB


def test_state_dict_matches_reference_keys(golden):
    sd = synth.seqgen_state_dict(n_layer=12)
    assert {k: list(v.shape) for k, v in sd.items()} == golden["param_shapes"]
    assert abs(float(sd["model.wpe.weight"].std()) - 0.02) < 1e-3
    assert abs(float(sd["start_of_sequence_tokens.weight"].std()) - 1.0) < 0.02
    w = sd["model.h.0.mlp.c_proj.weight"]                  # Conv1D [3072, 768]: fan-in 3072
    assert abs(float(w.std()) * math.sqrt(3072) - 1.0) < 0.02


def test_conv1d_packing_transposes():
    w = torch.randn(24, 40)                                 # Conv1D [in=24, out=40]
    wm, taps, cp = packing.conv1d_weight_matrix(w)
    assert (taps, cp) == (1, 24) and torch.equal(wm, w.t())


def test_split_seqgen_state_dict():
    sd = SC.weights(2)
    ck = {"model.diffusion_model.out.2.bias": torch.zeros(8), "cond_stage_models.1.model.wpe.weight": torch.zeros(1)}
    ck.update({f"cond_stage_models.0.{k}": v for k, v in sd.items()})
    ck["cond_stage_models.0.model.h.0.attn.bias"] = torch.ones(1, 1, 1024, 1024, dtype=torch.bool)
    ck["cond_stage_models.0.model.h.0.attn.masked_bias"] = torch.tensor(-1e4)
    ck["cond_stage_models.0.cond_stage_models.0.model.text_branch.x"] = torch.zeros(3)
    got = model.split_seqgen_state_dict(ck)
    assert set(got) == set(sd) - {"model.wte.weight"}
    assert all(got[k] is ck["cond_stage_models.0." + k] for k in got)
    un, vae, voc, sf = model.split_state_dict(ck)            # unchanged: the generator's keys are not part of it
    assert set(un) == {"out.2.bias"} and not vae and not voc
    del ck["cond_stage_models.0.model.ln_f.bias"]
    with pytest.raises(KeyError):
        model.split_seqgen_state_dict(ck)


class _FakeGen:
    def __init__(self):
        self.calls = []

    def generate(self, clap, t5, mask):
        self.calls.append((clap.shape[0], t5.shape[1]))
        return torch.full((clap.shape[0], 8, 768), 0.5)


def test_routing_encoder_outputs_generate_tokens():
    cfg = arch.model_config("audioldm2-full")
    prov = pipeline.SyntheticEncoderOutputs(cfg, t5_lens=(12, 5))
    cond = prov.cond({"text": ["a", "b", "c"]})
    assert cond["film_clap_cond1"].shape == (3, 1, 512) and cond["crossattn_flan_t5"][0].shape == (3, 12, 1024)
    assert cond["crossattn_flan_t5"][1].sum(1).tolist() == [12, 5, 12]
    assert torch.allclose(cond["film_clap_cond1"].norm(dim=-1), torch.ones(3, 1))
    g = _FakeGen()
    out = pipeline.route_conditioning(cfg, cond, lambda: g)
    assert list(out) == ["crossattn_audiomae_generated", "crossattn_flan_t5"] and g.calls == [(3, 12)]
    tok, ones = out["crossattn_audiomae_generated"]
    assert tok.shape == (3, 8, 768) and torch.equal(ones, torch.ones(3, 8))
    assert out["crossattn_flan_t5"][0] is cond["crossattn_flan_t5"][0]
    u = model.unpack_cond_dict(out)
    assert [c.shape[-1] for c in u["context_list"]] == [768, 1024]
    # tiling by n_gen happens after generation: B rows are generated, B * n_gen rows reach the UNet
    assert pipeline._tile(out, 3)["crossattn_audiomae_generated"][0].shape[0] == 9
    # the unconditional branch: SyntheticConditioning's one-prompt rows on every row, whatever the row count
    u1, u3 = prov.uncond(1), prov.uncond(3)
    ref = pipeline.SyntheticConditioning(cfg).uncond(1)
    for s_ in range(2):
        assert torch.equal(u1["context_list"][s_], ref["context_list"][s_])
        assert torch.equal(u3["context_list"][s_], ref["context_list"][s_].expand(3, -1, -1))
        assert torch.equal(u3["mask_list"][s_], torch.ones(3, ref["mask_list"][s_].shape[1]))
    assert not u3["context_list"][0].any() and u3["y"] is None


def test_routing_unet_boundary_never_builds_generator():
    cfg = arch.model_config("audioldm2-full")
    def boom():
        raise AssertionError("generator built for UNet-boundary conditioning")
    for cond in (pipeline.SyntheticConditioning(cfg).cond({"text": ["a"]}),
                 {"crossattn_audiomae_generated": [torch.zeros(1, 8, 768), torch.ones(1, 8)],
                  "crossattn_flan_t5": [torch.zeros(1, 4, 1024), torch.ones(1, 4)], "film_clap_cond1": torch.zeros(1, 1, 512)}):
        assert pipeline.route_conditioning(cfg, cond, boom) is cond


@pytest.mark.parametrize("name", ["audioldm_48k", "audioldm2-full-t5", "audioldm2-speech-gigaspeech"])
def test_routing_rejects_models_without_the_stage(name):
    cfg = arch.model_config(name)
    assert not arch.has_seqgen(cfg)
    cond = {"film_clap_cond1": torch.zeros(1, 1, 512), "crossattn_flan_t5": [torch.zeros(1, 4, 1024), torch.ones(1, 4)]}
    with pytest.raises(ValueError, match="no AudioMAE token generator"):
        pipeline.route_conditioning(cfg, cond, lambda: _FakeGen())
    with pytest.raises(ValueError):
        pipeline.SyntheticEncoderOutputs(cfg)
    assert arch.has_seqgen(arch.model_config("audioldm2-full-large-1150k"))
