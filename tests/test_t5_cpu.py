"""CPU checks of the Flan-T5 encoder: the float64 oracle against the reference fixtures, the planned program (run op by op
by an emulator that knows the encoder's op kinds) against them, the product path's bucket restatement against
transformers, the op-table structure, the checkpoint split, token validation and the conditioning routing."""
import math

import pytest
import torch

from audioldm2_b200 import _lib, arch, model, pipeline, plan, synth
from audioldm2_b200.t5 import check_tokens
from oracle import t5 as OT
from tests.conftest import rel_l2
from tests.emulator import Emulator
from tests.golden import t5_cases as TC

TOL = 2e-5          # relative L2 per batch row


@pytest.fixture(scope="module")
def golden():
    return TC.load()


def per_row(got, ref):
    return max(rel_l2(got[b], ref[b]) for b in range(ref.shape[0]))


def _case(name):
    return pytest.param(name, marks=pytest.mark.slow) if TC.CASES[name][0] == 24 else name


@pytest.mark.parametrize("name", [_case(n) for n in TC.CASES])
def test_oracle_matches_reference(golden, name):
    n_layer = TC.CASES[name][0]
    ids, mask = TC.inputs(name)
    got = OT.t5_encode(TC.weights(n_layer), ids, mask, n_layer)
    assert got.dtype == torch.float64 and got.shape == golden[name].shape
    assert per_row(got, golden[name]) < TOL


@pytest.mark.parametrize("name", ["tiny_uncond", pytest.param("full_uncond", marks=pytest.mark.slow)])
def test_oracle_matches_reference_uncond(golden, name):
    n_layer = TC.UNCOND[name]
    got = OT.t5_encode(TC.weights(n_layer), torch.tensor([[1]]), torch.ones(1, 1), n_layer)
    assert rel_l2(got, golden[name]) < TOL


def test_state_dict_matches_reference_keys(golden):
    sd = synth.t5_state_dict(n_layer=24)
    assert {k: list(v.shape) for k, v in sd.items()} == golden["param_shapes"]
    assert sd["encoder.embed_tokens.weight"] is sd["shared.weight"]


def test_bucket_restatement_matches_transformers():
    T5Attention = pytest.importorskip("transformers.models.t5.modeling_t5").T5Attention
    rp = torch.arange(-127, 128)[None, :]
    want = T5Attention._relative_position_bucket(rp, bidirectional=True, num_buckets=32, max_distance=128)
    assert torch.equal(plan.t5_relative_position_bucket(rp), want)
    assert torch.equal(OT.relative_position_bucket(rp), want)
    # the table is the bias of those buckets, head-major, offset j - i at column j - i + 127
    w = torch.randn(32, 16)
    tab = plan.t5_bias_table(w)
    assert tab.shape == (16, 255) and torch.equal(tab, w[want[0]].t())


class T5Emulator(Emulator):
    """tests/emulator.py plus the encoder's op kinds (include/aldm_b200.h), in plain fp32."""

    def write_io(self, name, value):
        kind, ref, shape = self.plan.io[name]
        if kind == "i32":
            self.mem[ref.region][ref.off:ref.off + 4 * value.numel()].view(torch.int32)[:] = value.reshape(-1)
        else:
            super().write_io(name, value)

    def op_t5_embed(self, o):
        ids = self.i64(o["ids"], o["rows"])
        assert bool(((ids >= 0) & (ids < o["vocab"])).all())
        self.f32(o["out"], o["rows"] * o["C"])[:] = self.f32(o["table"], o["vocab"] * o["C"]).reshape(-1, o["C"])[ids].reshape(-1)

    def op_t5_rmsnorm(self, o):
        R, C = o["rows"], o["C"]
        x = self.f32(o["x"], R * C).reshape(R, C).clone()
        assert torch.isfinite(x).all(), "rmsnorm reads garbage"
        y = OT.rms_norm(x, self.f32(o["gamma"], C), o["eps"])
        if o.get("out_f32") is not None:
            torch.as_strided(self.f32(o["out_f32"], (R - 1) * o["ldo"] + C), (R, C), (o["ldo"], 1))[:] = y
        else:
            self.write_planes(o["out_hi"], o.get("out_lo"), y, o["ldo"], R)

    def op_t5_attn(self, o):
        B, L, H, C, ld = o["B"], o["L"], o["heads"], o["C"], o["ld_qkv"]
        x = self.f32(o["qkv"], B * L * ld).reshape(B, L, ld)
        q, k, v = (x[..., j * C:(j + 1) * C].reshape(B, L, H, 64).transpose(1, 2) for j in range(3))
        assert torch.isfinite(q).all() and torch.isfinite(k).all() and torch.isfinite(v).all(), "attention reads garbage"
        tab = self.f32(o["bias"], H * 255).reshape(H, 255)
        pos = torch.arange(L)
        s = q @ k.transpose(-1, -2) + tab[:, pos[None, :] - pos[:, None] + 127][None]
        keep = self.f32(o["mask"], B * L).reshape(B, 1, 1, L) == 1
        s = s.masked_fill(~keep, float("-inf"))
        out = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B * L, C)
        self.write_planes(o["out_hi"], o.get("out_lo"), out, o["ldo"], B * L)

    def op_t5_gate(self, o):
        R, F, ld = o["rows"], o["F"], o["ld_x"]
        x = self.f32(o["x"], R * ld).reshape(R, ld)
        y = OT.gelu_new(x[:, :F]) * x[:, F:2 * F]
        n = int((~(y.abs() <= 65504)).sum())
        s = self.mem[o["sat"].region][o["sat"].off:o["sat"].off + 4].view(torch.int32)
        s += n
        self.write_planes(o["out_hi"], o.get("out_lo"), y, o["ldo"], R)


def emulate(ids, mask, weights):
    pl = plan.build_t5(None, ids.shape[0], ids.shape[1], weights=weights)
    em = T5Emulator(pl)
    em.write_io("ids", ids); em.write_io("mask", mask); em.write_io("sat", torch.zeros(weights.n_layer, dtype=torch.int32))
    em.run()
    sat = em.mem["ws"][pl.io["sat"][1].off:][:4 * weights.n_layer].view(torch.int32)
    return em.read_io("hidden"), sat.clone()


@pytest.fixture(scope="module")
def tiny_weights():
    return plan.pack_t5_weights(TC.weights(2))


@pytest.mark.parametrize("name", [n for n, c in TC.CASES.items() if c[0] == 2])
def test_planned_program_matches_reference(golden, tiny_weights, name):
    got, sat = emulate(*TC.inputs(name), tiny_weights)
    assert not sat.any()
    assert per_row(got, golden[name]) < TOL


def test_planned_program_counts_saturation(tiny_weights):
    sd = dict(TC.weights(2))
    sd["encoder.block.1.layer.1.DenseReluDense.wi_1.weight"] = sd["encoder.block.1.layer.1.DenseReluDense.wi_1.weight"] * 1e5
    ids, mask = TC.inputs("tiny_b3_l32")
    _, sat = emulate(ids, mask, plan.pack_t5_weights(sd))
    assert sat[0] == 0 and sat[1] > 0


@pytest.mark.parametrize("B,L", [(1, 1), (3, 32), (8, 128)])
def test_plan_structure(tiny_weights, B, L):
    pl = plan.build_t5(None, B, L, weights=tiny_weights)
    kinds = [o["kind"] for o in pl.ops]
    per_block = ["t5_rmsnorm", "gemm", "t5_attn", "gemm", "t5_rmsnorm", "gemm", "t5_gate", "gemm"]
    assert kinds == ["t5_embed"] + per_block * 2 + ["t5_rmsnorm"]
    assert len(kinds) == 8 * 2 + 2 and (pl.marks["begin"], pl.marks["end"]) == (0, len(kinds))
    assert pl.arena is tiny_weights.arena                      # the plan's own arena is empty: weights are shared
    gemms = [o for o in pl.ops if o["kind"] == "gemm"]
    assert [o["N"] for o in gemms[:4]] == [3072, 1024, 5632, 1024]
    assert all(o["a_lo"] is not None and o["H"] == B * L for o in gemms)     # two planes everywhere
    assert [o["res"] is not None for o in gemms[:4]] == [False, True, False, True]
    assert all(o["out_mode"] == _lib.OUT_F32 for o in gemms)
    gates = [o for o in pl.ops if o["kind"] == "t5_gate"]
    assert [g["sat"].off - pl.io["sat"][1].off for g in gates] == [0, 4]
    assert pl.io["hidden"][2] == (B, L, 1024) and pl.io["ids"][0] == "i64"
    with pytest.raises(ValueError):
        plan.build_t5(None, B, 129, weights=tiny_weights)


@pytest.mark.slow
def test_plan_24_layers():
    """The product shape: 24 blocks -> 194 launches; the shared arena holds shared.weight in fp32 (131 MB) and two fp16
    planes of every block matrix."""
    w = plan.pack_t5_weights(synth.t5_state_dict())
    assert w.n_layer == 24
    for B, L in [(1, 1), (3, 32), (8, 128)]:
        pl = plan.build_t5(None, B, L, weights=w)
        assert len(pl.ops) == 194 and pl.arena is w.arena
    C, F = arch.T5["d_model"], arch.T5["d_ff"]
    mats = 24 * (4 * C * C + 3 * C * F)
    assert 4 * mats + 4 * arch.T5["vocab"] * C <= w.arena.numel() < 4 * mats + 4 * arch.T5["vocab"] * C + 16e6


def test_split_t5_state_dict():
    sd = TC.weights(2)
    pre = "cond_stage_models.0.cond_stage_models.1.model."
    ck = {"model.diffusion_model.out.2.bias": torch.zeros(8), "cond_stage_models.1.model.shared.weight": torch.zeros(1)}
    ck.update({pre + k: v for k, v in sd.items()})
    got = model.split_t5_state_dict(ck, pre)
    assert set(got) == set(sd) - {"encoder.embed_tokens.weight"}
    assert all(got[k] is ck[pre + k] for k in got)
    un, vae, voc, sf = model.split_state_dict(ck)                # unchanged
    assert set(un) == {"out.2.bias"} and not vae and not voc
    bad = dict(ck)
    bad[pre + "encoder.block.1.layer.1.DenseReluDense.wo.weight"] = torch.zeros(1024, 1024)
    with pytest.raises(ValueError, match="wo.weight"):
        model.split_t5_state_dict(bad, pre)
    del ck[pre + "encoder.final_layer_norm.weight"]
    with pytest.raises(KeyError):
        model.split_t5_state_dict(ck, pre)
    with pytest.raises(KeyError):
        model.split_t5_state_dict(ck, "cond_stage_models.7.model.")


def test_token_validation():
    ids, mask = synth.token_ids([5, 3])
    check_tokens(ids, mask)
    check_tokens(ids.int(), mask.long())
    bad = [
        (ids.float(), mask),                                    # not integer
        (ids.clone().fill_(arch.T5["vocab"]), mask),            # id >= vocab
        (ids.clone().fill_(-1), mask),                          # id < 0
        (ids, mask * 0.5),                                      # mask not in {0, 1}
        (ids, torch.cat([mask[:1], torch.zeros_like(mask[1:])])),   # a row without tokens
        (ids[:, :3], mask),                                     # shape mismatch
        (torch.ones(1, 129, dtype=torch.long), torch.ones(1, 129)),  # longer than max_length
        (ids[0], mask[0]),                                      # not [B, L]
    ]
    for i, m in bad:
        with pytest.raises(ValueError):
            check_tokens(i, m)


class _FakeT5:
    def __init__(self):
        self.calls = []

    def encode(self, ids, mask):
        check_tokens(ids, mask)
        self.calls.append(("encode", tuple(ids.shape)))
        return ids[..., None].float().expand(*ids.shape, 1024) * 1e-3

    def unconditional(self, n):
        self.calls.append(("unconditional", n))
        return torch.full((n, 1, 1024), 0.25)


class _FakeGen:
    def __init__(self):
        self.calls = []

    def generate(self, clap, t5, mask):
        self.calls.append((clap.shape[0], tuple(t5.shape), t5.dtype))
        return torch.full((clap.shape[0], 8, 768), 0.5)


def test_routing_token_ids_become_hidden_states():
    cfg = arch.model_config("audioldm2-full")
    prov = pipeline.SyntheticTokenIds(cfg, lens=(12, 5))
    cond = prov.cond({"text": ["a", "b", "c"]})
    ids, mask = cond["crossattn_flan_t5"]
    assert ids.dtype == torch.int64 and ids.shape == (3, 12) and mask.sum(1).tolist() == [12, 5, 12]
    assert pipeline.is_token_level(cond) and not pipeline.is_encoder_level({"crossattn_flan_t5": [ids, mask]})
    t5, gen = _FakeT5(), _FakeGen()
    enc = pipeline.encode_tokens(cfg, cond, lambda: t5)
    assert list(enc) == ["film_clap_cond1", "crossattn_flan_t5"] and t5.calls == [("encode", (3, 12))]
    h, m = enc["crossattn_flan_t5"]
    assert h.shape == (3, 12, 1024) and h.dtype == torch.float32 and m.dtype == torch.float32 and torch.equal(m, mask)
    assert enc["film_clap_cond1"] is cond["film_clap_cond1"]
    out = pipeline.route_conditioning(cfg, enc, lambda: gen)          # then the existing routing: GPT-2, then the UNet
    assert list(out) == ["crossattn_audiomae_generated", "crossattn_flan_t5"] and gen.calls == [(3, (3, 12, 1024), torch.float32)]
    # the unconditional dict: T5("") through unconditional(n), zero AudioMAE tokens kept
    u = pipeline.encode_tokens(cfg, prov.uncond(4), lambda: t5, unconditional=True)
    assert t5.calls[-1] == ("unconditional", 4)
    assert torch.equal(u["crossattn_flan_t5"][0], torch.full((4, 1, 1024), 0.25)) and torch.equal(u["crossattn_flan_t5"][1], torch.ones(4, 1))
    assert not u["crossattn_audiomae_generated"][0].any()
    assert [c.shape[-1] for c in model.unpack_cond_dict(u)["context_list"]] == [768, 1024]
    # other ids in the unconditional dict are encoded, not replaced by T5("")
    pipeline.encode_tokens(cfg, {"crossattn_flan_t5": [ids, mask]}, lambda: t5, unconditional=True)
    assert t5.calls[-1] == ("encode", (3, 12))


def test_routing_t5_models_go_straight_to_the_unet():
    cfg = arch.model_config("audioldm2-full-t5")
    prov = pipeline.SyntheticTokenIds(cfg, lens=(7,))
    cond = prov.cond({"text": ["a", "b"]})
    assert list(cond) == ["crossattn_flan_t5"]
    t5 = _FakeT5()
    out = pipeline.route_conditioning(cfg, pipeline.encode_tokens(cfg, cond, lambda: t5), lambda: _FakeGen())
    assert list(out) == ["crossattn_flan_t5"] and out["crossattn_flan_t5"][0].shape == (2, 7, 1024)
    assert [c.shape[-1] for c in model.unpack_cond_dict(out)["context_list"]] == [1024]


def test_routing_leaves_float_states_untouched():
    cfg = arch.model_config("audioldm2-full")

    def boom():
        raise AssertionError("encoder built for hidden-state conditioning")
    for cond in (pipeline.SyntheticConditioning(cfg).cond({"text": ["a"]}),
                 pipeline.SyntheticEncoderOutputs(cfg).cond({"text": ["a", "b"]}),
                 pipeline.SyntheticEncoderOutputs(cfg).uncond(2)):
        assert pipeline.encode_tokens(cfg, cond, boom) is cond
        assert pipeline.encode_tokens(cfg, cond, boom, unconditional=True) is cond


def test_routing_rejects_models_without_t5():
    cfg = arch.model_config("audioldm_48k")
    assert not arch.has_t5(cfg) and arch.has_t5(arch.model_config("audioldm2-full-large-1150k"))
    ids, mask = synth.token_ids([3])
    with pytest.raises(ValueError, match="no Flan-T5 context"):
        pipeline.encode_tokens(cfg, {"crossattn_flan_t5": [ids, mask]}, lambda: _FakeT5())
    with pytest.raises(ValueError):
        pipeline.SyntheticTokenIds(cfg)


def test_model_without_t5_weights_rejects_token_ids():
    ld = pipeline.NativeAudioLDM2.__new__(pipeline.NativeAudioLDM2)
    ld._t5, ld._t5_sd, ld._t5_uncond_sd = None, None, None
    with pytest.raises(ValueError, match="Flan-T5 weights"):
        ld.t5_encoders()


def test_synthetic_weights_keep_activations_bounded():
    """Over 24 blocks the residual stream stays O(1) and the gated product far inside the fp16 range."""
    sd = synth.t5_state_dict()
    ids, mask = synth.token_ids([128, 40], seed=3)
    h = OT.t5_encode(sd, ids, mask, 24, dtype=torch.float32)
    assert torch.isfinite(h).all() and float(h.abs().max()) < 20
    assert math.isclose(float(sd["shared.weight"].std()), 1.0, rel_tol=0.01)
