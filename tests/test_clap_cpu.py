"""CPU checks of the CLAP text encoder: the float64 oracle against the reference fixtures, the planned program (run op by
op by an emulator that knows the encoder's op kinds) against them, the op-table structure, the trim to the longest valid
row, the pack-time fp16 bounds, the checkpoint split, token validation, the conditioning routing and the reference's
random replacement by CLAP("") (its draws, in one process and over two gloo ranks)."""
import os

import pytest
import torch
import torch.nn.functional as F

from audioldm2_b200 import _lib, arch, model, pipeline, plan, synth
from audioldm2_b200.clap import check_tokens, effective_length, empty_prompt, is_empty_prompt
from oracle import clap as OC
from tests.conftest import rel_l2
from tests.emulator import Emulator
from tests.golden import clap_cases as CC

TOL = 2e-6          # oracle (float64) against the reference (fp32 torch), relative L2 per row
EMU_TOL = 2e-5      # the emulated program (fp16 two-plane GEMM operands, fp32 arithmetic), relative L2 per row


@pytest.fixture(scope="module")
def golden():
    return CC.load()


def per_row(got, ref):
    return max(rel_l2(got[b], ref[b]) for b in range(ref.shape[0]))


def _case(name):
    return pytest.param(name, marks=pytest.mark.slow) if CC.CASES[name][0] == 12 else name


@pytest.mark.parametrize("name", [_case(n) for n in CC.CASES])
def test_oracle_matches_reference(golden, name):
    n_layer = CC.CASES[name][0]
    ids, mask = CC.inputs(name)
    got = OC.clap_text_embed(CC.weights(n_layer), ids, mask, n_layer)
    assert got.dtype == torch.float64 and got.shape == golden[name].shape
    assert per_row(got, golden[name]) < TOL


@pytest.mark.parametrize("name", ["tiny_uncond", pytest.param("full_uncond", marks=pytest.mark.slow)])
def test_oracle_matches_reference_uncond(golden, name):
    n_layer = CC.UNCOND[name]
    got = OC.clap_text_embed(CC.weights(n_layer), *empty_prompt(1), n_layer)
    assert rel_l2(got, golden[name]) < TOL


def test_position_ids_follow_transformers():
    """HF's position ids come from the ids (pad id 1), not from the mask: interior pad ids keep position 1 and do not
    advance the count."""
    create = pytest.importorskip("transformers.models.roberta.modeling_roberta").RobertaEmbeddings.create_position_ids_from_input_ids
    ids = torch.tensor([[0, 5, 1, 7, 2, 1, 1], [0, 1, 1, 9, 9, 2, 1]])
    assert torch.equal(OC.position_ids(ids), create(ids, 1))
    assert OC.position_ids(ids)[0].tolist() == [2, 3, 1, 4, 5, 1, 1]


def test_state_dict_matches_reference_keys(golden):
    sd = synth.clap_text_state_dict()
    ref = {k: v for k, v in golden["param_shapes"].items() if not k.endswith(("position_ids", "token_type_ids"))}
    assert {k: list(v.shape) for k, v in sd.items()} == ref


class ClapEmulator(Emulator):
    """tests/emulator.py plus the encoder's op kinds (include/aldm_b200.h), in plain fp32."""

    def op_clap_embed(self, o):
        B, L, C = o["B"], o["L"], o["C"]
        ids = self.i64(o["ids"], B * L).reshape(B, L)
        assert bool(((ids >= 0) & (ids < o["vocab"])).all())
        word = self.f32(o["word"], o["vocab"] * C).reshape(-1, C)
        pos = self.f32(o["pos"], o["n_pos"] * C).reshape(-1, C)
        x = (word[ids] + self.f32(o["type"], C)) + pos[OC.position_ids(ids, o["pad"])]
        self.f32(o["out"], B * L * C)[:] = x.reshape(-1)

    def op_clap_ln(self, o):
        R, C = o["rows"], o["C"]
        x = self.f32(o["x"], R * C).reshape(R, C).clone()
        assert torch.isfinite(x).all(), "layernorm reads garbage"
        y = F.layer_norm(x, (C,), self.f32(o["gamma"], C), self.f32(o["beta"], C), o["eps"])
        self.f32(o["out_f32"], R * C)[:] = y.reshape(-1)
        self.write_planes(o["out_hi"], o.get("out_lo"), y, o["ldo"], R)

    def op_clap_attn(self, o):
        B, L, H, C, ld = o["B"], o["L"], o["heads"], o["C"], o["ld_qkv"]
        x = self.f32(o["qkv"], B * L * ld).reshape(B, L, ld)
        q, k, v = (x[..., j * C:(j + 1) * C].reshape(B, L, H, 64).transpose(1, 2) for j in range(3))
        assert torch.isfinite(q).all() and torch.isfinite(k).all() and torch.isfinite(v).all(), "attention reads garbage"
        s = (q @ k.transpose(-1, -2)) * 0.125
        keep = self.f32(o["mask"], B * L).reshape(B, 1, 1, L) == 1
        out = (torch.softmax(s.masked_fill(~keep, float("-inf")), -1) @ v).transpose(1, 2).reshape(B * L, C)
        self.write_planes(o["out_hi"], o.get("out_lo"), out, o["ldo"], B * L)

    def op_clap_gelu(self, o):
        R, Fd, ld = o["rows"], o["F"], o["ld_x"]
        x = self.f32(o["x"], R * ld).reshape(R, ld)[:, :Fd]
        self.write_planes(o["out_hi"], o.get("out_lo"), F.gelu(x), o["ldo"], R)

    def op_clap_head(self, o):
        B, L, C, Pj = o["B"], o["L"], o["C"], o["P"]
        h = self.f32(o["x"], B * L * C).reshape(B, L, C)[:, 0]
        p = torch.tanh(h @ self.f32(o["wp_t"], C * C).reshape(C, C) + self.f32(o["bp"], C))
        t = torch.relu(p @ self.f32(o["w1_t"], C * Pj).reshape(C, Pj) + self.f32(o["b1"], Pj))
        y = t @ self.f32(o["w2_t"], Pj * Pj).reshape(Pj, Pj) + self.f32(o["b2"], Pj)
        self.f32(o["out"], B * Pj)[:] = F.normalize(y, dim=-1).reshape(-1)


def emulate(ids, mask, weights):
    """The encoder's host path on the emulator: validation, the trim to L_eff, the plan of (B, L_eff)."""
    check_tokens(ids, mask)
    L = effective_length(mask)
    pl = plan.build_clap_text(None, ids.shape[0], L, weights=weights)
    em = ClapEmulator(pl)
    em.write_io("ids", ids[:, :L]); em.write_io("mask", mask[:, :L])
    em.run()
    return em.read_io("embed")


@pytest.fixture(scope="module")
def tiny_weights():
    return plan.pack_clap_weights(CC.weights(2))


@pytest.mark.parametrize("name", [n for n, c in CC.CASES.items() if c[0] == 2])
def test_planned_program_matches_reference(golden, tiny_weights, name):
    ids, mask = CC.inputs(name)
    got = emulate(ids, mask, tiny_weights)
    assert per_row(got, golden[name]) < EMU_TOL
    ref = OC.clap_text_embed(CC.weights(2), ids, mask, 2)          # float64, all 512 positions
    assert per_row(got, ref) < EMU_TOL


def test_planned_program_matches_reference_uncond(golden, tiny_weights):
    assert rel_l2(emulate(*empty_prompt(1), tiny_weights), golden["tiny_uncond"]) < EMU_TOL


@pytest.mark.slow
def test_planned_program_12_layers(golden):
    w = plan.pack_clap_weights(CC.weights(12))
    ids, mask = CC.inputs("full_b3")
    assert per_row(emulate(ids, mask, w), golden["full_b3"]) < EMU_TOL


@pytest.mark.parametrize("B,L", [(1, 2), (3, 40), (8, 512)])
def test_plan_structure(tiny_weights, B, L):
    pl = plan.build_clap_text(None, B, L, weights=tiny_weights)
    kinds = [o["kind"] for o in pl.ops]
    per_block = ["gemm", "clap_attn", "gemm", "clap_ln", "gemm", "clap_gelu", "gemm", "clap_ln"]
    assert kinds == ["clap_embed", "clap_ln"] + per_block * 2 + ["clap_head"]
    assert (pl.marks["begin"], pl.marks["end"]) == (0, len(kinds))
    assert pl.arena is tiny_weights.arena                      # the plan's own arena is empty: weights are shared
    gemms = [o for o in pl.ops if o["kind"] == "gemm"]
    assert [o["N"] for o in gemms[:4]] == [2304, 768, 3072, 768]
    assert all(o["a_lo"] is not None and o["H"] == B * L and o["bias"] is not None for o in gemms)   # two planes, biases
    assert [o["res"] is not None for o in gemms[:4]] == [False, True, False, True]
    assert all(o["out_mode"] == _lib.OUT_F32 for o in gemms)
    assert pl.io["embed"][2] == (B, 512) and pl.io["ids"] == ("i64", pl.io["ids"][1], (B, L))
    with pytest.raises(ValueError):
        plan.build_clap_text(None, B, 513, weights=tiny_weights)


def test_plan_length_is_the_longest_valid_row():
    """512-padded tokenizer output is planned on L_eff, not 512; a mask hole inside a row does not shorten it."""
    ids, mask = synth.clap_token_ids([40, 13, 2])
    assert ids.shape == (3, 512) and effective_length(mask) == 40
    mask[0, 20:39] = 0
    assert effective_length(mask) == 40
    assert effective_length(empty_prompt(4)[1]) == 2


@pytest.mark.slow
def test_plan_12_layers():
    """The product shape: 12 blocks -> 99 launches; the shared arena holds the embeddings in fp32 and two fp16 planes of
    every block matrix, about half a gigabyte."""
    w = plan.pack_clap_weights(synth.clap_text_state_dict())
    assert w.n_layer == 12
    for B, L in [(1, 2), (8, 77), (8, 512)]:
        pl = plan.build_clap_text(None, B, L, weights=w)
        assert len(pl.ops) == 99 and pl.arena is w.arena
    A = arch.CLAP_TEXT
    C, Fd = A["d_model"], A["d_ff"]
    mats = 12 * (4 * C * C + 2 * C * Fd)
    emb = (A["vocab"] + A["max_positions"]) * C
    assert 4 * mats + 4 * emb <= w.arena.numel() < 4 * mats + 4 * emb + 16e6
    assert 0.45e9 < w.arena.numel() < 0.6e9


def test_fp16_bounds_hold_for_synthetic_weights():
    """The pack-time bounds cover every value the oracle's run writes into an operand plane (LayerNorm outputs, v, the
    intermediate pre-activation), and sit far inside the fp16 range for the synthetic weights."""
    sd = CC.weights(2)
    w = plan.pack_clap_weights(sd)
    assert len(w.bounds) == 1 + 4 * 2 and max(w.bounds.values()) < 200
    ids, mask = CC.inputs("tiny_b8")
    seen = {}
    sdd = {k: v.double() for k, v in sd.items()}
    e = "text_branch.embeddings"
    ln = lambda n, x: F.layer_norm(x, (768,), sdd[n + ".weight"], sdd[n + ".bias"], 1e-5)
    lin = lambda n, x: x @ sdd[n + ".weight"].t() + sdd[n + ".bias"]
    h = ln(f"{e}.LayerNorm", sdd[f"{e}.word_embeddings.weight"][ids] + sdd[f"{e}.token_type_embeddings.weight"][0]
           + sdd[f"{e}.position_embeddings.weight"][OC.position_ids(ids)])
    seen[f"{e}.LayerNorm"] = h
    ext = (1.0 - mask.double())[:, None, None, :] * torch.finfo(torch.float64).min
    for i in range(2):
        p = f"text_branch.encoder.layer.{i}"
        q, k, v = (lin(f"{p}.attention.self.{n}", h) for n in ("query", "key", "value"))
        seen[f"{p}.attention.self.value"] = v
        split = lambda t: t.reshape(8, 512, 12, 64).transpose(1, 2)
        o = (torch.softmax(split(q) @ split(k).transpose(-1, -2) / 8 + ext, -1) @ split(v)).transpose(1, 2).reshape(8, 512, 768)
        assert float(o.abs().max()) <= float(v.abs().max()) + 1e-9        # a convex combination of rows of v
        h = ln(f"{p}.attention.output.LayerNorm", lin(f"{p}.attention.output.dense", o) + h)
        seen[f"{p}.attention.output.LayerNorm"] = h
        u = lin(f"{p}.intermediate.dense", h)
        seen[f"{p}.intermediate.dense"] = u
        h = ln(f"{p}.output.LayerNorm", lin(f"{p}.output.dense", OC.gelu(u)) + h)
        seen[f"{p}.output.LayerNorm"] = h
    assert set(seen) == set(w.bounds)
    for name, t in seen.items():
        assert float(t.abs().max()) <= w.bounds[name], name


@pytest.mark.parametrize("key,scale,layer", [
    ("text_branch.encoder.layer.1.intermediate.dense.weight", 1e4, "text_branch.encoder.layer.1.intermediate.dense"),
    ("text_branch.encoder.layer.0.attention.self.value.bias", 1e6, "text_branch.encoder.layer.0.attention.self.value"),
    ("text_branch.encoder.layer.1.output.LayerNorm.weight", 5e3, "text_branch.encoder.layer.1.output.LayerNorm"),
])
def test_pack_refuses_weights_beyond_fp16(key, scale, layer):
    """A host-side check on the weights alone: no GPU, no run."""
    sd = dict(CC.weights(2))
    sd[key] = sd[key] * scale
    with pytest.raises(ValueError, match=layer.replace(".", r"\.")):
        plan.pack_clap_weights(sd)


def test_split_clap_text_state_dict(golden):
    sd = CC.weights(2)
    pre = "cond_stage_models.0.cond_stage_models.0.model."
    ck = {"model.diffusion_model.out.2.bias": torch.zeros(8), pre + "audio_branch.spectrogram_extractor.stft.conv_real.weight":
          torch.zeros(3), pre + "logit_scale_a": torch.zeros(()), pre + "text_branch.embeddings.position_ids":
          torch.arange(514)[None], pre + "text_branch.embeddings.token_type_ids": torch.zeros(1, 514, dtype=torch.long)}
    ck.update({pre + k: v for k, v in sd.items()})
    got = model.split_clap_text_state_dict(ck, pre)
    assert set(got) == set(sd) and all(got[k] is ck[pre + k] for k in got)
    # the reference's own names (HF RobertaModel under text_branch., text_projection) are what the split asks for
    ref12 = {k for k in golden["param_shapes"] if not k.endswith(("position_ids", "token_type_ids"))}
    assert set(arch.clap_text_param_shapes(12)) == ref12
    un, vae, voc, sf = model.split_state_dict(ck)                # unchanged
    assert set(un) == {"out.2.bias"} and not vae and not voc
    bad = dict(ck)
    bad[pre + "text_branch.encoder.layer.1.output.dense.weight"] = torch.zeros(768, 768)
    with pytest.raises(ValueError, match="output.dense.weight"):
        model.split_clap_text_state_dict(bad, pre)
    del ck[pre + "text_projection.2.bias"]
    with pytest.raises(KeyError):
        model.split_clap_text_state_dict(ck, pre)
    with pytest.raises(KeyError):
        model.split_clap_text_state_dict(ck, "cond_stage_models.7.model.")


def test_token_validation():
    ids, mask = synth.clap_token_ids([5, 3])
    check_tokens(ids, mask)
    check_tokens(ids.int(), mask.long())
    check_tokens(ids[:, :5], mask[:, :5])
    bad = [
        (ids.float(), mask),                                    # not integer
        (ids.clone().fill_(arch.CLAP_TEXT["vocab"]), mask),     # id >= vocab
        (ids.clone().fill_(-1), mask),                          # id < 0
        (ids, mask * 0.5),                                      # mask not in {0, 1}
        (ids, torch.cat([mask[:1], torch.zeros_like(mask[1:])])),   # a row without tokens
        (ids[:, :3], mask),                                     # shape mismatch
        (torch.ones(1, 513, dtype=torch.long), torch.ones(1, 513)),  # longer than max_length
        (ids[0], mask[0]),                                      # not [B, L]
    ]
    for i, m in bad:
        with pytest.raises(ValueError):
            check_tokens(i, m)


def test_empty_prompt():
    ids, mask = empty_prompt(3)
    assert ids.shape == (3, 512) and ids[0, :3].tolist() == [0, 2, 1] and mask[0, :3].tolist() == [1, 1, 0]
    assert is_empty_prompt(ids, mask) and is_empty_prompt(*empty_prompt(2, 2))
    i2, m2 = synth.clap_token_ids([2, 2])
    assert is_empty_prompt(i2, m2)
    i3, m3 = synth.clap_token_ids([3, 2])
    assert not is_empty_prompt(i3, m3)


# ----------------------------------------------------------------------------------------------
# routing
# ----------------------------------------------------------------------------------------------
class _FakeClap:
    def __init__(self):
        self.calls = []

    def embed(self, ids, mask):
        check_tokens(ids, mask)
        self.calls.append(("embed", tuple(ids.shape)))
        return F.normalize(ids[:, :8].float().repeat(1, 64) + 1.0, dim=-1)

    def unconditional(self):
        self.calls.append(("unconditional",))
        return torch.full((1, 512), 512 ** -0.5)


class _FakeT5:
    def encode(self, ids, mask):
        return ids[..., None].float().expand(*ids.shape, 1024) * 1e-3

    def unconditional(self, n):
        return torch.full((n, 1, 1024), 0.25)


class _FakeGen:
    def __init__(self):
        self.calls = []

    def generate(self, clap, t5, mask):
        self.calls.append((tuple(clap.shape), clap.dtype))
        return torch.full((clap.shape[0], 8, 768), 0.5)


NO_DRAWS = lambda n: [False] * n


def test_routing_48k_token_ids_become_the_film_vector():
    cfg = arch.model_config("audioldm_48k")
    prov = pipeline.SyntheticPromptTokens(cfg, lens=(12, 5))
    cond = prov.cond({"text": ["a", "b", "c"]})
    assert list(cond) == ["film_clap_cond1"]
    ids, mask = cond["film_clap_cond1"]
    assert ids.dtype == torch.int64 and ids.shape == (3, 512) and mask.sum(1).tolist() == [12, 5, 12]
    assert pipeline.is_clap_token_level(cond) and not pipeline.is_token_level(cond)
    clap = _FakeClap()
    out = pipeline.encode_clap_tokens(cfg, cond, lambda: clap, decide=NO_DRAWS)
    assert clap.calls == [("embed", (3, 512))]
    e = out["film_clap_cond1"]
    assert e.shape == (3, 1, 512) and e.dtype == torch.float32
    assert pipeline.route_conditioning(cfg, out, lambda: _FakeGen()) is out          # no generator for 48k
    y = model.unpack_cond_dict(out)["y"]
    assert y.shape == (3, 512) and torch.equal(y, e[:, 0])
    # the unconditional dict: the tokenization of "" goes through the cached CLAP("")
    u = pipeline.encode_clap_tokens(cfg, prov.uncond(4), lambda: clap, unconditional=True)
    assert clap.calls[-1] == ("unconditional",) and len(clap.calls) == 2
    assert u["film_clap_cond1"].shape == (4, 1, 512) and torch.equal(u["film_clap_cond1"][3, 0], clap.unconditional()[0])


def test_routing_full_clap_then_t5_then_gpt2():
    cfg = arch.model_config("audioldm2-full")
    prov = pipeline.SyntheticPromptTokens(cfg, lens=(12, 5), t5_lens=(9, 4))
    cond = prov.cond({"text": ["a", "b"]})
    assert list(cond) == ["film_clap_cond1", "crossattn_flan_t5"]
    assert pipeline.is_clap_token_level(cond) and pipeline.is_token_level(cond)
    clap, gen = _FakeClap(), _FakeGen()
    c = pipeline.encode_clap_tokens(cfg, cond, lambda: clap, decide=NO_DRAWS)
    c = pipeline.encode_tokens(cfg, c, lambda: _FakeT5())
    out = pipeline.route_conditioning(cfg, c, lambda: gen)
    assert list(out) == ["crossattn_audiomae_generated", "crossattn_flan_t5"] and gen.calls == [((2, 1, 512), torch.float32)]
    # next to T5 states instead of T5 ids
    h = {"film_clap_cond1": cond["film_clap_cond1"], "crossattn_flan_t5": [torch.randn(2, 9, 1024), torch.ones(2, 9)]}
    c = pipeline.encode_clap_tokens(cfg, h, lambda: clap, decide=NO_DRAWS)
    assert pipeline.is_encoder_level(c) and c["crossattn_flan_t5"] is h["crossattn_flan_t5"]
    # its unconditional dict has no CLAP entry (zero AudioMAE tokens, T5("")): nothing to encode
    u = prov.uncond(3)
    assert "film_clap_cond1" not in u and pipeline.encode_clap_tokens(cfg, u, lambda: clap, unconditional=True) is u


def test_routing_leaves_float_embeddings_untouched():
    def boom():
        raise AssertionError("encoder built for embedding-level conditioning")

    for name in ("audioldm2-full", "audioldm_48k"):
        cfg = arch.model_config(name)
        conds = [pipeline.SyntheticConditioning(cfg).cond({"text": ["a"]}), pipeline.SyntheticConditioning(cfg).uncond(2),
                 {"film_clap_cond1": torch.randn(2, 1, 512)}]
        if arch.has_seqgen(cfg):
            conds.append(pipeline.SyntheticEncoderOutputs(cfg).cond({"text": ["a", "b"]}))
        for cond in conds:
            assert pipeline.encode_clap_tokens(cfg, cond, boom, decide=boom) is cond
            assert pipeline.encode_clap_tokens(cfg, cond, boom, unconditional=True) is cond


def test_routing_rejects_models_without_clap():
    ids, mask = synth.clap_token_ids([3])
    for name in ("audioldm2-full-t5",):
        cfg = arch.model_config(name)
        assert not arch.has_clap(cfg)
        with pytest.raises(ValueError, match="no CLAP"):
            pipeline.encode_clap_tokens(cfg, {"film_clap_cond1": [ids, mask]}, lambda: _FakeClap(), decide=NO_DRAWS)
        with pytest.raises(ValueError):
            pipeline.SyntheticPromptTokens(cfg)
    cfg = arch.tiny_config(film=True)
    with pytest.raises(ValueError, match="no CLAP"):
        pipeline.encode_clap_tokens(cfg, {"film_clap_cond1": [ids, mask]}, lambda: _FakeClap(), decide=NO_DRAWS)


def test_model_without_clap_weights_rejects_token_ids():
    ld = pipeline.NativeAudioLDM2.__new__(pipeline.NativeAudioLDM2)
    ld._clap, ld._clap_sd = None, None
    with pytest.raises(ValueError, match="CLAP text weights"):
        ld.clap_encoder()


# ----------------------------------------------------------------------------------------------
# the reference's random replacement by CLAP("")
# ----------------------------------------------------------------------------------------------
def test_replacement_decisions_match_reference(golden):
    """CLAPAudioEmbeddingClassifierFreev2.forward draws torch.rand(1) once per prompt row, in row order, and replaces the
    rows below 0.1: the fixture's seeded call at B = 8 replaced rows ``forward_replaced``; the same seed gives the same
    rows here and leaves the CPU generator in the same state."""
    torch.manual_seed(int(golden["forward_seed"]))
    got = pipeline.clap_replacement_draws(8, extra=False)
    assert [i for i, r in enumerate(got) if r] == golden["forward_replaced"].tolist() and any(got)
    assert torch.equal(torch.get_rng_state(), golden["forward_rng_state"])


def test_replacement_applies_clap_empty(golden, tiny_weights):
    """The fixture's forward output: the embeddings of its rows, with the replaced rows holding CLAP("")."""
    ids, mask = CC.inputs(CC.FORWARD[1])
    clap = _FakeClap()
    clap.embed = lambda i, m: golden[CC.FORWARD[1]]
    clap.unconditional = lambda: golden["tiny_uncond"]
    torch.manual_seed(int(golden["forward_seed"]))
    out = pipeline.encode_clap_tokens(arch.model_config("audioldm_48k"), {"film_clap_cond1": [ids, mask]}, lambda: clap,
                                      decide=lambda n: pipeline.clap_replacement_draws(n, extra=False))
    assert rel_l2(out["film_clap_cond1"], golden["forward"]) < 1e-6
    for i in golden["forward_replaced"].tolist():
        assert torch.equal(out["film_clap_cond1"][i, 0], golden["tiny_uncond"][0])


class _NoEngine(pipeline.NativeAudioLDM2):
    """The pipeline's conditioning path with fake encoders, recording the CPU generator around it."""

    def __init__(self, cfg, prov):
        super().__init__(cfg, None, None, None, "cpu", cond_provider=prov, clap_sd={}, t5_sd={})
        self._clap = _FakeClap()
        self._t5 = (_FakeT5(), _FakeT5())
        self._seqgen = _FakeGen()


def test_second_call_makes_the_extra_draw():
    """get_input: from the model's second call on, conditional_dry_run_finished makes make_decision(0.0) draw one
    torch.rand(1) before the B replacement draws (ddpm.py:852-854, 916-917)."""
    cfg = arch.model_config("audioldm_48k")
    ld = _NoEngine(cfg, pipeline.SyntheticPromptTokens(cfg, lens=(6, 3)))
    batch = {"text": ["a", "b", "c"]}
    for extra in (0, 1, 1):
        torch.manual_seed(5)
        ld.conditioning(batch)
        after = torch.get_rng_state()
        torch.manual_seed(5)
        torch.rand(3 + extra)
        assert torch.equal(after, torch.get_rng_state()), extra
    # float embeddings draw nothing, first call or not
    ld2 = _NoEngine(cfg, pipeline.SyntheticConditioning(cfg))
    for _ in range(2):
        torch.manual_seed(5)
        before = torch.get_rng_state()
        ld2.conditioning(batch)
        assert torch.equal(before, torch.get_rng_state())


def test_replaced_rows_hold_clap_empty(golden):
    """The pipeline's first call replaces the rows the reference's seeded call replaced."""
    cfg = arch.model_config("audioldm_48k")
    ld = _NoEngine(cfg, pipeline.SyntheticPromptTokens(cfg, lens=(6, 3)))
    torch.manual_seed(int(golden["forward_seed"]))
    c = ld.conditioning({"text": ["x"] * 8})["film_clap_cond1"]
    u = ld._clap.unconditional()[0]
    assert [i for i in range(8) if torch.equal(c[i, 0], u)] == golden["forward_replaced"].tolist()


def _sharded_decisions(rank, world, port, out):
    import torch.distributed as dist
    from audioldm2_b200 import parallel
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    try:
        cfg = arch.model_config("audioldm_48k")
        ld = _NoEngine(cfg, pipeline.SyntheticPromptTokens(cfg, lens=(6, 3)))
        batch = {"text": [f"p{i}" for i in range(8)]}
        rows = []
        for call in range(2):
            torch.manual_seed(0)
            shard = parallel.current_shard(8)
            _, _, lo, hi = shard
            torch.randn(8, 3)                                           # the posterior draw comes first
            c = ld._sharded_conditioning(batch, lo, hi)
            rows.append((lo, hi, c["film_clap_cond1"].clone(), torch.get_rng_state()))
        torch.save(rows, os.path.join(out, f"r{rank}.pt"))
    finally:
        dist.destroy_process_group()


def test_sharded_decisions_match_one_process(tmp_path):
    """Two gloo ranks, each keeping its 4 prompts of 8: the replacement decisions are made for all 8 global rows on every
    rank (after the posterior draw), so each rank's rows and the generator state equal one process's."""
    import socket
    import torch.multiprocessing as mp
    cfg = arch.model_config("audioldm_48k")
    ld = _NoEngine(cfg, pipeline.SyntheticPromptTokens(cfg, lens=(6, 3)))
    batch = {"text": [f"p{i}" for i in range(8)]}
    ref = []
    for call in range(2):
        torch.manual_seed(0)
        torch.randn(8, 3)
        ref.append((ld.conditioning(batch)["film_clap_cond1"].clone(), torch.get_rng_state()))
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    mp.spawn(_sharded_decisions, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    for r in range(2):
        rows = torch.load(tmp_path / f"r{r}.pt")
        for (lo, hi, c, st), (full, st_ref) in zip(rows, ref):
            assert (lo, hi) == (4 * r, 4 * r + 4)
            assert torch.equal(c, full[lo:hi]) and torch.equal(st, st_ref)
    assert any(torch.equal(ref[0][0][i, 0], ld._clap.unconditional()[0]) for i in range(8))
