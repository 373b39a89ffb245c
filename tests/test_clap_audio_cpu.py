"""CPU checks of the CLAP audio encoder and the native re-ranker: the float64 oracle against the reference fixtures, the
host-built tables (resample taps, bicubic weights, relative-position gather, shift masks) against torchaudio, torch and
the reference module's buffers, the checkpoint split, the pack-time fp16 bounds, the planned program (structure, and run
op by op on an emulator) and the ranker's draw order."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from audioldm2_b200 import _lib, arch, model, pipeline, plan, synth
from audioldm2_b200.clap import NativeCLAPRanker
from oracle import clap_audio as OA
from tests.conftest import rel_l2
from tests.emulator import Emulator
from tests.golden import clap_audio_cases as CA

TOL = 2e-5          # oracle (float64) against the reference (fp32 torch), relative L2 per clip
EMU_TOL = 2e-5      # the planned program on the emulator (fp16 two-plane GEMM operands) against the reference


@pytest.fixture(scope="module")
def golden():
    return CA.load()


def per_clip(got, ref):
    return max(rel_l2(got[b], ref[b]) for b in range(ref.shape[0]))


@pytest.mark.parametrize("name", list(CA.CASES))
def test_oracle_matches_reference(golden, name):
    depths, sr, _, _, _ = CA.CASES[name]
    got = OA.clap_audio_embed(CA.weights(depths), CA.inputs(name), sr, depths=depths)
    assert per_clip(got, golden[name]) < TOL


def test_oracle_cos_similarity_matches_reference(golden):
    """The seeded cos_similarity call: the same replaced rows (audio draws first), the same chosen candidates and the
    same CPU generator state afterwards."""
    from oracle import clap as OC
    wav, texts, B = CA.rank_inputs()
    sd_t = CA.text_weights()
    ids, mask = synth.clap_tokenize(texts)
    uncond = OC.clap_text_embed(sd_t, *synth.clap_tokenize([""]), CA.TEXT_LAYERS)
    torch.manual_seed(int(golden["rank_seed"]))
    sim, ra, rt = OA.cos_similarity(lambda: OA.clap_audio_embed(CA.weights(CA.SMALL), wav, 16000, depths=CA.SMALL),
                                    lambda: OC.clap_text_embed(sd_t, ids, mask, CA.TEXT_LAYERS), uncond)
    assert torch.equal(torch.get_rng_state(), golden["rank_rng_state"])
    assert ra == golden["rank_audio_replaced"].tolist() and rt == golden["rank_text_replaced"].tolist()
    assert ra and rt
    assert OA.select(sim, B) == golden["rank_best"].tolist()
    assert (sim - golden["rank_similarity"].double()).abs().max() < 1e-5


# ---- host tables -------------------------------------------------------------------------------------------------
def test_relative_position_index_matches_reference(golden):
    assert torch.equal(plan.htsat_relative_position_index(), golden["relative_position_index"].long())
    assert torch.equal(OA.relative_position_index(), golden["relative_position_index"].long())


@pytest.mark.parametrize("R", [64, 32, 16])
def test_shift_masks_match_reference(golden, R):
    m = plan.htsat_shift_mask(R)
    assert m.shape == ((R // 8) ** 2, 64, 64)
    assert bool(((m == 0) | (m == -100)).all())
    bits = np.unpackbits(golden[f"attn_mask_bits.{R}"].numpy())[:m.numel()]
    assert np.array_equal(bits, (m != 0).numpy().reshape(-1).astype(np.uint8))
    assert torch.equal(OA.shift_mask(R, 8, 4), m)


def test_resample_taps_reproduce_torchaudio():
    """On unit impulses at every phase and near both ends, the taps give torchaudio.functional.resample's output."""
    ta = pytest.importorskip("torchaudio")
    taps = plan.htsat_resample_taps()
    assert taps.shape == (3, 15)
    L = 40
    for p in (0, 1, 6, 7, 20, 32, 39):
        x = torch.zeros(1, L)
        x[0, p] = 1.0
        want = ta.functional.resample(x, 16000, 48000)[0]
        got = torch.zeros(3 * L)
        for i in range(3 * L):
            q, j = divmod(i, 3)
            m = p - q + 7
            if 0 <= m < 15:
                got[i] = taps[j, m]
        assert torch.equal(got, want), p
        assert (OA.resample_16k_to_48k(x)[0] - want).abs().max() < 1e-6


@pytest.mark.parametrize("T", [2, 33, 501, 1001])
def test_bicubic_weights_reproduce_interpolate(T):
    """On impulses at both ends and inside, the host / kernel weights reproduce F.interpolate to a few fp32 ulps (torch's
    CPU kernel may evaluate the same cubic-convolution expressions in another order)."""
    rows, w = plan.htsat_bicubic(T)
    for p in sorted({0, 1, T // 2, T - 2, T - 1}):
        x = torch.zeros(1, 1, T, 64)
        x[0, 0, p, :] = 1.0
        want = F.interpolate(x, (1024, 64), mode="bicubic", align_corners=True)[0, 0, :, 5]
        xt = x[0, 0, :, 5]
        got = xt[rows[:, 0]] * w[:, 0]                                 # the kernel's order: taps i0 - 1 .. i0 + 2
        for k in range(1, 4):
            got = got + xt[rows[:, k]] * w[:, k]
        assert (got - want).abs().max() <= 4e-6, (T, p)          # fp32 weights: within a few ulps of torch's


# ---- weights ---------------------------------------------------------------------------------------------------------
def test_state_dict_matches_reference_names(golden):
    ref = {k: v for k, v in golden["param_shapes"].items()
           if not k.endswith(("relative_position_index", "attn_mask", "num_batches_tracked"))
           and not k.startswith(("audio_branch.tscam_conv.", "audio_branch.head."))}
    assert {k: list(v) for k, v in arch.clap_audio_param_shapes().items()} == ref
    sd = synth.clap_audio_state_dict(depths=CA.SMALL)
    assert {k: list(v.shape) for k, v in sd.items()} == {k: list(v) for k, v in arch.clap_audio_param_shapes(CA.SMALL).items()}


def _ckpt(sd, prefix="clap.model."):
    out = {prefix + k: v for k, v in sd.items()}
    out[prefix + "audio_branch.tscam_conv.weight"] = torch.zeros(527, 1024, 2, 3)
    out[prefix + "audio_branch.head.weight"] = torch.zeros(527, 527)
    out[prefix + "audio_branch.layers.0.blocks.1.attn_mask"] = plan.htsat_shift_mask(64)
    out[prefix + "audio_branch.layers.0.blocks.0.attn.relative_position_index"] = plan.htsat_relative_position_index()
    out[prefix + "audio_branch.bn0.num_batches_tracked"] = torch.tensor(0)
    out[prefix + "text_branch.pooler.dense.bias"] = torch.zeros(768)
    return out


def test_split_clap_audio_state_dict():
    sd = CA.weights(CA.SMALL)
    got = model.split_clap_audio_state_dict(_ckpt(sd), "clap.model.")
    assert set(got) == set(sd) and all(torch.equal(got[k], sd[k]) for k in sd)
    bad = _ckpt(sd)
    bad["clap.model.audio_branch.spectrogram_extractor.stft.conv_imag.weight"] = -bad[
        "clap.model.audio_branch.spectrogram_extractor.stft.conv_imag.weight"]
    with pytest.raises(ValueError, match="DFT basis"):
        model.split_clap_audio_state_dict(bad, "clap.model.")
    bad = _ckpt(sd)
    bad["clap.model.audio_branch.logmel_extractor.melW"] = torch.zeros(513, 32)
    with pytest.raises(ValueError):
        model.split_clap_audio_state_dict(bad, "clap.model.")
    bad = _ckpt(sd)
    del bad["clap.model.audio_projection.2.bias"]
    with pytest.raises(KeyError):
        model.split_clap_audio_state_dict(bad, "clap.model.")


@pytest.mark.parametrize("key,layer", [("audio_branch.layers.1.blocks.0.norm1.weight", "layers.1.blocks.0.norm1"),
                                       ("audio_branch.layers.0.blocks.1.mlp.fc1.weight", "layers.0.blocks.1.mlp.fc1"),
                                       ("audio_branch.layers.2.downsample.norm.bias", "layers.2.downsample.norm")])
def test_pack_refuses_weights_beyond_fp16(key, layer):
    sd = dict(CA.weights(CA.SMALL))
    sd[key] = sd[key] * 1e6
    with pytest.raises(ValueError, match=layer.replace(".", r"\.")):
        plan.pack_clap_audio_weights(sd)


def test_fp16_bounds_hold_for_synthetic_weights():
    w = plan.pack_clap_audio_weights(CA.weights(CA.BASE))
    assert max(w.bounds.values()) < plan.FP16_MAX / 100
    assert len(w.bounds) == 18 * 4 + 3


# ---- the planned program ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def small_weights():
    return plan.pack_clap_audio_weights(CA.weights(CA.SMALL))


@pytest.mark.parametrize("n,L,sr", [(1, 5120, 16000), (6, 40000, 16000), (3, 491520, 48000)])
def test_plan_structure(small_weights, n, L, sr):
    pl = plan.build_clap_audio(None, n, L, sr, weights=small_weights)
    kinds = [o["kind"] for o in pl.ops]
    blocks = sum(CA.SMALL)
    gelu_launches = sum(-(-n * (64 >> i) ** 2 // plan.HTSAT_GELU_ROWS) * d for i, d in enumerate(CA.SMALL))
    assert kinds[:2] == ["htsat_logmel", "htsat_patch"] and kinds[-1] == "htsat_head"
    assert kinds.count("htsat_attn") == blocks and kinds.count("prep") == 2 * blocks
    assert kinds.count("gemm") == 4 * blocks + 3 and kinds.count("htsat_merge") == 3
    assert kinds.count("clap_gelu") == gelu_launches
    assert len(pl.ops) == 2 + blocks * 7 + gelu_launches + 3 * 2 + 1
    att = [o for o in pl.ops if o["kind"] == "htsat_attn"]
    assert [o["shift"] for o in att] == [0, 4, 0, 4, 0, 4, 0, 0]
    assert all((o["mask"] is None) == (o["shift"] == 0) for o in att)
    lm = pl.ops[0]
    assert lm["T"] == arch.clap_audio_frames(L, sr) and (lm["up"] == 3) == (sr == 16000)
    assert (lm["taps"] is None) == (sr == 48000)
    pl.resolve(1 << 32, 1 << 40)                     # every op kind has a descriptor


def test_plan_full_depth_launches():
    w = plan.pack_clap_audio_weights(CA.weights(CA.BASE))
    pl = plan.build_clap_audio(None, 24, 163840, 16000, weights=w)
    # 18 blocks of 7 ops + the GELU launches (24 x 4096 rows in chunks of 32768: 3 per stage-1 block, 1 elsewhere)
    assert len(pl.ops) == 2 + 18 * 7 + (2 * 3 + 2 + 12 + 2) + 3 * 2 + 1


def test_plan_rejects_bad_inputs(small_weights):
    with pytest.raises(ValueError):
        plan.build_clap_audio(None, 1, 170, 16000, weights=small_weights)       # 510 samples at 48 kHz
    with pytest.raises(ValueError):
        plan.build_clap_audio(None, 1, 512, 48000, weights=small_weights)
    with pytest.raises(ValueError):
        plan.build_clap_audio(None, 1, 40000, 22050, weights=small_weights)
    plan.build_clap_audio(None, 1, 171, 16000, weights=small_weights)          # 513 samples: the shortest accepted


class AudioEmulator(Emulator):
    """tests/emulator.py plus the audio encoder's op kinds (include/aldm_b200.h), in plain fp32."""

    def op_clap_gelu(self, o):
        R, Fd, ld = o["rows"], o["F"], o["ld_x"]
        x = self.f32(o["x"], R * ld).reshape(R, ld)[:, :Fd]
        self.write_planes(o["out_hi"], o.get("out_lo"), F.gelu(x), o["ldo"], R)

    def op_htsat_logmel(self, o):
        n, L, T, up = o["n"], o["L"], o["T"], o["up"]
        x = self.f32(o["wav"], n * L).reshape(n, L)
        if up == 3:
            taps = self.f32(o["taps"], 45).reshape(3, 15)
            y = F.conv1d(F.pad(x, (7, 8))[:, None], taps[:, None]).transpose(1, 2).reshape(n, -1)[:, :3 * L]
            x = y
        x = x[:, :o["L48"]]
        basis = model.htsat_dft_basis()
        sd = {"audio_branch.spectrogram_extractor.stft.conv_real.weight": basis[0].float(),
              "audio_branch.spectrogram_extractor.stft.conv_imag.weight": basis[1].float(),
              "audio_branch.logmel_extractor.melW": self.f32(o["melW"], 513 * 64).reshape(513, 64)}
        for k, r in (("running_mean", "bn_mean"), ("running_var", "bn_var"), ("weight", "bn_w"), ("bias", "bn_b")):
            sd[f"audio_branch.bn0.{k}"] = self.f32(o[r], 64)
        y = OA.logmel(sd, x, o["eps"])
        assert y.shape == (n, T, 64)
        self.f32(o["out"], n * T * 64)[:] = y.reshape(-1)

    def op_htsat_patch(self, o):
        n, T = o["n"], o["T"]
        mel = self.f32(o["mel"], n * T * 64).reshape(n, T, 64)
        rows, w = plan.htsat_bicubic(T)
        xt = (mel[:, rows] * w[None, :, :, None]).sum(2)                       # [n, 1024, 64]
        img = xt.permute(0, 2, 1).reshape(n, 64, 4, 256).permute(0, 2, 1, 3).reshape(n, 1, 256, 256)
        h = F.conv2d(img, self.f32(o["w"], 2048).reshape(128, 1, 4, 4), self.f32(o["bias"], 128), stride=4)
        h = F.layer_norm(h.flatten(2).transpose(1, 2), (128,), self.f32(o["gamma"], 128), self.f32(o["beta"], 128), o["eps"])
        self.f32(o["out"], n * 4096 * 128)[:] = h.reshape(-1)

    def op_htsat_attn(self, o):
        n, R, s, H, C = o["n"], o["R"], o["shift"], o["heads"], o["C"]
        x = self.f32(o["qkv"], n * R * R * 3 * C).reshape(n, R, R, 3 * C)
        assert torch.isfinite(x).all(), "attention reads garbage"
        if s:
            x = torch.roll(x, (-s, -s), (1, 2))
        xw = OA.partition(x, 8).reshape(-1, 64, 3, H, 32).permute(2, 0, 3, 1, 4)
        att = (xw[0] * o["scale"]) @ xw[1].transpose(-1, -2) + self.f32(o["bias"], H * 4096).reshape(1, H, 64, 64)
        if s:
            att = (att.view(n, -1, H, 64, 64) + self.f32(o["mask"], (R // 8) ** 2 * 4096).reshape(1, -1, 1, 64, 64)).view(
                -1, H, 64, 64)
        out = OA.unpartition((torch.softmax(att, -1) @ xw[2]).transpose(1, 2).reshape(-1, 8, 8, C), 8, R, R)
        if s:
            out = torch.roll(out, (s, s), (1, 2))
        self.write_planes(o["out_hi"], o.get("out_lo"), out.reshape(-1, C), o["ldo"], n * R * R)

    def op_htsat_merge(self, o):
        n, R, C = o["n"], o["R"], o["C"]
        x = self.f32(o["x"], n * R * R * C).reshape(n, R, R, C)
        cat = torch.cat([x[:, 0::2, 0::2], x[:, 1::2, 0::2], x[:, 0::2, 1::2], x[:, 1::2, 1::2]], -1).reshape(-1, 4 * C)
        y = F.layer_norm(cat, (4 * C,), self.f32(o["gamma"], 4 * C), self.f32(o["beta"], 4 * C), o["eps"])
        self.write_planes(o["out_hi"], o.get("out_lo"), y, o["ldo"], y.shape[0])

    def op_htsat_head(self, o):
        n, t, C, Pj = o["n"], o["ntok"], o["C"], o["P"]
        x = self.f32(o["x"], n * t * C).reshape(n, t, C)
        m = F.layer_norm(x, (C,), self.f32(o["gamma"], C), self.f32(o["beta"], C), o["eps"]).mean(1)
        h = torch.relu(m @ self.f32(o["w1_t"], C * Pj).reshape(C, Pj) + self.f32(o["b1"], Pj))
        y = h @ self.f32(o["w2_t"], Pj * Pj).reshape(Pj, Pj) + self.f32(o["b2"], Pj)
        self.f32(o["out"], n * Pj)[:] = F.normalize(y, dim=-1).reshape(-1)


@pytest.mark.parametrize("name", ["small_16k_short", "small_48k_10s"])
def test_planned_program_matches_reference(golden, small_weights, name):
    _, sr, L, n, _ = CA.CASES[name]
    pl = plan.build_clap_audio(None, n, L, sr, weights=small_weights)
    em = AudioEmulator(pl)
    em.write_io("wav", CA.inputs(name))
    em.run()
    got = em.read_io("embed")
    assert per_clip(got, golden[name]) < EMU_TOL


# ---- the ranker's draws ----------------------------------------------------------------------------------------------
class _StubAudio:
    """A distinct unit row per waveform, derived from its samples (a wrong row mapping changes the similarities)."""

    def embed(self, w):
        return F.normalize(w.repeat(1, 6)[:, :512], dim=-1)


class _StubText:
    def __init__(self):
        self.u = F.normalize(torch.ones(1, 512), dim=-1)

    def unconditional(self):
        return self.u

    def embed(self, ids, mask):
        return F.normalize(torch.cat([ids[:, 1:], ids[:, :1]], 1).float() + 1.0, dim=-1)


def test_ranker_draw_order():
    """2 n draws: n for the audio rows, then n for the text rows; a replaced row is CLAP("")."""
    rk = NativeCLAPRanker(_StubAudio(), _StubText(), synth.clap_tokenize)
    wav, texts = torch.randn(6, 100), [f"t{i}" for i in range(6)]
    for seed in range(200):
        torch.manual_seed(seed)
        sim = rk(wav, texts)
        st = torch.get_rng_state()
        torch.manual_seed(seed)
        da = [float(torch.rand(1)) < 0.1 for _ in range(6)]
        dt = [float(torch.rand(1)) < 0.1 for _ in range(6)]
        assert torch.equal(st, torch.get_rng_state())
        a, t = _StubAudio().embed(wav), _StubText().embed(*synth.clap_tokenize(texts))
        u = _StubText().u
        for i in range(6):
            a_i = u[0] if da[i] else a[i]
            t_i = u[0] if dt[i] else t[i]
            assert abs(float(sim[i]) - float(F.cosine_similarity(a_i, t_i, dim=0))) < 1e-6
        if any(da) and any(dt):
            break
    else:
        raise AssertionError("no seed replaced both an audio and a text row")


def test_ranker_sharded_rows_match_one_process():
    """A rank holding global rows ``rows`` of a call of n_total rows makes all 2 n_total draws in global order: its
    similarities are the single process's at those rows, and the generator state after the call is the same."""
    rk = NativeCLAPRanker(_StubAudio(), _StubText(), synth.clap_tokenize)
    B, n_gen = 4, 3
    wav, texts = torch.randn(B * n_gen, 100), [f"p{i % B}" for i in range(B * n_gen)]
    torch.manual_seed(3)
    full = rk(wav, texts)
    st = torch.get_rng_state()
    for lo, hi in ((0, 2), (2, 4)):
        rows = [i + k * B for k in range(n_gen) for i in range(lo, hi)]
        torch.manual_seed(3)
        part = rk(wav[rows], [texts[r] for r in rows], rows=rows, n_total=B * n_gen)
        assert torch.equal(torch.get_rng_state(), st)
        assert torch.allclose(part, full[rows], atol=1e-6)


def test_build_model_rejects_ranker_and_clap_tokenize():
    import inspect
    p = inspect.signature(pipeline.build_model).parameters["clap_tokenize"]
    assert p.kind == inspect.Parameter.KEYWORD_ONLY and p.default is None
    with pytest.raises(ValueError, match="not both"):
        pipeline.build_model(model_name="audioldm_48k", ranker=lambda w, t: torch.zeros(len(t)),
                             clap_tokenize=synth.clap_tokenize, device="cpu")


def test_clap_tokenize_is_deterministic():
    a, ma = synth.clap_tokenize(["a dog", "", "rain on a roof"])
    b, mb = synth.clap_tokenize(["rain on a roof", "a dog"])
    assert torch.equal(a[0], b[1]) and torch.equal(a[2], b[0]) and torch.equal(ma[0], mb[1])
    assert a[1, :3].tolist() == [0, 2, 1] and ma[1].sum() == 2
    assert not torch.equal(synth.clap_tokenize(["a dog"], seed=1)[0], synth.clap_tokenize(["a dog"], seed=2)[0])
