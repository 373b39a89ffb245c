"""GPU tests of audio-to-audio style transfer: the stochastic_encode kernel bit for bit against torch fp32 inside guard
bands, AudioLDM 1's latent guard decided on the device, decode against a full DDIM run, the engine against the unmodified
reference's fixtures (tests/golden/make_style_golden.py), the public call against the oracle fed with the replayed draws,
and rank shards.  Tolerances are those of tests/test_gpu_nets.py: TINY_WAVE_TOL on the tiny topologies, 1e-3 (the
north-star tolerance) at full size."""
import numpy as np
import pytest
import torch

from audioldm2_b200 import _lib, arch, engine, parallel, synth
from audioldm2_b200.sampler import DDIMSampler
from oracle import functional as OF
from oracle import style as OS
from tests.conftest import rel_l2
from tests.golden import cases, style_cases
from tests.test_gpu_kernel_conformance import _flat, _Slab
from tests.test_gpu_kernel_matrix import Win, _n_sm
from tests.test_gpu_nets import DEV, TINY_WAVE_TOL, WAVE_TOL, _check, _engine, _oracle_wave, _to

pytestmark = pytest.mark.gpu


def _coefs(S=10, t_enc=5):
    steps = OF.ddim_schedule(OF.ddpm_tables(), S, 1.0)
    c0, c1 = OS.encode_coefficients(steps, t_enc)
    return float(c0), float(c1)


def _torch_fp32(x, z, c0, c1, clip):
    x = torch.clip(x, -10, 10) if clip else x
    return torch.tensor(c0, dtype=torch.float32) * x + torch.tensor(c1, dtype=torch.float32) * z


# ----------------------------------------------------------------------------------------------
# the kernel (aldm_stochastic_encode)
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flag", [None, 0, 1])
def test_stochastic_encode_bit_exact_in_guard_bands(flag):
    """n / 4 > 8 * SMs * 256 float4, so every thread runs the grid-stride loop two or three times, with values beyond
    +-10 so that the clip matters.  Equal bit for bit to torch's fp32 c0 * x + c1 * n (clip(x, -10, 10) first when the
    guard word is set); nothing outside the output is written."""
    c0, c1 = _coefs()
    n = 4 * (8 * _n_sm() * 256 * 2 + 777)
    g = torch.Generator().manual_seed(3 + (flag or 0))
    X, Z = 30 * torch.randn(n, generator=g), torch.randn(n, generator=g)
    slab = _Slab()
    ox, oz = slab.put(X), slab.put(Z)
    of = slab.put(torch.tensor([flag or 0], dtype=torch.int32))
    oo = slab.region(n * 4)
    L = _lib.lib()
    ws = slab.run(lambda ptr, s: _lib.check(L.aldm_stochastic_encode(ptr(ox), ptr(oz), ptr(oo), n, c0, c1,
                                                                     ptr(of) if flag is not None else None, s),
                                            "stochastic_encode"), [Win(oo, 1, n, n, 4)])
    got = _flat(ws, oo, n).cpu()
    assert torch.equal(got, _torch_fp32(X, Z, c0, c1, bool(flag)))
    if flag:
        assert not torch.equal(got, _torch_fp32(X, Z, c0, c1, False))


def _guarded(x, z, c0, c1):
    """The device path: flags by torch reductions on the device, decision, one kernel pass."""
    xd, zd = x.to(DEV).contiguous(), z.to(DEV).contiguous()
    flag = parallel.latent_guard_flag(xd)
    return int(flag), engine.stochastic_encode(xd, zd, c0, c1, flag).cpu()


@pytest.mark.parametrize("case", ["max_exactly_100", "just_above_100", "plus_inf", "minus_inf", "nan_present",
                                  "nan_and_over"])
def test_latent_guard_cases(case):
    c0, c1 = _coefs()
    g = torch.Generator().manual_seed(9)
    x, z = 5 * torch.randn(2, 8, 32, 8, generator=g), torch.randn(2, 8, 32, 8, generator=g)
    x[0, 0, 0, 0] = 40.0                                     # beyond the clip bound, below the guard's threshold
    over = torch.nextafter(torch.tensor(100.0), torch.tensor(200.0))
    val = {"max_exactly_100": 100.0, "just_above_100": float(over), "plus_inf": float("inf"),
           "minus_inf": float("-inf"), "nan_present": float("nan"), "nan_and_over": float("nan")}[case]
    x[1, 3, 7, 2] = val
    if case == "nan_and_over":
        x[0, 1, 1, 1] = 1e4
    want_clip = case in ("just_above_100", "plus_inf", "minus_inf")
    flag, got = _guarded(x, z, c0, c1)
    assert flag == int(want_clip)
    ref = _torch_fp32(OS.latent_guard(x), z, c0, c1, False)
    torch.testing.assert_close(got, ref, rtol=0, atol=0, equal_nan=True)
    if case.startswith("nan"):
        assert torch.isnan(got[1, 3, 7, 2]) and int(torch.isnan(got).sum()) == 1     # NaN passed through, not clipped


def test_stochastic_encode_rejects_overlap_on_device_buffers():
    x = torch.zeros(64, device=DEV)
    L = _lib.lib()
    assert L.aldm_stochastic_encode(x.data_ptr(), x.data_ptr(), x.data_ptr() + 16, 32, 1.0, 0.0, None, None) == -1
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------
# decode against a full DDIM run
# ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny():
    return _engine(arch.tiny_config(), 2, 5, with_encoder=True)


@pytest.mark.parametrize("k", [1, 4, 10])
def test_decode_continues_a_ddim_run_bit_for_bit(k, tiny):
    """A full native DDIM run of S steps, and decode(t_start = k) started from that run's state after S - k steps with the
    same remaining noise, end bit-identical: decode runs the last k entries of the same schedule with the same step."""
    cfg, S = arch.tiny_config(), 10
    _, _, cond, unc = cases.unet_inputs(cfg, 2, t5_len=5)
    x_T, noises, _ = cases.sampler_noise(cfg, 2, S)
    nz = [t.to(DEV) for t in noises]
    full = tiny.generate_latent(_to(cond, DEV), _to(unc, DEV), ddim_steps=S, guidance=3.5, eta=1.0, x_T=x_T,
                                noise_fn=lambda i, kind: nz[i]).clone()
    s = DDIMSampler(tiny)
    s.make_schedule(S, ddim_eta=1.0)
    s.steps = s.steps[:S - k]
    mid = s.ddim_sampling(_to(cond, DEV), x_T.shape, x_T=x_T, unconditional_guidance_scale=3.5,
                          unconditional_conditioning=_to(unc, DEV), noise_fn=lambda i, kind: nz[i]).clone()
    d = DDIMSampler(tiny)
    d.make_schedule(S, ddim_eta=1.0)
    out = d.decode(mid, _to(cond, DEV), k, 3.5, _to(unc, DEV), noise_fn=lambda i, kind: nz[S - k + i])
    assert torch.equal(out, full), rel_l2(out, full)


# ----------------------------------------------------------------------------------------------
# the engine against the reference's fixtures
# ----------------------------------------------------------------------------------------------
_ENGINES = {}


def _style_engine(key, B, t5_len, scale_factor):
    k = (key, B, scale_factor)
    if k not in _ENGINES:
        _ENGINES.clear()
        torch.cuda.empty_cache()
        _ENGINES[k] = _engine(style_cases.config(key), B, t5_len, with_encoder=True, scale_factor=scale_factor)
    return _ENGINES[k]


def _run_fixture(name):
    key, B, S, t_enc, guidance, scale_factor, t5_len, _ = style_cases.CASES[name]
    cfg = style_cases.config(key)
    eng = _style_engine(key, B, t5_len, scale_factor)
    _, _, cond, unc = cases.unet_inputs(cfg, B, t5_len=t5_len)
    post, enc, steps, _ = style_cases.style_noise(cfg, B, t_enc)
    x0 = eng.get_first_stage_encoding(eng.encode_first_stage_moments(style_cases.mel(cfg, B).to(DEV)), post)
    nz = [t.to(DEV) for t in steps]
    z = eng.style_transfer_latent(x0, _to(cond, DEV), _to(unc, DEV), t_enc, ddim_steps=S, guidance=guidance,
                                  noise=enc.to(DEV), noise_fn=lambda i, kind: nz[i])
    return eng, z


@pytest.mark.parametrize("name", sorted(n for n, c in style_cases.CASES.items() if c[0].startswith("tiny")))
def test_style_tiny_vs_reference(name):
    fx = cases.load(name)
    _, z = _run_fixture(name)
    _check(name, rel_l2(z, fx["latent"]), TINY_WAVE_TOL)


@pytest.mark.parametrize("name", ["style_full", "style_48k_full"])
def test_style_full_vs_reference(name):
    """audioldm2-full (S = 20) and audioldm_48k (S = 10), B = 1, strength 0.5: latent, mel and waveform within the
    north-star tolerance."""
    fx = cases.load(name)
    eng, z = _run_fixture(name)
    e_lat = rel_l2(z, fx["latent"])
    mel = eng.decode_first_stage(z)
    e_mel = rel_l2(mel, fx["mel"])
    e_wav = rel_l2(eng.mel_spectrogram_to_waveform(mel), fx["wave"])
    print(f"{name}: latent {e_lat:.2e} mel {e_mel:.2e} waveform {e_wav:.2e}")
    assert e_lat < WAVE_TOL and e_mel < WAVE_TOL and e_wav < WAVE_TOL
    _ENGINES.clear()
    torch.cuda.empty_cache()


# ----------------------------------------------------------------------------------------------
# the public call, against the oracle fed with the replayed draws
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant,duration", [("", 1.25), ("48k", 0.625)])
def test_pipeline_style_transfer_tiny(variant, duration):
    import audioldm2_b200 as A
    from audioldm2_b200 import frontend
    from oracle import mel as OM
    cfg = arch.tiny_config(variant=variant)
    vc = cfg["vocoder"]
    ld = A.build_model(config=cfg, t5_len=5)
    B, S, strength, seed = 2, 10, 0.5, 11
    t_enc = int(strength * S)
    wav_in = cases.wav_input(5000).numpy()[0]
    out = A.style_transfer(ld, "a cat meowing", None, strength, seed=seed, duration=duration, batchsize=B, ddim_steps=S,
                           waveform=wav_in, waveform_sr=vc["sampling_rate"])
    after_cuda, after_cpu = torch.randn(4, device=DEV).cpu(), torch.randn(4)
    C_, T, F_ = cfg["latent"]
    frames = T * 2 ** (len(cfg["vae"]["ch_mult"]) - 1)
    x = np.clip(frontend.prepare_waveform(wav_in, 4000, 4000, frames * vc["hop_size"]), -1, 1)
    logmel, _ = OM.stft_mel(x, vc["n_fft"], vc["hop_size"], vc["num_mels"], vc["sampling_rate"], vc["fmin"], vc["fmax"])
    fb = torch.from_numpy(logmel[0].T[:frames]).float()
    torch.manual_seed(seed)
    post = torch.randn(B, C_, T, F_)                                   # CPU draw (distributions.py:38)
    assert torch.equal(after_cpu, torch.randn(4)), "the CPU generator is not where the reference's draws leave it"
    torch.cuda.manual_seed(seed)
    enc = torch.randn(B, C_, T, F_, device=DEV).cpu()                   # randn_like in stochastic_encode
    steps = [torch.randn(B, C_, T, F_, device=DEV).cpu() for _ in range(t_enc)]
    assert torch.equal(after_cuda, torch.randn(4, device=DEV).cpu()), "the CUDA generator is not where the reference's draws leave it"
    vsd = synth.vae_state_dict(cfg["vae"])
    with torch.no_grad():
        mom = OF.vae_encode_moments(vsd, cfg["vae"], fb[None, None].expand(B, 1, -1, -1).contiguous())
        x0 = OF.posterior_sample(mom, post, 1.0)
        cond, unc = synth.conditioning(cfg, B, seed=77, t5_len=5)
        z = OS.style_transfer_latent(synth.unet_state_dict(cfg["unet"]), cfg["unet"], x0, cond, unc, S, t_enc, 2.5, enc,
                                     steps, OF.ddpm_tables(cfg["linear_start"], cfg["linear_end"], cfg["timesteps"]))
        ref = _oracle_wave(cfg, z)
    assert isinstance(out, np.ndarray) and out.dtype == np.float32 and out.shape == tuple(ref.shape)
    _check(f"pipeline style_transfer tiny {variant or '16k'}", rel_l2(torch.from_numpy(out), ref), TINY_WAVE_TOL)


# ----------------------------------------------------------------------------------------------
# rank shards
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("trip", ["none", "rank1_only"])
def test_rank_shards_reproduce_single_process_call(trip, tiny):
    """Two ranks (B = 1 each: full-batch noise drawn through ShardedNoise and sliced, guard flags combined with MAX as
    parallel.reduce_guard_flags does across ranks) == one process with B = 2, including the case where only rank 1's
    row trips the guard; every rank's generator ends where the single process's does."""
    cfg, S, t_enc = arch.tiny_config(), 10, 6
    cond, unc = synth.conditioning(cfg, 2, seed=77, t5_len=5)
    x0 = 3 * cases.latent(cfg, 2, seed=21)
    if trip == "rank1_only":
        x0[1, 2, 5, 3] = 150.0
    x0 = x0.to(DEV)
    sn = parallel.ShardedNoise(2, 0, 2, cfg["latent"], DEV, seed=42)
    z_full = tiny.style_transfer_latent(x0, _to(cond, DEV), _to(unc, DEV), t_enc, ddim_steps=S, guidance=3.5,
                                        noise=sn.x_T(), noise_fn=sn).clone()
    flags = [parallel.guard_flags(x0[r:r + 1]) for r in range(2)]
    reduced = torch.maximum(flags[0], flags[1])                        # dist.all_reduce(MAX) of the two ranks' flags
    assert int(parallel.guard_decision(reduced)) == int(trip != "none")
    e1 = _engine(cfg, 1, 5)
    for r in range(2):
        sr_ = parallel.ShardedNoise(2, r, r + 1, cfg["latent"], DEV, seed=42)
        c, u = parallel.shard_rows(cond, r, r + 1), parallel.shard_rows(unc, r, r + 1)
        z = e1.style_transfer_latent(x0[r:r + 1].contiguous(), _to(c, DEV), _to(u, DEV), t_enc, ddim_steps=S,
                                     guidance=3.5, clip_flag=parallel.guard_decision(reduced), noise=sr_.x_T(),
                                     noise_fn=sr_)
        assert rel_l2(z, z_full[r:r + 1]) < 1e-3, r      # B = 1 and B = 2 plans may split K differently
        assert torch.equal(sr_.gen.get_state(), sn.gen.get_state()), r
        if trip == "rank1_only" and r == 0:              # rank 0's own rows alone would not have clipped
            assert int(parallel.latent_guard_flag(x0[0:1])) == 0
