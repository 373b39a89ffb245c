"""CPU tests of audio-to-audio style transfer: the oracle against the unmodified reference DDIMSampler's
stochastic_encode / decode (tests/golden/make_style_golden.py), the host path's call and draw order, the argument checks
made before any draw, the sizes, the public signature, the C-ABI's argument checks and the 2-rank guard-flag
reduction."""
import ctypes as C
import inspect
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import audioldm2_b200 as A
from audioldm2_b200 import _lib, arch, model, parallel, pipeline, synth
from audioldm2_b200.sampler import DDIMSampler, ddpm_tables, transfer_steps
from oracle import functional as OF
from oracle import style as OS
from tests.conftest import rel_l2
from tests.golden import cases, style_cases

TOL = 2e-5
TINY = sorted(n for n, c in style_cases.CASES.items() if c[0].startswith("tiny"))
FULL = sorted(n for n, c in style_cases.CASES.items() if not c[0].startswith("tiny"))


@pytest.mark.parametrize("name", TINY)
def test_oracle_matches_reference_style_transfer(name):
    key, B, S, t_enc, guidance, scale_factor, t5_len, _ = style_cases.CASES[name]
    cfg = style_cases.config(key)
    fx = cases.load(name)
    post, enc, steps, rng_after = style_cases.style_noise(cfg, B, t_enc)
    assert torch.equal(rng_after, fx["rng_after"])           # the replay makes as many draws as the reference made
    _, _, cond, unc = cases.unet_inputs(cfg, B, t5_len=t5_len)
    with torch.no_grad():
        mom = OF.vae_encode_moments(synth.vae_state_dict(cfg["vae"]), cfg["vae"], style_cases.mel(cfg, B))
        x0 = OF.posterior_sample(mom, post, scale_factor)
        assert rel_l2(OS.latent_guard(x0), fx["init_latent"]) < TOL
        tables = OF.ddpm_tables(cfg["linear_start"], cfg["linear_end"], cfg["timesteps"])
        z_enc = OS.stochastic_encode(fx["init_latent"], OF.ddim_schedule(tables, S, 1.0), t_enc, enc)
        assert torch.equal(z_enc, fx["z_enc"])               # from the reference's own x0: the same fp32 expression
        z = OS.style_transfer_latent(synth.unet_state_dict(cfg["unet"]), cfg["unet"], x0, cond, unc, S, t_enc, guidance,
                                     enc, steps, tables)
    assert rel_l2(z, fx["latent"]) < TOL


def test_guard_fixture_is_clipped():
    fx = cases.load("style_tiny_guard")
    assert float(fx["init_latent"].abs().max()) == 10.0


@pytest.mark.parametrize("name", FULL)
def test_full_fixtures_replay_their_draws(name):
    key, B, S, t_enc, *_ = style_cases.CASES[name]
    cfg = style_cases.config(key)
    assert torch.equal(style_cases.style_noise(cfg, B, t_enc)[3], cases.load(name)["rng_after"])


def test_latent_guard_semantics():
    x = torch.zeros(2, 3)
    x[0, 0] = 100.0                                          # strict comparison: exactly 100 is not clipped
    assert torch.equal(OS.latent_guard(x), x)
    x[1, 1] = 100.5                                          # one row trips the guard: the whole batch is clipped
    x[0, 1] = -30.0
    assert torch.equal(OS.latent_guard(x), torch.clip(x, -10, 10))
    x[1, 2] = float("nan")                                   # a NaN makes the max NaN: nothing is clipped
    assert torch.equal(OS.latent_guard(x).nan_to_num(), x.nan_to_num())
    for v, want in ((100.0, 0), (100.5, 1), (float("inf"), 1), (float("-inf"), 1)):
        y = torch.zeros(4)
        y[2] = v
        assert int(parallel.latent_guard_flag(y)) == want, v
    y[0] = float("nan")
    assert int(parallel.latent_guard_flag(y)) == 0


# ----------------------------------------------------------------------------------------------
# the host path: calls, indices and draws
# ----------------------------------------------------------------------------------------------
def _toy_eps(x, t):
    return 0.3 * x + 0.01 * t + torch.sin(x)


class _FakeModel:
    """The surface DDIMSampler.stochastic_encode / decode drive, in torch on the CPU: every call is recorded and computed
    with the oracle's arithmetic from a toy eps(x, t)."""

    def __init__(self):
        self.num_timesteps, self.device = 1000, torch.device("cpu")
        for k, v in ddpm_tables().items():
            setattr(self, k, v)
        self.calls = []

    def set_conditioning(self, cond, uncond):
        self.calls.append(("cond", cond, uncond))

    def stochastic_encode(self, x0, noise, c0, c1, clip_flag=None):
        self.calls.append(("encode", c0, c1, None if clip_flag is None else int(clip_flag)))
        x = torch.clip(x0, -10, 10) if clip_flag is not None and int(clip_flag) else x0
        return torch.tensor(c0, dtype=torch.float32) * x + torch.tensor(c1, dtype=torch.float32) * noise

    def p_sample_ddim(self, x, st, noise, guidance, out=None, pred_x0=None):
        self.calls.append(("step", st["index"], st["t"]))
        e = _toy_eps(x, st["t"])
        out.copy_(OF.ddim_update(x, e, e, noise, st, guidance)[0])
        return out


def _oracle_toy(x0, S, t_enc, enc, step_noises, guidance):
    steps = OF.ddim_schedule(OF.ddpm_tables(), S, 1.0)
    z = OS.stochastic_encode(OS.latent_guard(x0), steps, t_enc, enc)
    for i, st in enumerate(OS.decode_steps(steps, t_enc)):
        e = _toy_eps(z, st["t"])
        z, _ = OF.ddim_update(z, e, e, step_noises[i], st, guidance)
    return z


@pytest.mark.parametrize("S,t_enc", [(10, 0), (10, 1), (10, 5), (10, 9), (6, 0), (6, 3), (6, 6), (200, 100), (200, 199)])
def test_call_and_draw_order(S, t_enc):
    """make_schedule(S, eta=1.0), one stochastic_encode at index t_enc with fp32 sqrt(ddim_alphas)[t_enc] and
    ddim_sqrt_one_minus_alphas[t_enc], then p_sample_ddim at indices t_enc - 1, ..., 0; torch.randn draws: one of the
    latent's shape for the encode, then one per step -- the reference's count and order."""
    m = _FakeModel()
    shape = (2, 3, 8, 4)
    x0 = 3 * torch.randn(shape, generator=torch.Generator().manual_seed(5))
    torch.manual_seed(11)
    z = model.NativeLatentDiffusion.style_transfer_latent(m, x0, "c", "u", t_enc, ddim_steps=S, guidance=3.5)
    after = torch.randn(4)
    torch.manual_seed(11)
    enc = torch.randn(shape)
    noises = [torch.randn(shape) for _ in range(t_enc)]
    assert torch.equal(after, torch.randn(4))
    steps = OF.ddim_schedule(OF.ddpm_tables(), S, 1.0)
    st = next(s for s in steps if s["index"] == t_enc)
    want = [("encode", float(np.sqrt(np.float32(st["a_t"]))), st["sqrt_one_minus_at"], 0)]
    if t_enc:
        want.append(("cond", "c", "u"))
    want += [("step", t_enc - 1 - i, steps[len(steps) - t_enc + i]["t"]) for i in range(t_enc)]
    assert m.calls == want
    # decoding starts one schedule entry below the encode's noise level (the reference's own offset)
    if t_enc:
        assert m.calls[2][2] < st["t"]
    assert torch.allclose(z, _oracle_toy(x0, S, t_enc, enc, noises, 3.5), rtol=1e-6, atol=1e-6)


def test_decode_guidance_one_loads_the_conditional_branch_twice():
    m = _FakeModel()
    model.NativeLatentDiffusion.style_transfer_latent(m, torch.zeros(1, 3, 8, 4), "c", "u", 3, ddim_steps=10, guidance=1.0)
    assert ("cond", "c", None) in m.calls


def test_recorded_noise_is_used_instead_of_draws():
    m = _FakeModel()
    shape = (1, 3, 8, 4)
    g = torch.Generator().manual_seed(3)
    enc, noises = torch.randn(shape, generator=g), [torch.randn(shape, generator=g) for _ in range(4)]
    log = []
    torch.manual_seed(1)
    z = model.NativeLatentDiffusion.style_transfer_latent(
        m, torch.ones(shape), "c", None, 4, ddim_steps=10, guidance=3.5, noise=enc,
        noise_fn=lambda i, k: (log.append((i, k)), noises[i])[1])
    after = torch.randn(4)
    torch.manual_seed(1)
    assert torch.equal(after, torch.randn(4))                # nothing drawn
    assert log == [(i, "step") for i in range(4)]
    assert torch.allclose(z, _oracle_toy(torch.ones(shape), 10, 4, enc, noises, 3.5), rtol=1e-6, atol=1e-6)


def test_guard_word_reaches_the_encode():
    m = _FakeModel()
    x0 = torch.zeros(1, 3, 8, 4)
    x0[0, 0, 0, 0] = 250.0
    model.NativeLatentDiffusion.style_transfer_latent(m, x0, "c", None, 0, ddim_steps=10)
    assert m.calls[0][3] == 1
    m = _FakeModel()
    model.NativeLatentDiffusion.style_transfer_latent(m, x0, "c", None, 0, ddim_steps=10,
                                                      clip_flag=torch.zeros(1, dtype=torch.int32))
    assert m.calls[0][3] == 0                                # a caller's (all-reduced) decision is used as given


def test_sampler_surface_rejects_what_audioldm_never_passes():
    s = DDIMSampler(_FakeModel())
    s.make_schedule(10, ddim_eta=1.0)
    x = torch.zeros(2, 3, 8, 4)
    with pytest.raises(NotImplementedError):
        s.stochastic_encode(x, 3, use_original_steps=True)
    with pytest.raises(NotImplementedError):
        s.stochastic_encode(x, torch.tensor([3, 4]))
    with pytest.raises(NotImplementedError):
        s.decode(x, "c", 3, use_original_steps=True)
    with pytest.raises(ValueError):
        s.stochastic_encode(x, 10)
    with pytest.raises(ValueError):
        s.decode(x, "c", 11)
    s.stochastic_encode(x, torch.tensor([3, 3]))             # AudioLDM's torch.tensor([t_enc] * B)


# ----------------------------------------------------------------------------------------------
# argument checks before any draw, sizes, signature, export
# ----------------------------------------------------------------------------------------------
def test_transfer_steps():
    assert transfer_steps(0.29, 100) == 28                   # Python float arithmetic, as the reference computes it
    assert transfer_steps(0.5, 200) == 100 and transfer_steps(0.0, 200) == 0 and transfer_steps(0.999, 200) == 199
    assert transfer_steps(1.0, 6) == 6                       # S = 6: 7 schedule entries
    for strength, S in ((1.0, 200), (-0.5, 200), (1.0, 10), (1.5, 6)):
        with pytest.raises(ValueError, match=r"\[0, "):
            transfer_steps(strength, S)


class _Untouchable:
    """A latent_diffusion whose every engine call fails: the checks must come first."""

    cfg = arch.tiny_config()

    def __getattr__(self, name):
        raise AssertionError(f"{name} touched before the argument checks")


@pytest.mark.parametrize("strength,duration", [(1.0, 1.25), (-0.5, 1.25), (0.5, 1.0)])
def test_invalid_calls_raise_before_any_draw(strength, duration):
    wav = np.zeros(8000, dtype=np.float32)                   # 2 s at the tiny config's 4 kHz
    with pytest.raises(ValueError):
        A.style_transfer(_Untouchable(), "x", None, strength, seed=5, duration=duration, ddim_steps=200, waveform=wav,
                         waveform_sr=4000)
    after = torch.randn(4)
    torch.manual_seed(5)
    assert torch.equal(after, torch.randn(4))


def test_sizes():
    assert pipeline.style_transfer_sizes(arch.model_config("audioldm2-full"), 10) == (256, 1024)
    assert pipeline.style_transfer_sizes(arch.model_config("audioldm_48k"), 10) == (128, 1024)
    assert pipeline.style_transfer_sizes(arch.model_config("audioldm2-full"), 5.0)[1] == int(5.0 * 102.4)
    with pytest.raises(ValueError):
        pipeline.style_transfer_sizes(arch.model_config("audioldm2-full"), 3.2)      # 81 latent frames


class _Recorder:
    cfg = arch.model_config("audioldm2-full")
    device = torch.device("cpu")

    def generate_batch_style_transfer(self, batch, transfer_strength, ddim_steps, unconditional_guidance_scale):
        self.got = (batch, transfer_strength, ddim_steps, unconditional_guidance_scale, self.latent_t_size)
        return np.zeros((len(batch["text"]), 1, 8), dtype=np.float32)


@pytest.mark.parametrize("audio_s,duration,want", [(3.2, 10, 5.0), (10.0, 10, 10), (12.0, 10, 10), (7.4, 7.5, 10.0)])
def test_duration_round_up(monkeypatch, audio_s, duration, want):
    assert A.round_up_duration(3.2) == 5.0 and A.round_up_duration(10.0) == 12.5
    seen = {}

    def fbank(ld, original_audio_file_path=None, target_length=1024, waveform=None, sr=None):
        seen["frames"] = target_length
        return torch.zeros(target_length, 64), None

    monkeypatch.setattr(pipeline, "wav_to_fbank", fbank)
    r = _Recorder()
    out = A.style_transfer(r, ["a", "b"], None, 0.5, duration=duration, batchsize=2,
                           waveform=np.zeros(int(audio_s * 16000), np.float32), waveform_sr=16000)
    latent_t, frames = pipeline.style_transfer_sizes(r.cfg, want)
    assert seen["frames"] == frames and r.got[4] == latent_t
    batch, strength, S, g, _ = r.got
    assert batch["text"] == ["a", "b"] and tuple(batch["log_mel_spec"].shape) == (2, frames, 64)
    assert (strength, S, g) == (0.5, 200, 2.5) and out.shape == (2, 1, 8)


def test_signature_and_defaults():
    """AudioLDM 1's style_transfer(latent_diffusion, text, original_audio_file_path, transfer_strength, seed=42,
    duration=10, batchsize=1, guidance_scale=2.5, ddim_steps=200, config=None), plus the keyword-only waveform and
    waveform_sr of super_resolution_and_inpainting."""
    ps = inspect.signature(A.style_transfer).parameters.values()
    pos = [p for p in ps if p.kind == p.POSITIONAL_OR_KEYWORD]
    assert [p.name for p in pos] == ["latent_diffusion", "text", "original_audio_file_path", "transfer_strength", "seed",
                                     "duration", "batchsize", "guidance_scale", "ddim_steps", "config"]
    assert [p.default for p in pos if p.default is not p.empty] == [42, 10, 1, 2.5, 200, None]
    kw = {p.name: p.default for p in ps if p.kind == p.KEYWORD_ONLY}
    assert kw == {"waveform": None, "waveform_sr": None}


def test_export():
    assert A.style_transfer is pipeline.style_transfer and "style_transfer" in A.__all__
    assert callable(A.NativeAudioLDM2.generate_batch_style_transfer)


# ----------------------------------------------------------------------------------------------
# the C-ABI (checked before anything is launched, so these run without a GPU)
# ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def L():
    _lib.build()
    return _lib.lib()


def test_stochastic_encode_argument_checks(L):
    n = 1024
    x, nz, out, flag = (C.c_void_p(a) for a in (1 << 20, 2 << 20, 3 << 20, 4 << 20))
    f = lambda x_=x, n_=nz, o=out, k=n, fl=None: L.aldm_stochastic_encode(x_, n_, o, k, 0.9, 0.4, fl, None)
    assert f(x_=None) == -1 and f(n_=None) == -1 and f(o=None) == -1
    assert f(k=0) == -2 and f(k=1022) == -2 and f(k=-4) == -2
    assert f(x_=C.c_void_p((1 << 20) + 4)) == -3 and f(o=C.c_void_p((3 << 20) + 8)) == -3
    assert f(fl=C.c_void_p((4 << 20) + 2)) == -3
    assert f(o=x) == -1 and f(o=C.c_void_p((1 << 20) + 16)) == -1 and f(o=nz) == -1     # out overlaps x0 / noise
    assert f(o=C.c_void_p((1 << 20) - 4 * n + 16)) == -1
    assert f(fl=C.c_void_p((3 << 20) + 64)) == -1 and b"clip_flag" in L.aldm_last_error()
    assert "aldm_stochastic_encode" in _lib.EXPORTED


# ----------------------------------------------------------------------------------------------
# the guard flags of a sharded call: one MAX all-reduce
# ----------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _guard_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    parallel.init_from_env(backend="gloo")
    out = []
    # (rank 0's rows, rank 1's rows): only one rank over 100; one rank with a NaN; neither over; exactly 100
    for r0, r1 in (((5.0,), (150.0,)), ((500.0,), (float("nan"),)), ((5.0,), (-7.0,)), ((100.0,), (-100.0,)),
                   ((float("-inf"),), (1.0,))):
        x = torch.tensor(r0 if rank == 0 else r1)
        flags = parallel.guard_flags(x)
        mine = flags.clone()
        out.append((mine.tolist(), parallel.reduce_guard_flags(flags).tolist(), int(parallel.latent_guard_flag(x))))
    q.put((rank, out))
    dist.destroy_process_group()


@pytest.mark.timeout(120)
def test_two_rank_guard_flag_reduction():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_guard_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=100) for _ in procs)
    for p in procs:
        p.join(30)
        assert p.exitcode == 0
    want_flags = [[1, 0], [1, 1], [0, 0], [0, 0], [1, 0]]
    want_clip = [1, 0, 0, 0, 1]
    assert [o[0] for o in res[0]] == [[0, 0], [1, 0], [0, 0], [0, 0], [1, 0]]       # the local flags differ by rank
    for r in (0, 1):
        assert [o[1] for o in res[r]] == want_flags and [o[2] for o in res[r]] == want_clip, r
