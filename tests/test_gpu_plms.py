"""GPU tests of the PLMS sampler (use_plms=True): the plms_step kernel against float64 inside guard bands, the engine
seam's argument checks, the tiny and full-size samplers against the unmodified reference PLMSSampler's fixtures
(tests/golden/make_plms_golden.py), the public pipeline calls against the oracle fed with the replayed CUDA draws,
lanes, and rank shards.  Tolerances are those of tests/test_gpu_nets.py: TINY_WAVE_TOL on the tiny topology, 1e-3
(the north-star tolerance) at full size."""
import numpy as np
import pytest
import torch

from audioldm2_b200 import _lib, arch, parallel, synth
from oracle import functional as OF
from oracle import plms as OP
from tests.conftest import rel_l2
from tests.golden import cases, plms_cases
from tests.test_gpu_kernel_conformance import U, _flat, _Slab, _within
from tests.test_gpu_kernel_matrix import Win, _n_sm
from tests.test_gpu_nets import DEV, TINY_WAVE_TOL, WAVE_TOL, _check, _engine, _oracle_wave, _to

pytestmark = pytest.mark.gpu

AB = {1: [1.0], 2: [3.0, -1.0], 3: [23.0, -16.0, 5.0], 4: [55.0, -59.0, 37.0, -9.0]}
DEN = {0: 2.0, 1: 1.0, 2: 2.0, 3: 12.0, 4: 24.0}


# ----------------------------------------------------------------------------------------------
# the kernel (aldm_plms_step)
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("with_px0", [True, False])
@pytest.mark.parametrize("guidance", [1.0, 3.5])
@pytest.mark.parametrize("order", [0, 1, 2, 3, 4])
def test_plms_step(order, guidance, with_px0):
    """plms_step on n / 4 > 8 * SMs * 256 float4 (every thread runs the grid-stride loop two or three times), at step
    index 7 of a 10-step schedule.  Reference: float64 with the launcher's fp32 coefficients.  Bound: each fp32
    operation rounds at u of its operands' magnitude: |d e| <= 3 u (|U| + g (|C| + |U|)); for e' = sum c_j v_j / den
    (v_0 = e, order 0: (h1 + e) / 2), |d e'| <= (|c_0| |d e| + 2 k u sum |c_j v_j|) / den + u |e'| with k terms;
    |d p0| <= (s1m |d e'| + 3 u (|X| + s1m |e'|)) / sqrt(a_t) + u |p0|; |d x'| <= sqrt(a_prev) |d p0| + dir |d e'| +
    3 u (sqrt(a_prev) |p0| + dir |e'|).  Every operation is rounded in the reference's order, so x_prev, pred_x0 and
    e_t also equal, bit for bit, the reference's fp32 expressions evaluated by torch on the CPU.  Regions not written
    (pred_x0 when NULL, e_t with the first-step average) stay untouched."""
    st = OF.ddim_schedule(OF.ddpm_tables(), 10, 0.0)[7]
    f = np.float32
    sqrt_at, s1m = float(np.sqrt(f(st["a_t"]))), float(f(st["sqrt_one_minus_at"]))
    sqrt_ap, dr = float(np.sqrt(f(st["a_prev"]))), float(np.sqrt(f(f(1.0) - f(st["a_prev"]))))
    n = 4 * (8 * _n_sm() * 256 * 2 + 777)
    g = torch.Generator().manual_seed(order + int(10 * guidance))
    X, Uu, Cn, H1, H2, H3 = (torch.randn(n, generator=g) for _ in range(6))
    nh = 1 if order == 0 else order - 1
    slab = _Slab()
    offs = [slab.put(t) for t in (X, Uu, Cn, H1, H2, H3)]
    o_et, o_xp, o_px = slab.region(n * 4), slab.region(n * 4), slab.region(n * 4)
    store = order != 0
    L = _lib.lib()

    def go(ptr, s):
        held = [ptr(offs[3 + j]) if j < nh else None for j in range(3)]
        _lib.check(L.aldm_plms_step(ptr(offs[0]), ptr(offs[1]), ptr(offs[2]), *held, order, ptr(o_et) if store else None,
                                    ptr(o_xp), ptr(o_px) if with_px0 else None, n, st["a_t"], st["a_prev"],
                                    st["sqrt_one_minus_at"], guidance, s), "plms_step")

    wins = [Win(o_xp, 1, n, n, 4)] + ([Win(o_px, 1, n, n, 4)] if with_px0 else []) + ([Win(o_et, 1, n, n, 4)] if store else [])
    ws = slab.run(go, wins)
    x, u_, cn, h1, h2, h3 = (t.to(DEV, torch.float64) for t in (X, Uu, Cn, H1, H2, H3))
    e = u_ + guidance * (cn - u_)
    de = 3 * U * (u_.abs() + guidance * (cn.abs() + u_.abs()))
    if order == 0:
        terms, c0 = [h1, e], 1.0
    else:
        terms, c0 = [c * v for c, v in zip(AB[order], [e, h1, h2, h3])], AB[order][0]
    ep = sum(terms) / DEN[order]
    dep = (abs(c0) * de + 2 * len(terms) * U * sum(t.abs() for t in terms)) / DEN[order] + U * ep.abs()
    p0 = (x - s1m * ep) / sqrt_at
    xp = sqrt_ap * p0 + dr * ep
    dp = (s1m * dep + 3 * U * (x.abs() + s1m * ep.abs())) / sqrt_at + U * p0.abs()
    dx = sqrt_ap * dp + dr * dep + 3 * U * (sqrt_ap * p0.abs() + dr * ep.abs())
    name = f"plms order={order} g={guidance}"
    _within(f"{name} x_prev", _flat(ws, o_xp, n), xp, dx, 1e-6)
    if with_px0:
        _within(f"{name} pred_x0", _flat(ws, o_px, n), p0, dp, 1e-6)
    # the reference's fp32 expressions (plms.py:288-358), on the CPU
    e32 = Uu + guidance * (Cn - Uu)
    if order == 0:
        ep32 = (H1 + e32) / 2
    elif order == 1:
        ep32 = e32
    else:
        ep32 = OP.plms_eps_prime(e32, [H3, H2, H1][3 - (order - 1):])
    xp32, p032 = OP.plms_update(X.reshape(1, -1), ep32.reshape(1, -1), st)
    assert torch.equal(_flat(ws, o_xp, n).cpu(), xp32.reshape(-1)), f"{name}: x_prev differs from the fp32 reference"
    if with_px0:
        assert torch.equal(_flat(ws, o_px, n).cpu(), p032.reshape(-1)), f"{name}: pred_x0 differs from the fp32 reference"
    if store:
        assert torch.equal(_flat(ws, o_et, n).cpu(), e32), f"{name}: stored e_t differs from e_u + g (e_c - e_u)"


def test_engine_plms_step_rejects_bad_arguments(tiny):
    """Checked before the UNet runs: the order's held values, x_prev aliasing x_base, the first-step average storing."""
    L, st = _lib.lib(), torch.cuda.current_stream().cuda_stream
    x = torch.zeros(2, *arch.tiny_config()["latent"], device=DEV)
    y, h = torch.empty_like(x), torch.zeros_like(x)
    p = lambda t: t.data_ptr()
    call = lambda xb, held, order, et, out: L.aldm_engine_plms_step(tiny._engine, p(x), 501, p(xb), *held, order, et, 0.5,
                                                                    0.6, 0.7, 3.5, p(out), None, st)
    assert call(x, [p(h), None, None], 3, p(y), h) == -1
    assert call(x, [None, None, None], _lib.PLMS_AVERAGE, None, y) == -1
    assert call(x, [p(h), None, None], _lib.PLMS_AVERAGE, p(h), y) == -1
    assert call(x, [p(h), p(h), p(h)], 5, None, y) == -1
    assert call(x, [None, None, None], 1, None, x) == -1                # x_prev == x_base
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------
# the sampler against the reference's PLMSSampler
# ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny():
    return _engine(arch.tiny_config(), 2, 5)


TINY = {"plms_tiny": (5, 3.5, False), "plms_tiny_g1": (5, 1.0, False), "plms_tiny_masked": (5, 3.5, True),
        "plms_tiny_s6": (6, 3.5, False)}


@pytest.mark.parametrize("name", sorted(TINY))
def test_plms_tiny_vs_reference(name, tiny):
    S, guidance, masked = TINY[name]
    cfg = arch.tiny_config()
    fx = cases.load(name)
    _, _, cond, unc = cases.unet_inputs(cfg, 2, t5_len=5)
    x_T, qn, steps, _ = plms_cases.plms_noise(cfg, 2, S, masked=masked)
    mask = x0 = None
    if masked:
        mask, x0 = (t.to(DEV) for t in cases.inpaint_mask(cfg, 2))
    log = []
    z = tiny.generate_latent(_to(cond, DEV), _to(unc, DEV), ddim_steps=S, guidance=guidance, eta=1.0, x_T=x_T,
                             noise_fn=plms_cases.noise_fn(qn, steps, DEV, log), mask=mask, x0=x0, use_plms=True)
    assert len(log) == sum(len(s) for s in steps) + len(qn)
    _check(name, rel_l2(z, fx["latent"]), TINY_WAVE_TOL)


@pytest.fixture(scope="module")
def full():
    return _engine(arch.model_config("audioldm2-full"), 1, 32)


@pytest.mark.parametrize("S", [10, 50])
def test_plms_full_vs_reference(S, full):
    """audioldm2-full, B = 1, guidance 3.5: latent, mel and waveform within the north-star tolerance.  The AB
    combinations' coefficients sum to up to 160 / 24 in absolute value, so the UNet's rounding is amplified more than
    in DDIM's update."""
    cfg = arch.model_config("audioldm2-full")
    fx = cases.load(f"plms_full_{S}")
    _, _, cond, unc = cases.unet_inputs(cfg, 1)
    x_T, qn, steps, _ = plms_cases.plms_noise(cfg, 1, S)
    z = full.generate_latent(_to(cond, DEV), _to(unc, DEV), ddim_steps=S, guidance=3.5, eta=1.0, x_T=x_T,
                             noise_fn=plms_cases.noise_fn(qn, steps, DEV), use_plms=True)
    e_lat = rel_l2(z, fx["latent"])
    mel = full.decode_first_stage(z)
    e_mel = rel_l2(mel, fx["mel"])
    e_wav = rel_l2(full.mel_spectrogram_to_waveform(mel), fx["wave"])
    print(f"plms S={S}: latent {e_lat:.2e} mel {e_mel:.2e} waveform {e_wav:.2e}")
    assert e_lat < WAVE_TOL and e_mel < WAVE_TOL and e_wav < WAVE_TOL


# ----------------------------------------------------------------------------------------------
# the public pipeline calls, against the oracle fed with the replayed CUDA draws
# ----------------------------------------------------------------------------------------------
def _replay_cuda_plms(seed, shape, S, masked):
    """x_T, then per step [q_sample noise] and one draw per update (two at the first step) on the CUDA generator;
    -> (x_T, q draws, torch.randn(4) on the device after the loop)."""
    torch.manual_seed(seed); torch.cuda.manual_seed(seed)
    x_T = torch.randn(shape, device=DEV).cpu()
    qn = []
    for i in range(plms_cases.plms_num_steps(S)):
        if masked:
            qn.append(torch.randn(shape, device=DEV).cpu())
        for _ in range(2 if i == 0 else 1):
            torch.randn(shape, device=DEV)
    return x_T, qn, torch.randn(4, device=DEV).cpu()


def test_pipeline_text_to_audio_plms_tiny():
    import audioldm2_b200 as A
    cfg = arch.tiny_config()
    ld = A.build_model(config=cfg, t5_len=5)
    B, S, seed = 2, 4, 7
    wav = A.text_to_audio(ld, "a dog barking", seed=seed, ddim_steps=S, duration=1.25, batchsize=B, n_candidate_gen_per_text=1,
                          use_plms=True)
    after = torch.randn(4, device=DEV).cpu()
    C_, T, F_ = cfg["latent"]
    x_T, _, want_after = _replay_cuda_plms(seed, (B, C_, T, F_), S, False)
    assert torch.equal(after, want_after), "the CUDA generator is not where the reference's draws leave it"
    cond, unc = synth.conditioning(cfg, B, seed=77, t5_len=5)
    with torch.no_grad():
        z = OP.plms_sample(synth.unet_state_dict(cfg["unet"]), cfg["unet"], x_T, cond, unc, S, 3.5,
                           OF.ddpm_tables(cfg["linear_start"], cfg["linear_end"], cfg["timesteps"]))
        ref = _oracle_wave(cfg, z)
    assert isinstance(wav, np.ndarray) and wav.shape == tuple(ref.shape)
    _check("pipeline text_to_audio plms tiny", rel_l2(torch.from_numpy(wav), ref), TINY_WAVE_TOL)


def test_pipeline_super_resolution_and_inpainting_plms_tiny():
    import audioldm2_b200 as A
    from audioldm2_b200 import frontend
    from oracle import mel as OM
    cfg = arch.tiny_config()
    vc = cfg["vocoder"]
    ld = A.build_model(config=cfg, t5_len=5)
    B, S, seed = 2, 4, 11
    wav_in = cases.wav_input(5000).numpy()[0]
    out = A.super_resolution_and_inpainting(ld, "x", seed=seed, ddim_steps=S, duration=1.28, batchsize=B,
                                            n_candidate_gen_per_text=1, waveform=wav_in, waveform_sr=vc["sampling_rate"],
                                            use_plms=True)
    after = torch.randn(4, device=DEV).cpu()
    x = np.clip(frontend.prepare_waveform(wav_in, 4000, 4000, 128 * vc["hop_size"]), -1, 1)
    logmel, _ = OM.stft_mel(x, vc["n_fft"], vc["hop_size"], vc["num_mels"], vc["sampling_rate"], vc["fmin"], vc["fmax"])
    fb = torch.from_numpy(logmel[0].T[:128]).float()
    C_, T, F_ = cfg["latent"]
    torch.manual_seed(seed)
    post = torch.randn(B, C_, T, F_)                                     # CPU draw (distributions.py:38)
    x_T, qn, want_after = _replay_cuda_plms(seed, (B, C_, T, F_), S, True)
    assert torch.equal(after, want_after), "the CUDA generator is not where the reference's draws leave it"
    vsd = synth.vae_state_dict(cfg["vae"])
    with torch.no_grad():
        mom = OF.vae_encode_moments(vsd, cfg["vae"], fb[None, None].expand(B, 1, -1, -1).contiguous())
        x0 = OF.posterior_sample(mom, post, 1.0)
        mask = torch.ones(B, 1, T, F_)
        mask[:, :, int(T * 0.40):int(T * 0.6), :] = 0
        cond, unc = synth.conditioning(cfg, B, seed=77, t5_len=5)
        z = OP.plms_sample(synth.unet_state_dict(cfg["unet"]), cfg["unet"], x_T, cond, unc, S, 2.5,
                           OF.ddpm_tables(cfg["linear_start"], cfg["linear_end"], cfg["timesteps"]), mask=mask, x0=x0,
                           q_noises=qn)
        ref = _oracle_wave(cfg, z)
    assert out.shape == tuple(ref.shape)
    _check("pipeline sr_inpainting plms tiny", rel_l2(torch.from_numpy(out), ref), TINY_WAVE_TOL)


# ----------------------------------------------------------------------------------------------
# lanes and rank shards
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("masked", [False, True])
def test_two_lanes_equal_two_single_lane_runs(masked):
    """Lane l of a 2-lane engine (B = 4) runs the B = 2 plan on rows [2 l, 2 l + 2): its PLMS result, history ring
    slices included, equals bit for bit a 1-lane B = 2 engine run on those rows."""
    cfg = arch.tiny_config()
    _, _, cond, unc = cases.unet_inputs(cfg, 4, t5_len=5)
    x_T, qn, steps, _ = plms_cases.plms_noise(cfg, 4, 5, masked=masked)
    mask = x0 = None
    if masked:
        mask, x0 = cases.inpaint_mask(cfg, 4)
        mask[1, :, :, :3] = 0
    kw = lambda lo, hi: dict(x_T=x_T[lo:hi], noise_fn=plms_cases.noise_fn([q[lo:hi] for q in qn],
                                                                          [[s[lo:hi] for s in st] for st in steps], DEV),
                             mask=None if mask is None else mask[lo:hi].to(DEV), x0=None if x0 is None else x0[lo:hi].to(DEV))
    two = _engine(cfg, 4, 5, lanes=2)
    assert two.lanes == 2
    z2 = two.generate_latent(_to(cond, DEV), _to(unc, DEV), ddim_steps=5, guidance=3.5, use_plms=True, **kw(0, 4)).clone()
    del two
    one = _engine(cfg, 2, 5, lanes=1)
    for lo in (0, 2):
        c, u = parallel.shard_rows(cond, lo, lo + 2), parallel.shard_rows(unc, lo, lo + 2)
        z1 = one.generate_latent(_to(c, DEV), _to(u, DEV), ddim_steps=5, guidance=3.5, use_plms=True, **kw(lo, lo + 2))
        assert torch.equal(z1, z2[lo:lo + 2]), f"rows {lo}..{lo + 1}: {rel_l2(z1, z2[lo:lo + 2]):.3e}"


def test_rank_shards_reproduce_single_process_batch(tiny):
    """Two ranks (B = 1 each, full-batch noise drawn through ShardedNoise and sliced) == one process with B = 2, and every
    rank's generator ends where the single process's does: ShardedNoise draws once per call, in the sampler's order."""
    cfg = arch.tiny_config()
    S = 4
    cond, unc = synth.conditioning(cfg, 2, seed=77, t5_len=5)
    sn = parallel.ShardedNoise(2, 0, 2, cfg["latent"], DEV, seed=42)
    z_full = tiny.generate_latent(_to(cond, DEV), _to(unc, DEV), ddim_steps=S, guidance=3.5, x_T=sn.x_T(), noise_fn=sn,
                                  use_plms=True).clone()
    e1 = _engine(cfg, 1, 5)
    for r in range(2):
        sr_ = parallel.ShardedNoise(2, r, r + 1, cfg["latent"], DEV, seed=42)
        c, u = parallel.shard_rows(cond, r, r + 1), parallel.shard_rows(unc, r, r + 1)
        z = e1.generate_latent(_to(c, DEV), _to(u, DEV), ddim_steps=S, guidance=3.5, x_T=sr_.x_T(), noise_fn=sr_,
                               use_plms=True)
        assert rel_l2(z, z_full[r:r + 1]) < 1e-3, r      # B = 1 and B = 2 plans may split K differently
        assert torch.equal(sr_.gen.get_state(), sn.gen.get_state()), r
