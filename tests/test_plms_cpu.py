"""CPU tests of the PLMS sampler (use_plms=True): the oracle against the reference fixtures, the host loop's call, history
and RNG order against the reference's, its schedule, the options it rejects, and the C-ABI's argument checks."""
import ctypes as C

import pytest
import torch

from audioldm2_b200 import _lib, arch, synth
from audioldm2_b200.sampler import DDIMSampler, PLMSSampler, ddpm_tables
from oracle import functional as OF
from oracle import plms as OP
from tests.conftest import rel_l2
from tests.golden import cases, plms_cases

TOL = 2e-5
TINY = {"plms_tiny": (5, 3.5, False), "plms_tiny_g1": (5, 1.0, False), "plms_tiny_masked": (5, 3.5, True),
        "plms_tiny_s6": (6, 3.5, False)}


@pytest.mark.parametrize("name", sorted(TINY))
def test_oracle_matches_reference_plms(name):
    S, g, masked = TINY[name]
    cfg = arch.tiny_config()
    fx = cases.load(name)
    _, _, cond, unc = cases.unet_inputs(cfg, 2, t5_len=5)
    x_T, qn, _, rng_after = plms_cases.plms_noise(cfg, 2, S, masked=masked)
    assert torch.equal(rng_after, fx["rng_after"])           # the replay makes as many draws as the reference made
    mask = x0 = None
    if masked:
        mask, x0 = cases.inpaint_mask(cfg, 2)
    with torch.no_grad():
        z = OP.plms_sample(synth.unet_state_dict(cfg["unet"]), cfg["unet"], x_T, cond, unc, S, g,
                           OF.ddpm_tables(cfg["linear_start"], cfg["linear_end"], cfg["timesteps"]), mask, x0, qn)
    assert rel_l2(z, fx["latent"]) < TOL


def test_full_fixtures_replay_their_draws():
    cfg = arch.model_config("audioldm2-full")
    for name, S in (("plms_full_10", 10), ("plms_full_50", 50)):
        assert torch.equal(plms_cases.plms_noise(cfg, 1, S)[3], cases.load(name)["rng_after"]), name


def _toy_eps(x, t):
    return 0.3 * x + 0.01 * t + torch.sin(x)


class _FakeModel:
    """The surface PLMSSampler drives, in torch on the CPU: each p_sample_plms call is recorded and computed with the
    oracle's e' and update from a toy eps(x, t)."""

    def __init__(self):
        self.num_timesteps, self.device = 1000, torch.device("cpu")
        for k, v in ddpm_tables().items():
            setattr(self, k, v)
        self.calls, self.cond = [], None

    def set_conditioning(self, cond, uncond):
        self.cond = (cond, uncond)

    def masked_blend(self, img, x0, mask, q_noise, st):
        self.calls.append(("blend", st["t"]))
        img.copy_(OF.masked_blend(img, x0, mask, q_noise, st))

    def p_sample_plms(self, x_in, t, x_base, held, order, st, guidance, e_t_out=None, out=None, pred_x0=None):
        assert all(h is not x_in and h is not out for h in held) and (e_t_out is None or e_t_out is not out)
        self.calls.append((t, st["t"], order, x_base is x_in, len(held), e_t_out is not None))
        e = _toy_eps(x_in, t)
        if order == _lib.PLMS_AVERAGE:
            ep = (held[0] + e) / 2
        elif order == 1:
            ep = e
        else:
            ep = OP.plms_eps_prime(e, held[::-1])
        x_prev, _ = OP.plms_update(x_base, ep, st)
        if e_t_out is not None:
            e_t_out.copy_(e)
        out.copy_(x_prev)
        return out


def _expected_calls(steps, masked):
    """plms.py:212-258: per step the blend when masked, then the evaluations with (t, step t, order, base is the input)."""
    out = []
    for i, st in enumerate(steps):
        t_next = steps[min(i + 1, len(steps) - 1)]["t"]
        if masked:
            out.append(("blend", st["t"]))
        if i == 0:
            out += [(st["t"], st["t"], 1, True, 0, True), (t_next, st["t"], _lib.PLMS_AVERAGE, False, 1, False)]
        else:
            k = min(i, 3)
            out.append((st["t"], st["t"], k + 1, True, k, True))
    return out


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("S", [1, 2, 5, 6, 10])
def test_loop_order_history_and_draws(S, masked):
    m = _FakeModel()
    shape = (2, 3, 8, 4)
    g = torch.Generator().manual_seed(5)
    x_T = torch.randn(shape, generator=g)
    x0 = torch.randn(shape, generator=g)
    mask = torch.ones(2, 1, 8, 4)
    mask[:, :, 3:5] = 0
    n = plms_cases.plms_num_steps(S)
    qn = [torch.randn(shape, generator=g) for _ in range(n)]
    steps_noise = [[torch.randn(shape, generator=g) for _ in range(2 if i == 0 else 1)] for i in range(n)]
    log = []
    kw = dict(mask=mask, x0=x0) if masked else {}
    z, _ = PLMSSampler(m).sample(S, 2, shape[1:], conditioning="c", eta=1.0, unconditional_guidance_scale=3.5,
                                 unconditional_conditioning="u", x_T=x_T,
                                 noise_fn=plms_cases.noise_fn(qn, steps_noise, log=log), **kw)
    steps = OF.ddim_schedule(ddpm_tables(), S, 0.0)
    assert m.cond == ("c", "u")
    assert m.calls == _expected_calls(steps, masked)
    want = []
    for i in range(n):
        want += ([(i, "q")] if masked else []) + [(i, "step")] * (2 if i == 0 else 1)
    assert log == want
    ref = OP.plms_loop(_toy_eps, steps, x_T, mask if masked else None, x0, qn)
    assert torch.allclose(z, ref, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("masked", [False, True])
def test_default_draws_match_the_reference_count(masked):
    """Without noise_fn the sampler draws with torch.randn as plms.py does: x_T, [q_sample], one per update."""
    m = _FakeModel()
    shape, S = (2, 3, 8, 4), 5
    kw = dict(mask=torch.ones(2, 1, 8, 4), x0=torch.zeros(shape)) if masked else {}
    torch.manual_seed(3)
    PLMSSampler(m).sample(S, 2, shape[1:], conditioning="c", **kw)
    after = torch.randn(4)
    torch.manual_seed(3)
    torch.randn(shape)
    for i in range(S):
        for _ in range((1 if masked else 0) + (2 if i == 0 else 1)):
            torch.randn(shape)
    assert torch.equal(after, torch.randn(4))


def test_guidance_one_loads_the_conditional_branch_twice():
    m = _FakeModel()
    PLMSSampler(m).sample(2, 2, (3, 8, 4), conditioning="c", unconditional_guidance_scale=1.0,
                          unconditional_conditioning="u")
    assert m.cond == ("c", None)


@pytest.mark.parametrize("S", [1, 6, 10, 50, 200])
def test_schedule_is_ddim_with_zero_sigma(S):
    p, d = PLMSSampler(_FakeModel()), DDIMSampler(_FakeModel())
    p.make_schedule(S, ddim_eta=1.0)                    # forced to 0, as plms.py:30 does
    d.make_schedule(S, ddim_eta=0.0)
    assert p.steps == d.steps and all(s["sigma_t"] == 0.0 for s in p.steps)
    assert len(p.steps) == plms_cases.plms_num_steps(S)


@pytest.mark.parametrize("kw", [dict(quantize_x0=True), dict(temperature=0.5), dict(noise_dropout=0.1),
                                dict(score_corrector=object()), dict(ddim_use_original_steps=True), dict(timesteps=3)])
def test_out_of_scope_options_raise(kw):
    with pytest.raises(NotImplementedError):
        PLMSSampler(_FakeModel()).sample(5, 2, (3, 8, 4), conditioning="c", **kw)


def test_schedule_past_the_table_raises_as_the_reference_does():
    """S = 3: range(0, 1000, 333) + 1 ends at timestep 1000, outside the 1000-entry table; the reference's
    make_ddim_sampling_parameters raises IndexError there, and so does this schedule."""
    with pytest.raises(IndexError):
        PLMSSampler(_FakeModel()).make_schedule(3)


def test_quad_discretisation_raises():
    with pytest.raises(AssertionError):
        PLMSSampler(_FakeModel()).make_schedule(5, ddim_discretize="quad")


@pytest.fixture(scope="module")
def L():
    _lib.build()
    return _lib.lib()


def test_plms_step_argument_checks(L):
    """Checked before anything is launched, so these run without a GPU."""
    p = C.c_void_p(256)                                    # a 16-byte aligned dummy address
    odd = C.c_void_p(260)
    f = lambda *a, **k: L.aldm_plms_step(*a)
    args = lambda **o: [o.get("x", p), p, p, o.get("h1", p), o.get("h2", p), o.get("h3", p), o.get("order", 4),
                        o.get("et", p), o.get("xp", p), None, o.get("n", 1024), 0.5, 0.4, 0.7, 3.5, None]
    assert f(*args(x=None)) == -1
    assert f(*args(xp=None)) == -1
    assert f(*args(order=5)) == -1 and f(*args(order=-1)) == -1
    assert f(*args(order=2, h1=None)) == -1
    assert f(*args(order=3, h2=None)) == -1
    assert f(*args(order=4, h3=None)) == -1 and b"held3" in L.aldm_last_error()
    assert f(*args(order=_lib.PLMS_AVERAGE, h1=None, h2=None, h3=None, et=None)) == -1      # the average needs held1
    assert f(*args(order=_lib.PLMS_AVERAGE, h2=None, h3=None)) == -1                       # ... and stores nothing
    assert f(*args(n=1022)) == -2 and f(*args(n=0)) == -2
    assert f(*args(h2=odd)) == -3 and f(*args(et=odd)) == -3
    assert L.aldm_engine_plms_step(None, p, 1, p, p, p, p, 4, p, 0.5, 0.4, 0.7, 3.5, p, None, None) == -1
