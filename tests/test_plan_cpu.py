"""CPU checks of the host side: planner + weight packing, executed by the op-table emulator and
compared with the reference-module fixtures (tests/golden).  These validate everything the GPU
will be told to do -- graph wiring, K ordering, GEGLU row permutation, polyphase transposed
convolutions, buffer reuse -- without a GPU.  Tolerance: the emulator keeps operands as fp16 planes like the
kernels do -- hi + lo (2^-22) for weights and convolution inputs, a single plane (2^-12) for the
token-side activations of the UNet -- so first-stage networks agree with the fp32 reference to ~1e-6
(bound 2e-4) and a UNet evaluation to a few 1e-4 (bound UNET_TOL)."""
import pytest
import torch

from audioldm2_b200 import _lib, arch, packing, plan, synth
from tests.conftest import rel_l2
from tests.emulator import Emulator
from tests.golden import cases

TOL = 2e-4
UNET_TOL = 3e-3          # 32-channel toy topologies with single-plane token operands: measured 0.5-1.5e-3 per evaluation
                         # (full size: 4e-4, tests/test_gpu_nets.py; the end-to-end budget is 1e-3 on the waveform)


def test_pack_roundtrip_and_swizzle():
    g = torch.Generator().manual_seed(0)
    for (N, K, bn) in [(128, 64, 128), (96, 200, 32), (1, 72, 32), (64, 130, 64)]:
        w = torch.randn(N, K, generator=g)
        packed, plain, Npad, Kpad = packing.pack_tiles(w, bn)
        assert packed.numel() == Npad * Kpad * 4
        back = packing.unpack_tiles(packed, N, K, bn)
        assert rel_l2(back, w) < 1e-6
        # address formula used by the kernels: row r, logical chunk j -> r*128 + ((j ^ (r&7))<<4)
        hi = packed.view(torch.float16).reshape(Npad // bn, Kpad // 64, 2, bn * 64)[0, 0, 0]
        r, j = min(5, N - 1), 3
        off = (r * 128 + ((j ^ (r & 7)) << 4)) // 2
        want = plain[r, j * 8:(j + 1) * 8].to(torch.float16)
        assert torch.equal(hi[off:off + 8], want)


def test_geglu_row_order():
    o = packing.geglu_row_order(256, 128)
    assert o.shape[0] == 512 and sorted(o.tolist()) == list(range(512))
    assert o[:64].tolist() == list(range(64)) and o[64:128].tolist() == list(range(256, 320))


def test_conv_transpose_phases_match_torch():
    g = torch.Generator().manual_seed(1)
    for (u, k) in [(5, 16), (4, 16), (2, 8), (2, 4), (6, 12), (5, 10)]:
        cin, cout, L = 8, 6, 11
        w = torch.randn(cin, cout, k, generator=g)
        x = torch.randn(1, cin, L, generator=g)
        ref = torch.nn.functional.conv_transpose1d(x, w, stride=u, padding=(k - u) // 2)[0]   # [cout, Lout]
        Lout = ref.shape[1]
        out = torch.zeros(cout, Lout)
        for ph in packing.conv_transpose_phases(w, u):
            wm = ph["weight"].reshape(cout, len(ph["taps"]), ph["cp"])[:, :, :cin]
            for q in range((Lout - ph["r"] + u - 1) // u):
                for mi, d in enumerate(ph["taps"]):
                    i = q + d
                    if 0 <= i < L:
                        out[:, q * u + ph["r"]] += wm[:, mi] @ x[0, :, i]
        assert rel_l2(out, ref) < 1e-5


def _run_unet(cfg, B, t5_len, fixture, film=False):
    film = film or cfg["unet"].get("extra_film_condition_dim") is not None
    sd = synth.unet_state_dict(cfg["unet"])
    x, t, cond, unc = cases.unet_inputs(cfg, B, t5_len=t5_len)
    lens = tuple(c.shape[1] for c in cond["context_list"]) or (8,)
    pl = plan.build_unet(sd, cfg["unet"], cfg["latent"], B, ctx_max_len=lens, keep_plain=True)   # impl=tc: split-K on
    assert any(o["kind"] == "gemm" and o["splitk"] > 1 for o in pl.ops)
    em = Emulator(pl)
    em.write_io("x", x)
    em.write_io("t", torch.cat([t, t]))
    for s in range(len(cond["context_list"])):
        cu, cc = unc["context_list"][s], cond["context_list"][s]
        L = lens[s]
        ctx = torch.zeros(2 * B, L, cc.shape[2]); msk = torch.zeros(2 * B, L)
        ctx[:B, :cu.shape[1]] = cu; msk[:B, :cu.shape[1]] = unc["mask_list"][s]
        ctx[B:, :cc.shape[1]] = cc; msk[B:, :cc.shape[1]] = cond["mask_list"][s]
        em.write_io(f"ctx{s}", ctx); em.write_io(f"mask{s}", msk)
    if film:
        em.write_io("y", torch.cat([unc["y"], cond["y"]]))
    em.run(pl.marks["cond_begin"], pl.marks["cond_end"])
    em.run(pl.marks["step_begin"], pl.marks["step_end"])
    eps = em.read_io("eps")
    g = cases.load(fixture)
    eu, ec = rel_l2(eps[:B], g["eps_uncond"]), rel_l2(eps[B:], g["eps_cond"])
    print(f"{fixture}: eps rel L2 uncond {eu:.2e} cond {ec:.2e}")
    assert eu < UNET_TOL and ec < UNET_TOL
    # second evaluation on the same workspace (buffer reuse must not depend on stale state)
    em.run(pl.marks["step_begin"], pl.marks["step_end"])
    assert rel_l2(em.read_io("eps")[B:], g["eps_cond"]) < UNET_TOL


def test_unet_tiny_plan():
    _run_unet(arch.tiny_config(), 2, 5, "unet_tiny")


def test_unet_tiny_film_plan():
    _run_unet(arch.tiny_config(film=True), 2, 32, "unet_tiny_film", film=True)


def test_unet_tiny_large_plan():
    """audioldm2-full-large topology: 4 STs per site (last one self-attention), transformer_depth 2."""
    _run_unet(arch.tiny_config(variant="large"), 2, 5, "unet_tiny_large")


def test_tiny_48k_plans():
    """audioldm_48k topology: FiLM UNet on a 16-channel latent, 4-level VAE, HiFi-GAN with 4 MRF kernels (k=15)."""
    cfg = arch.tiny_config(variant="48k")
    _run_unet(cfg, 2, 32, "unet_tiny_48k")
    sd = synth.vae_state_dict(cfg["vae"])
    g = cases.load("vae_tiny_48k")
    pl = plan.build_vae_decoder(sd, cfg["vae"], cfg["latent"], 2, keep_plain=True)
    em = Emulator(pl); em.write_io("z", cases.latent(cfg, 2, seed=5)); em.run()
    assert rel_l2(em.read_io("mel"), g["mel"]) < TOL
    mel = cases.mel_input(cfg, 2)
    pl = plan.build_vae_encoder(sd, cfg["vae"], tuple(mel.shape[2:]), 2, keep_plain=True)
    em = Emulator(pl); em.write_io("mel", mel); em.run()
    assert rel_l2(em.read_io("moments").permute(0, 3, 1, 2), g["moments"]) < TOL
    gv = cases.load("vocoder_tiny_48k")
    pl = plan.build_vocoder(synth.vocoder_state_dict(cfg["vocoder"]), cfg["vocoder"], 16, 2, keep_plain=True)
    em = Emulator(pl); em.write_io("mel", cases.vocoder_input(cfg, 2, 16).permute(0, 2, 1).contiguous()); em.run()
    assert rel_l2(em.read_io("wave"), gv["wave"]) < TOL


def test_vae_tiny_plans():
    cfg = arch.tiny_config()
    sd = synth.vae_state_dict(cfg["vae"])
    g = cases.load("vae_tiny")
    pl = plan.build_vae_decoder(sd, cfg["vae"], cfg["latent"], 2, keep_plain=True)
    em = Emulator(pl)
    em.write_io("z", cases.latent(cfg, 2, seed=5))
    em.run()
    assert rel_l2(em.read_io("mel"), g["mel"]) < TOL
    mel = cases.mel_input(cfg, 2)
    pl = plan.build_vae_encoder(sd, cfg["vae"], tuple(mel.shape[2:]), 2, keep_plain=False)   # exercises unpack_tiles
    em = Emulator(pl)
    em.write_io("mel", mel)
    em.run()
    mom = em.read_io("moments").permute(0, 3, 1, 2)
    assert rel_l2(mom, g["moments"]) < TOL


def test_vocoder_tiny_plan():
    cfg = arch.tiny_config()
    sd = synth.vocoder_state_dict(cfg["vocoder"])
    g = cases.load("vocoder_tiny")
    pl = plan.build_vocoder(sd, cfg["vocoder"], 24, 2, keep_plain=True)
    em = Emulator(pl)
    em.write_io("mel", cases.vocoder_input(cfg, 2, 24).permute(0, 2, 1).contiguous())
    em.run()
    assert rel_l2(em.read_io("wave"), g["wave"]) < TOL


def test_pool_allocator_reuses_and_never_overlaps():
    p = plan.Pool()
    a = p.alloc(1000); b = p.alloc(5000); c = p.alloc(300)
    p.release(b)
    d = p.alloc(4000)
    assert d == b                      # first fit into the hole
    e = p.alloc(2000)                  # does not fit the remaining hole -> grows
    live = sorted((o, n) for o, n in p.live.items())
    for (o1, n1), (o2, n2) in zip(live, live[1:]):
        assert o1 + n1 <= o2
    assert p.peak >= e + 2000 and a == 0 and c > b


def test_half_width_tiles_rule():
    """Short-K GEMMs whose 128-wide tiles fill at most half the SMs get 64-wide tiles (plan.Planner.wmat); everything else keeps
    the widest tile (long K: split-K territory; GEGLU; more than half a wave; explicit tile width)."""
    import math
    P = plan.Planner()
    mk = lambda N, K: torch.zeros(N, K)
    assert P.wmat(mk(640, 640), None, 1, 640, m_rows=1024).bn == 64          # 40 tiles on 132 SMs, 10 k-blocks
    assert P.wmat(mk(640, 1280), None, 1, 1280, m_rows=1024).bn == 64
    assert P.wmat(mk(640, 5760), None, 9, 640, m_rows=1024).bn == 128        # long K: left to split-K
    assert P.wmat(mk(384, 384), None, 1, 384, m_rows=4096).bn == 128         # 96 tiles: halving would need a second wave
    assert P.wmat(mk(256, 256), None, 1, 256, m_rows=16384).bn == 128
    assert P.wmat(mk(5120, 640), torch.zeros(5120), 1, 640, geglu=True, m_rows=1024).bn == 128
    assert P.wmat(mk(640, 640), None, 1, 640, m_rows=1024, bn=128).bn == 128 # explicit width wins
    assert P.wmat(mk(640, 640), None, 1, 640).bn == 128                      # no row count: no rule


def test_groupnorm_scratch_outside_the_pool():
    """The GroupNorm scratch holds ticket counters that must stay zero between runs: it may not come from the pool's free list
    (holes there are rewritten by other ops on every run) -- finish() places it above the high-water mark."""
    P = plan.Planner()
    a = plan.F32(P.raw(4 * 64 * 128 * 4), 4 * 64, 128)
    hole = P.raw(1 << 22); P.free(hole)               # a hole large enough for the scratch
    g, b = P.vec(torch.ones(128)), P.vec(torch.zeros(128))
    P.prep(_lib.PREP_GN_SILU, a, None, g, b, eps=1e-5, B=4, HW=64)
    peak_before = P.pool.peak
    pl = P.finish({})
    scr = [o["scratch"] for o in pl.ops if o["kind"] == "prep"]
    assert scr and all(isinstance(r, plan.Ref) and r.region == "ws" and r.off >= peak_before for r in scr)
    assert pl.ws_bytes >= scr[0].off + 4 * (64 * 32 * 2 * 8 + 32 * 2 * 4 + 4)
