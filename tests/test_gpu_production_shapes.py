"""Every GEMM and attention launch of the shipped plans, at its production shape, against the float64 references of
tests/test_gpu_kernel_matrix.py.

The hand-written matrix reaches every kernel variant at small shapes; the networks are checked end to end, where an
error confined to one tile, one image or one tile edge of one launch is diluted across the whole program.  Here the
plans the engine runs are built on the CPU with the seeded synthetic weights (the UNets of audioldm2-full,
audioldm_48k and audioldm2-full-large-1150k with the classifier-free-guidance halves batched and the context lengths of
bench.py; the VAE decoder, VAE encoder and vocoder of the first two; each at latent batch 8 and 1, which changes the
split-K and N-tile choices), and every distinct launch becomes a test case:

  * GEMM: deduplicated on every non-pointer field of the resolved aldm_gemm_desc, which pointers are set, and the kernel
    variant and A mode the selection reports for it (pointer alignment feeds that choice).  _spec translates the op into
    a GEMM_MATRIX spec (the input's channel count is not in the op: Cin = Cp); test_descriptors_match checks on the CPU
    that the spec plans to the same descriptor, variant and A mode, and test_production_gemm runs it through
    test_gemm_matrix: 0xFF workspace, guard bands, padding columns, split-K scratch guard, float64 reference in row chunks.
  * attention: deduplicated on (B, heads, Nq, Nk, mask, kv_bmod, ldq, ldk, ld_t, q_col, k_col) and run through
    test_attention_matrix with Q / K entries of sigma 1 and 6 (scores of ~50-100 across all 16 key tiles at Nk = 1024);
    masked cross-attention masks the keys after a per-batch length, as padded T5 / GPT-2 contexts are.
  * GroupNorm and LayerNorm at the largest production prep shapes, with the statistics' reference in float64 per image.

Every GPU case stays under MEM_LIMIT bytes of device memory (asserted)."""
import functools
from collections import OrderedDict

import pytest
import torch

from audioldm2_b200 import _lib, arch, plan, synth
from tests import test_gpu_kernel_matrix as KM
from tests.test_gpu_conv_halo import HALO_CASES

MODELS = ("audioldm2-full", "audioldm_48k", "audioldm2-full-large-1150k")
DECODER_MODELS = ("audioldm2-full", "audioldm_48k")
BATCHES = (8, 1)
T5_LEN = 32                  # bench.py's default context length
MEM_LIMIT = 16 << 30

_PTRS = ("a_hi", "a_lo", "w_packed", "w_plain", "bias", "rowvec", "res", "out", "out_hi", "out_lo", "out2_hi", "out2_lo", "ws")
_FIELDS = ("B", "H", "W", "Cp", "up", "bmod", "OH", "OW", "sy", "sx", "ntaps", "N", "K", "Kpad", "bn", "ldo", "ld_res",
           "ld_rowvec", "OHF", "OWF", "osy", "ooy", "act", "out_mode", "accumulate", "splitk", "impl", "n_split",
           "tok_per_batch", "ld_t", "alpha")


def desc_signature(d) -> tuple:
    """Every non-pointer field of an aldm_gemm_desc (the taps as far as ntaps) and which pointers are set."""
    return (tuple((f, getattr(d, f)) for f in _FIELDS) + (("taps", tuple((d.dy[t], d.dx[t]) for t in range(d.ntaps))),)
            + (("set", tuple(bool(getattr(d, p)) for p in _PTRS)),))


def _resolve(op: dict):
    arr = plan.Plan([op], None, 0, {}).resolve(1 << 32, 1 << 40)
    return arr[0].u.gemm


def _networks():
    """(model, network, latent batch, plan builder) of every shipped program but the token generator."""
    for m in MODELS:
        cfg = arch.model_config(m)
        n_ctx = len([c for c in cfg["unet"]["context_dim"] if c is not None])
        lens = (8, T5_LEN) if n_ctx > 1 else (T5_LEN,)           # model.build_synthetic
        _, T, Fq = cfg["latent"]
        ds = 2 ** (len(cfg["vae"]["ch_mult"]) - 1)
        for B in BATCHES:
            yield m, "unet", B, lambda cfg=cfg, B=B, lens=lens: plan.build_unet(
                _sd("unet", m, cfg), cfg["unet"], cfg["latent"], B, cfg_batched=True, ctx_max_len=lens)
            if m in DECODER_MODELS:
                yield m, "vae_dec", B, lambda cfg=cfg, B=B: plan.build_vae_decoder(_sd("vae", m, cfg), cfg["vae"], cfg["latent"], B)
                yield m, "vae_enc", B, lambda cfg=cfg, B=B, ds=ds: plan.build_vae_encoder(_sd("vae", m, cfg), cfg["vae"],
                                                                                            (T * ds, Fq * ds), B)
                yield m, "vocoder", B, lambda cfg=cfg, B=B, ds=ds: plan.build_vocoder(_sd("vocoder", m, cfg), cfg["vocoder"],
                                                                                        T * ds, B)


_SD = {}


def _sd(kind: str, model: str, cfg: dict):
    if (kind, model) not in _SD:
        _SD.clear()          # one model's weights at a time
        f = {"unet": synth.unet_state_dict, "vae": synth.vae_state_dict, "vocoder": synth.vocoder_state_dict}[kind]
        _SD[(kind, model)] = f(cfg[kind])
    return _SD[(kind, model)]


def _kind(op: dict) -> str:
    if op["out_mode"] == _lib.OUT_QKV:
        return "qkv" if op["N"] - op["n_split"] == op["n_split"] // 2 else "kv"
    k = f"t{op['ntaps']}" + ("_up" if op["up"] else "") + (f"_s{op['sy']}" if op["sy"] > 1 else "") \
        + (f"_ph{op['osy']}" if op["OHF"] != op["OH"] else "")
    k += {_lib.ACT_GEGLU: "_geglu", _lib.ACT_SILU: "_silu", _lib.ACT_TANH: "_tanh"}.get(op["act"], "")
    k += {_lib.OUT_PLANES: "_planes", _lib.OUT_NCHW: "_nchw"}.get(op["out_mode"], "")
    return k + ("_res" if op["res"] is not None else "") + ("_emb" if op["rowvec"] is not None else "") \
        + ("_acc" if op["accumulate"] else "")


@functools.lru_cache(maxsize=None)
def production():
    """(gemms, attns): OrderedDicts id -> record of the distinct launches, in plan order.  A GEMM record holds the op,
    its resolved signature, variant and A mode, and the column of its row vector inside the row."""
    gemms, attns, seen_g, seen_a = OrderedDict(), OrderedDict(), set(), set()
    _lib.build()
    for m, net, B, build in _networks():
        pl = build()
        ops = pl.ops
        del pl
        rv_base = {}
        for o in ops:
            if o["kind"] == "gemm" and o["rowvec"] is not None:
                rv_base[o["ld_rowvec"]] = min(rv_base.get(o["ld_rowvec"], 1 << 62), o["rowvec"].off)
        for o in ops:
            if o["kind"] == "gemm":
                d = _resolve(o)
                key = (desc_signature(d), _lib.gemm_variant(d), _lib.gemm_a_mode(d))
                if key in seen_g:
                    continue
                seen_g.add(key)
                col = (o["rowvec"].off - rv_base[o["ld_rowvec"]]) // 4 if o["rowvec"] is not None else None
                M = o["B"] * o["OH"] * o["OW"]
                name = f"{m}/{net}_b{B}/{_kind(o)}_{M}x{o['N']}x{o['K']}"
                while name in gemms:
                    name += "+"
                gemms[name] = dict(op=o, sig=key[0], variant=key[1], a_mode=key[2], rowvec_col=col)
            elif o["kind"] == "attn":
                key = tuple(o[f] for f in ("B", "heads", "Nq", "Nk")) + (o["mask"] is not None,) + \
                    tuple(o[f] for f in ("kv_bmod", "ldq", "ldk", "ld_t", "q_col", "k_col"))
                if key in seen_a:
                    continue
                seen_a.add(key)
                B_, h, Nq, Nk, masked = key[:5]
                kind = "self" if o["q_hi"] == o["k_hi"] else "cross"
                name = f"{kind}_b{B_}_h{h}_nq{Nq}_nk{Nk}" + ("_mask" if masked else "")
                while name in attns:
                    name += "+"
                attns[name] = dict(op=o, key=key, model=m)
    return gemms, attns


def _spec(rec: dict) -> dict:
    """The GEMM_MATRIX spec of a production GEMM op (ValueError for an op the matrix cannot express)."""
    o = rec["op"]
    geglu = o["act"] == _lib.ACT_GEGLU
    n_out = o["N"] // 2 if geglu else o["N"]
    if o["OWF"] != o["OW"]:
        raise ValueError(f"OWF {o['OWF']} != OW {o['OW']}")
    s = dict(B=o["B"], H=o["H"], W=o["W"], Cin=o["Cp"], N=o["N"], taps=tuple(o["taps"]), OH=o["OH"], OW=o["OW"],
             sy=o["sy"], sx=o["sx"], up=o["up"], bmod=o["bmod"], act=o["act"], alpha=o["alpha"],
             accumulate=bool(o["accumulate"]), a_planes=1 if o["a_lo"] is None else 2, bias=o["bias"] is not None,
             bn=o["bn"], splitk=o["splitk"], static_b=bool(o["impl"] & _lib.GEMM_STATIC_B))
    if (o["OHF"], o["osy"], o["ooy"]) != (o["OH"], 1, 0):
        s["ophase"] = (o["OHF"], o["osy"], o["ooy"])
    if o["res"] is not None:
        s.update(res=True, res_pad=o["ld_res"] - n_out)
    if o["rowvec"] is not None:
        s.update(rowvec=True, ld_rowvec=o["ld_rowvec"], rowvec_col=rec["rowvec_col"])
    if o["out_mode"] == _lib.OUT_QKV:
        tpb = o["tok_per_batch"]
        if o["B"] != 1 or o["H"] % tpb or o["W"] != 1:
            raise ValueError("QKV op over more than one image row")
        s.update(qkv=(None, o["H"] // tpb), n_split=o["n_split"], H=tpb, B=1, planes_out=1 if o["out_lo"] is None else 2)
    elif o["out_mode"] == _lib.OUT_PLANES:
        s.update(out="planes", planes_out=1 if o["out_lo"] is None else 2, pad_cols=o["ldo"] - n_out)
    elif o["out_mode"] == _lib.OUT_NCHW:
        if o["ldo"] != n_out:
            raise ValueError(f"NCHW output with ldo {o['ldo']} != {n_out}")
        s["out"] = "nchw"
    else:
        s["pad_cols"] = o["ldo"] - n_out
        if o["out_hi"] is not None:
            s["dual"] = 1 if o["out_lo"] is None else 2
    return s


def _gemm_ids():
    return list(production()[0])


def _attn_ids():
    return list(production()[1])


# ----------------------------------------------------------------------------------------------
# CPU: enumeration, translation, reach
# ----------------------------------------------------------------------------------------------
def test_enumeration():
    gemms, attns = production()
    assert len(gemms) > 150 and len(attns) >= 10, (len(gemms), len(attns))
    nets = {name.split("/")[1].split("_b")[0] for name in gemms}
    assert nets == {"unet", "vae_dec", "vae_enc", "vocoder"}, nets
    rows = max(r["op"]["B"] * r["op"]["OH"] * r["op"]["OW"] for r in gemms.values())
    assert rows >= 3_932_288, rows                # the 48k vocoder at batch 8
    assert max(r["op"]["K"] for r in gemms.values()) >= 11520
    assert max(a["op"]["Nk"] for a in attns.values()) == 1024


@pytest.mark.parametrize("name", _gemm_ids())
def test_descriptors_match(name):
    """The translated case plans to the production descriptor on every non-pointer field, with the same pointers set,
    and the selection gives it the same kernel variant and A mode."""
    rec = production()[0][name]
    d = KM._gemm_desc(KM.plan_gemm(name, plan.H100_SMS, _spec(rec)))
    want, got = dict(rec["sig"]), dict(desc_signature(d))
    diff = {k: (got[k], want[k]) for k in want if got[k] != want[k]}
    assert not diff, f"{name}: (case, production) differ in {diff}"
    assert _lib.gemm_variant(d) == rec["variant"], (_lib.gemm_variant(d), rec["variant"])
    assert _lib.gemm_a_mode(d) == rec["a_mode"]


def _pairs(specs: dict) -> dict:
    """(variant, A mode) -> the first case reaching it."""
    out = {}
    for name, spec in specs.items():
        d = KM._gemm_desc(KM.plan_gemm(name, plan.H100_SMS, spec))
        if spec.get("splitk", 1) > 1:
            d.splitk = spec["splitk"]
        out.setdefault((_lib.gemm_variant(d), _lib.gemm_a_mode(d)), name)
    return out


def _reachable_pairs() -> set:
    """Every (variant, A mode) the selection can return: the gather with every variant, and the halo path (64-wide N
    tiles, no GEGLU, no split-K) with each epilogue body and store it can take."""
    out = {(v, _lib.AMODE_GATHER) for v in KM._reachable_variants()}
    for ap in (1, 2):
        out |= {((64, epi, ap, _lib.RED_NONE, st), _lib.AMODE_HALO)
                for epi, st in ((_lib.EPI_FAST, _lib.STORE_ROW), (_lib.EPI_F32N, _lib.STORE_COMPACT),
                                (_lib.EPI_PLN, _lib.STORE_COMPACT), (_lib.EPI_PLN, _lib.STORE_PAIR_PLN),
                                (_lib.EPI_GENERIC, _lib.STORE_ROW))}
    return out


def test_every_variant_and_a_mode_has_a_case():
    """Hand-written cases (the matrix and the halo cases) reach every (variant, A mode) pair the selection can return,
    and every pair the production plans use."""
    _lib.build()
    hand = _pairs(dict(KM.GEMM_MATRIX, **HALO_CASES))
    missing = _reachable_pairs() - set(hand)
    assert not missing, f"(variant, A mode) pairs no hand-written case reaches: {sorted(missing)}"
    assert set(hand) <= _reachable_pairs(), sorted(set(hand) - _reachable_pairs())
    used = {(r["variant"], r["a_mode"]): name for name, r in production()[0].items()}
    unreached = {k: v for k, v in used.items() if k not in hand}
    assert not unreached, f"production pairs without a hand-written case: {unreached}"


# ----------------------------------------------------------------------------------------------
# GPU: production GEMMs
# ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", _gemm_ids())
def test_production_gemm(name, monkeypatch):
    rec = production()[0][name]
    monkeypatch.setitem(KM.GEMM_MATRIX, name, _spec(rec))
    c = KM.plan_gemm(name, KM._n_sm())
    d = KM._gemm_desc(c)
    assert (_lib.gemm_variant(d), _lib.gemm_a_mode(d)) == (rec["variant"], rec["a_mode"])
    del c
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    KM.test_gemm_matrix(name)
    peak = torch.cuda.max_memory_allocated()
    print(f"{name}: peak device memory {peak / 2 ** 30:.2f} GiB")
    assert peak < MEM_LIMIT, f"{name}: {peak / 2 ** 30:.2f} GiB of device memory"


# ----------------------------------------------------------------------------------------------
# GPU: production attention
# ----------------------------------------------------------------------------------------------
def _attn_cases() -> dict:
    """test_attention_matrix cases of the production attention launches: self-attention at sigma 1 and 6, masked
    cross-attention with a tail mask (keys after a per-batch length masked)."""
    out = {}
    for name, a in production()[1].items():
        B, heads, Nq, Nk, masked, kv_bmod = a["key"][:6]
        for sigma in (1.0, 6.0):
            out[f"{name}_s{int(sigma)}"] = (B, heads, Nq, Nk, "tail" if masked else None, kv_bmod, sigma)
    return out


def test_attention_cases_match_production():
    """Each case plans the production layout: ldq, ldk, ld_t, q_col and k_col as the plan's op."""
    for name, a in production()[1].items():
        o = a["op"]
        Cc = o["heads"] * 32
        assert o["ldo"] == Cc and o["scale"] == pytest.approx(32 ** -0.5), name
        if name.startswith("self"):
            assert (o["ldq"], o["ldk"], o["q_col"], o["k_col"], o["ld_t"]) == (2 * Cc, 2 * Cc, 0, Cc, plan.round_up(o["Nk"], 8))
        else:
            assert (o["ldq"], o["ldk"], o["q_col"], o["k_col"], o["ld_t"]) == (Cc, Cc, 0, 0, plan.round_up(o["Nk"], 8))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_attn_cases()))
def test_production_attention(name, monkeypatch):
    case = _attn_cases()[name]
    monkeypatch.setitem(KM.ATTN_CASES, name, case)
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    KM.test_attention_matrix(name, monkeypatch)
    assert torch.cuda.max_memory_allocated() < MEM_LIMIT


# ----------------------------------------------------------------------------------------------
# GPU: production GroupNorm / LayerNorm sizes
# ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("B,HW,C,c1", [(8, 262144, 256, 0), (8, 65536, 512, 0), (16, 4096, 384, 128)])
def test_production_groupnorm(B, HW, C, c1):
    """The largest GroupNorm preps at latent batch 8: the 48k VAE decoder's 2,097,152 x 256 and 524,288 x 512, and the
    UNet's concat of 256 + 128 channels over 16 images of 4,096 pixels; test_groupnorm_offset's inputs and bounds, with
    the float64 statistics computed image by image."""
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    KM.test_groupnorm_offset(B, HW, C, c1, 30)
    assert torch.cuda.max_memory_allocated() < MEM_LIMIT


@pytest.mark.gpu
def test_production_layernorm():
    """The largest LayerNorm of the UNets at latent batch 8: 16,384 tokens of 256 channels."""
    from tests.test_gpu_kernel_conformance import test_layernorm
    test_layernorm(16384, 256)
