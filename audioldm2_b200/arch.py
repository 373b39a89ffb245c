"""Architecture specs for the three networks on the AudioLDM2 sampling hot path.

The specs are plain Python data derived from the same config keys the reference
uses (``unet_config.params``, ``first_stage_config.params.ddconfig`` and the
HiFi-GAN config dict), so the planner, the weight packer and the oracle all walk
one description of the module tree.  Parameter names are the reference
``state_dict`` keys (SURVEY.md 8b), relative to the sub-module prefix:

* UNet     : ``model.diffusion_model.``      (openaimodel.py:446-885)
* VAE      : ``first_stage_model.``          (model.py:419-686, autoencoder.py:103-117)
* vocoder  : ``first_stage_model.vocoder.``  (hifigan/models.py:112-174)
* AudioMAE token generator: ``cond_stage_models.<i>.`` (audiomae_gen/sequence_input.py:11-60, HF GPT2Model)

Nothing here touches torch; it is pure bookkeeping.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

# --------------------------------------------------------------------------------------
# model-name -> config (restated from audioldm2/utils.py:116-702; only hot-path keys)
# --------------------------------------------------------------------------------------

_UNET_BASE = dict(
    in_channels=8, out_channels=8, model_channels=128, attention_resolutions=[8, 4, 2],
    num_res_blocks=2, channel_mult=[1, 2, 3, 5], num_head_channels=32,
    transformer_depth=1, context_dim=[768, 1024], extra_film_condition_dim=None,
    extra_sa_layer=True,
)

_VAE_16K = dict(ch=128, ch_mult=[1, 2, 4], num_res_blocks=2, z_channels=8, in_channels=1,
                out_ch=1, embed_dim=8, double_z=True, mel_bins=64)
_VAE_48K = dict(ch=128, ch_mult=[1, 2, 4, 8], num_res_blocks=2, z_channels=16, in_channels=1,
                out_ch=1, embed_dim=16, double_z=True, mel_bins=256)

_VOC_16K = dict(upsample_rates=[5, 4, 2, 2, 2], upsample_kernel_sizes=[16, 16, 8, 4, 4],
                upsample_initial_channel=1024, resblock_kernel_sizes=[3, 7, 11],
                resblock_dilation_sizes=[[1, 3, 5]] * 3, num_mels=64,
                n_fft=1024, hop_size=160, win_size=1024, sampling_rate=16000, fmin=0, fmax=8000)
_VOC_48K = dict(upsample_rates=[6, 5, 4, 2, 2], upsample_kernel_sizes=[12, 10, 8, 4, 4],
                upsample_initial_channel=1536, resblock_kernel_sizes=[3, 7, 11, 15],
                resblock_dilation_sizes=[[1, 3, 5]] * 4, num_mels=256,
                n_fft=2048, hop_size=480, win_size=2048, sampling_rate=48000, fmin=20, fmax=24000)


def model_config(model_name: str = "audioldm2-full") -> dict:
    """Hot-path subset of ``default_audioldm_config`` (utils.py:116-192).

    Returns ``{"unet", "vae", "vocoder", "latent": (C, T, F), "sampling_rate",
    "latent_t_per_second", "linear_start", "linear_end", "timesteps"}``.
    """
    unet = dict(_UNET_BASE)
    vae, voc = dict(_VAE_16K), dict(_VOC_16K)
    latent = (8, 256, 16)
    sr, tps = 16000, 25.6
    if "-large-" in model_name:                      # utils.py:118-120
        unet["context_dim"] = [768, 1024, None]
        unet["transformer_depth"] = 2
    if "-speech-" in model_name:                     # utils.py:121-123
        unet["context_dim"] = [768]
    if "48k" in model_name:                          # utils.py:413-561
        unet.update(in_channels=16, out_channels=16, context_dim=[None],
                    extra_film_condition_dim=512)
        vae, voc = dict(_VAE_48K), dict(_VOC_48K)
        latent = (16, 128, 32)
        sr, tps = 48000, 12.8
    if "t5" in model_name:                           # utils.py:563-702
        unet["context_dim"] = [1024]
    return dict(name=model_name, unet=unet, vae=vae, vocoder=voc, latent=latent,
                sampling_rate=sr, latent_t_per_second=tps,
                linear_start=0.0015, linear_end=0.0195, timesteps=1000)


def tiny_config(film: bool = False, variant: str = "") -> dict:
    """Shrunken configs with the same topology as the real ones (fast parity tests).

    variant "" / film : audioldm2-full topology (3 STs per site) / audioldm_48k UNet topology (FiLM, 2 self-attn STs)
    variant "large"   : audioldm2-full-large topology: context_dim [.., .., None], transformer_depth 2 (utils.py:118-120)
    variant "48k"     : audioldm_48k first stage: 4-level VAE (ch_mult [1,2,4,8]), HiFi-GAN with 4 MRF kernels
                        (3,7,11,15) and the 48 k upsampling plan (6,5,4,2,2) (utils.py:475-493, utilities/model.py:39-75)
    """
    unet = dict(_UNET_BASE)
    unet.update(model_channels=32, context_dim=[48, 64])
    if film:
        unet.update(context_dim=[None], extra_film_condition_dim=24)
    if variant == "large":
        unet.update(context_dim=[48, 64, None], transformer_depth=2)
    vae = dict(ch=32, ch_mult=[1, 2, 4], num_res_blocks=1, z_channels=8, in_channels=1,
               out_ch=1, embed_dim=8, double_z=True, mel_bins=32)
    voc = dict(upsample_rates=[5, 4, 2, 2, 2], upsample_kernel_sizes=[16, 16, 8, 4, 4],
               upsample_initial_channel=128, resblock_kernel_sizes=[3, 7, 11],
               resblock_dilation_sizes=[[1, 3, 5]] * 3, num_mels=32,
               n_fft=256, hop_size=40, win_size=256, sampling_rate=4000, fmin=0, fmax=2000)
    latent = (8, 32, 8)
    if variant == "48k":
        unet.update(in_channels=16, out_channels=16, context_dim=[None], extra_film_condition_dim=24)
        vae = dict(ch=32, ch_mult=[1, 2, 4, 8], num_res_blocks=1, z_channels=16, in_channels=1,
                   out_ch=1, embed_dim=16, double_z=True, mel_bins=64)
        voc = dict(upsample_rates=[6, 5, 4, 2, 2], upsample_kernel_sizes=[12, 10, 8, 4, 4],
                   upsample_initial_channel=192, resblock_kernel_sizes=[3, 7, 11, 15],
                   resblock_dilation_sizes=[[1, 3, 5]] * 4, num_mels=64,
                   n_fft=256, hop_size=40, win_size=256, sampling_rate=4000, fmin=0, fmax=2000)
        latent = (16, 16, 8)
    name = "tiny" + ("-film" if film else "") + (("-" + variant) if variant else "")
    return dict(name=name, unet=unet, vae=vae, vocoder=voc,
                latent=latent, sampling_rate=4000, latent_t_per_second=25.6,
                linear_start=0.0015, linear_end=0.0195, timesteps=1000)


# --------------------------------------------------------------------------------------
# UNet spec (openaimodel.py:576-811)
# --------------------------------------------------------------------------------------

@dataclass
class Layer:
    kind: str                 # conv | res | st | down | up
    name: str                 # state_dict prefix relative to the net, e.g. "input_blocks.4.0"
    cin: int = 0
    cout: int = 0
    heads: int = 0
    ctx_dim: Optional[int] = None   # construction-time context_dim of the ST (None => self-attn weights)
    depth: int = 1
    ctx_slot: int = -1              # index into context_list used at run time, -1 => None (self-attention)


@dataclass
class UNetSpec:
    cfg: dict
    emb_ch: int               # width of `emb` fed to ResBlocks (time_embed_dim or 2x with FiLM)
    time_embed_dim: int
    input_blocks: List[List[Layer]] = field(default_factory=list)
    middle: List[Layer] = field(default_factory=list)
    output_blocks: List[List[Layer]] = field(default_factory=list)
    skip_ch: List[int] = field(default_factory=list)   # channels pushed by each input block


def _route_contexts(layers: List[Layer], n_ctx: int) -> None:
    """TimestepEmbedSequential.forward (openaimodel.py:81-103): the i-th SpatialTransformer
    of a block gets ([None] + context_list)[i], or None when out of range."""
    st_id = 0
    for l in layers:
        if l.kind == "st":
            l.ctx_slot = (st_id - 1) if (1 <= st_id <= n_ctx) else -1
            st_id += 1


def unet_spec(cfg: dict) -> UNetSpec:
    mc = cfg["model_channels"]
    ted = mc * 4
    film = cfg.get("extra_film_condition_dim") is not None
    emb_ch = ted * 2 if film else ted
    context_dim = cfg.get("context_dim")
    if context_dim is None:
        context_dim = [None]
    if not isinstance(context_dim, list):
        context_dim = [context_dim]
    # number of *run-time* contexts: entries of context_dim that are real cross-attn dims
    n_ctx = len([c for c in context_dim if c is not None])
    nhc = cfg["num_head_channels"]
    depth = cfg.get("transformer_depth", 1)
    extra_sa = cfg.get("extra_sa_layer", True)
    spec = UNetSpec(cfg=cfg, emb_ch=emb_ch, time_embed_dim=ted)

    def st_layers(prefix: str, start: int, ch: int) -> List[Layer]:
        out = []
        idx = start
        if extra_sa:
            out.append(Layer("st", f"{prefix}.{idx}", ch, ch, ch // nhc, None, depth)); idx += 1
        for cd in context_dim:
            out.append(Layer("st", f"{prefix}.{idx}", ch, ch, ch // nhc, cd, depth)); idx += 1
        return out

    spec.input_blocks.append([Layer("conv", "input_blocks.0.0", cfg["in_channels"], mc)])
    chans = [mc]
    ch, ds, bi = mc, 1, 1
    cm = cfg["channel_mult"]
    for level, mult in enumerate(cm):
        for _ in range(cfg["num_res_blocks"]):
            layers = [Layer("res", f"input_blocks.{bi}.0", ch, mult * mc)]
            ch = mult * mc
            if ds in cfg["attention_resolutions"]:
                layers += st_layers(f"input_blocks.{bi}", 1, ch)
            spec.input_blocks.append(layers); chans.append(ch); bi += 1
        if level != len(cm) - 1:
            spec.input_blocks.append([Layer("down", f"input_blocks.{bi}.0", ch, ch)])
            chans.append(ch); bi += 1; ds *= 2
    spec.skip_ch = list(chans)

    mid = [Layer("res", "middle_block.0", ch, ch)]
    mid += st_layers("middle_block", 1, ch)
    mid.append(Layer("res", f"middle_block.{len(mid)}", ch, ch))
    spec.middle = mid

    bo = 0
    for level, mult in list(enumerate(cm))[::-1]:
        for i in range(cfg["num_res_blocks"] + 1):
            ich = chans.pop()
            layers = [Layer("res", f"output_blocks.{bo}.0", ch + ich, mc * mult)]
            ch = mc * mult
            if ds in cfg["attention_resolutions"]:
                layers += st_layers(f"output_blocks.{bo}", 1, ch)
            if level and i == cfg["num_res_blocks"]:
                layers.append(Layer("up", f"output_blocks.{bo}.{len(layers)}", ch, ch))
                ds //= 2
            spec.output_blocks.append(layers); bo += 1

    for blk in spec.input_blocks + [spec.middle] + spec.output_blocks:
        _route_contexts(blk, n_ctx)
    return spec


def unet_param_shapes(cfg: dict) -> Dict[str, Tuple[int, ...]]:
    """name -> shape for every UNet parameter (the reference ``state_dict`` of UNetModel)."""
    s = unet_spec(cfg)
    mc, ted = cfg["model_channels"], s.time_embed_dim
    P: Dict[str, Tuple[int, ...]] = {}

    def lin(n, o, i, bias=True):
        P[n + ".weight"] = (o, i)
        if bias:
            P[n + ".bias"] = (o,)

    def conv(n, o, i, k):
        P[n + ".weight"] = (o, i, k, k); P[n + ".bias"] = (o,)

    def norm(n, c):
        P[n + ".weight"] = (c,); P[n + ".bias"] = (c,)

    lin("time_embed.0", ted, mc); lin("time_embed.2", ted, ted)
    if cfg.get("extra_film_condition_dim") is not None:
        lin("film_emb", ted, cfg["extra_film_condition_dim"])

    def add(l: Layer):
        n = l.name
        if l.kind == "conv":
            conv(n, l.cout, l.cin, 3)
        elif l.kind == "res":
            norm(n + ".in_layers.0", l.cin); conv(n + ".in_layers.2", l.cout, l.cin, 3)
            lin(n + ".emb_layers.1", l.cout, s.emb_ch)
            norm(n + ".out_layers.0", l.cout); conv(n + ".out_layers.3", l.cout, l.cout, 3)
            if l.cin != l.cout:
                conv(n + ".skip_connection", l.cout, l.cin, 1)
        elif l.kind == "down":
            conv(n + ".op", l.cout, l.cin, 3)
        elif l.kind == "up":
            conv(n + ".conv", l.cout, l.cin, 3)
        elif l.kind == "st":
            c = l.cin
            norm(n + ".norm", c); conv(n + ".proj_in", c, c, 1); conv(n + ".proj_out", c, c, 1)
            for d in range(l.depth):
                b = f"{n}.transformer_blocks.{d}"
                for a, cd in (("attn1", None), ("attn2", l.ctx_dim)):
                    kd = c if cd is None else cd
                    lin(f"{b}.{a}.to_q", c, c, bias=False)
                    lin(f"{b}.{a}.to_k", c, kd, bias=False)
                    lin(f"{b}.{a}.to_v", c, kd, bias=False)
                    lin(f"{b}.{a}.to_out.0", c, c)
                lin(f"{b}.ff.net.0.proj", 8 * c, c); lin(f"{b}.ff.net.2", c, 4 * c)
                for k in ("norm1", "norm2", "norm3"):
                    norm(f"{b}.{k}", c)

    for blk in s.input_blocks + [s.middle] + s.output_blocks:
        for l in blk:
            add(l)
    norm("out.0", mc); conv("out.2", cfg["out_channels"], mc, 3)
    return P


# --------------------------------------------------------------------------------------
# VAE spec (model.py:419-686) -- Decoder and Encoder, attn_resolutions == []
# --------------------------------------------------------------------------------------

def vae_param_shapes(cfg: dict, encoder: bool = True, decoder: bool = True) -> Dict[str, Tuple[int, ...]]:
    P: Dict[str, Tuple[int, ...]] = {}
    ch, cm, nrb = cfg["ch"], cfg["ch_mult"], cfg["num_res_blocks"]
    zc, ed = cfg["z_channels"], cfg["embed_dim"]

    def conv(n, o, i, k):
        P[n + ".weight"] = (o, i, k, k); P[n + ".bias"] = (o,)

    def norm(n, c):
        P[n + ".weight"] = (c,); P[n + ".bias"] = (c,)

    def res(n, i, o):
        norm(n + ".norm1", i); conv(n + ".conv1", o, i, 3)
        norm(n + ".norm2", o); conv(n + ".conv2", o, o, 3)
        if i != o:
            conv(n + ".nin_shortcut", o, i, 1)

    def attn(n, c):
        norm(n + ".norm", c)
        for k in ("q", "k", "v", "proj_out"):
            conv(f"{n}.{k}", c, c, 1)

    if decoder:
        bi = ch * cm[-1]
        conv("decoder.conv_in", bi, zc, 3)
        res("decoder.mid.block_1", bi, bi); attn("decoder.mid.attn_1", bi); res("decoder.mid.block_2", bi, bi)
        for lvl in reversed(range(len(cm))):
            bo = ch * cm[lvl]
            for ib in range(nrb + 1):
                res(f"decoder.up.{lvl}.block.{ib}", bi, bo); bi = bo
            if lvl != 0:
                conv(f"decoder.up.{lvl}.upsample.conv", bi, bi, 3)
        norm("decoder.norm_out", bi); conv("decoder.conv_out", cfg["out_ch"], bi, 3)
        conv("post_quant_conv", zc, ed, 1)
    if encoder:
        conv("encoder.conv_in", ch, cfg["in_channels"], 3)
        in_mult = (1,) + tuple(cm)
        bi = ch
        for lvl in range(len(cm)):
            bi = ch * in_mult[lvl]; bo = ch * cm[lvl]
            for ib in range(nrb):
                res(f"encoder.down.{lvl}.block.{ib}", bi, bo); bi = bo
            if lvl != len(cm) - 1:
                conv(f"encoder.down.{lvl}.downsample.conv", bi, bi, 3)
        res("encoder.mid.block_1", bi, bi); attn("encoder.mid.attn_1", bi); res("encoder.mid.block_2", bi, bi)
        norm("encoder.norm_out", bi)
        conv("encoder.conv_out", 2 * zc if cfg.get("double_z", True) else zc, bi, 3)
        conv("quant_conv", 2 * ed, 2 * zc, 1)
    return P


# --------------------------------------------------------------------------------------
# HiFi-GAN spec (hifigan/models.py:112-147); weight-norm already folded (utilities/model.py:139)
# --------------------------------------------------------------------------------------

def vocoder_param_shapes(cfg: dict) -> Dict[str, Tuple[int, ...]]:
    P: Dict[str, Tuple[int, ...]] = {}
    c0 = cfg["upsample_initial_channel"]
    P["conv_pre.weight"] = (c0, cfg["num_mels"], 7); P["conv_pre.bias"] = (c0,)
    nk = len(cfg["resblock_kernel_sizes"])
    ch = c0
    for i, (u, k) in enumerate(zip(cfg["upsample_rates"], cfg["upsample_kernel_sizes"])):
        cin, ch = c0 // (2 ** i), c0 // (2 ** (i + 1))
        P[f"ups.{i}.weight"] = (cin, ch, k); P[f"ups.{i}.bias"] = (ch,)   # ConvTranspose1d: [Cin,Cout,k]
        for j, ks in enumerate(cfg["resblock_kernel_sizes"]):
            for m in range(3):
                for cs in ("convs1", "convs2"):
                    P[f"resblocks.{i * nk + j}.{cs}.{m}.weight"] = (ch, ch, ks)
                    P[f"resblocks.{i * nk + j}.{cs}.{m}.bias"] = (ch,)
    P["conv_post.weight"] = (1, ch, 7); P["conv_post.bias"] = (1,)
    return P


def vocoder_out_len(cfg: dict, n_frames: int) -> int:
    L = n_frames
    for u, k in zip(cfg["upsample_rates"], cfg["upsample_kernel_sizes"]):
        L = (L - 1) * u - 2 * ((k - u) // 2) + k
    return L


# --------------------------------------------------------------------------------------
# AudioMAE token generator (SequenceGenAudioMAECond / Sequence2AudioMAE, audiomae_gen/sequence_input.py:11-60):
# GPT-2 small (GPT2Config() defaults: 12 layers, 12 heads, width 768, 1024 positions, gelu_new, LayerNorm eps 1e-5),
# input projections CLAP 512 -> 768 and Flan-T5 1024 -> 768, SOS / EOS embeddings nn.Embedding(32, 768).
# --------------------------------------------------------------------------------------

SEQGEN = dict(n_embd=768, n_head=12, n_positions=1024, vocab=50257, n_inner=3072, ln_eps=1e-5,
              input_dims=(512, 1024), gen_len=8)          # sequence_input_embed_dim / sequence_gen_length (utils.py:362-368)


def seqgen_param_shapes(n_layer: int = 12, with_wte: bool = True) -> Dict[str, Tuple[int, ...]]:
    """name -> shape relative to ``cond_stage_models.<i>.``.  ``model.*`` are HF GPT-2 keys; its linear layers are
    ``Conv1D`` with weights [in, out] (y = x W + b).  ``model.wte.weight`` is never read (inputs_embeds)."""
    C, F = SEQGEN["n_embd"], SEQGEN["n_inner"]
    P: Dict[str, Tuple[int, ...]] = {"model.wpe.weight": (SEQGEN["n_positions"], C)}
    if with_wte:
        P["model.wte.weight"] = (SEQGEN["vocab"], C)
    for i in range(n_layer):
        h = f"model.h.{i}"
        for ln in ("ln_1", "ln_2"):
            P[f"{h}.{ln}.weight"] = (C,); P[f"{h}.{ln}.bias"] = (C,)
        for n, (k, o) in (("attn.c_attn", (C, 3 * C)), ("attn.c_proj", (C, C)), ("mlp.c_fc", (C, F)), ("mlp.c_proj", (F, C))):
            P[f"{h}.{n}.weight"] = (k, o); P[f"{h}.{n}.bias"] = (o,)
    P["model.ln_f.weight"] = (C,); P["model.ln_f.bias"] = (C,)
    P["start_of_sequence_tokens.weight"] = (32, C)
    P["end_of_sequence_tokens.weight"] = (32, C)
    for j, d in enumerate(SEQGEN["input_dims"]):
        P[f"input_sequence_embed_linear.{j}.weight"] = (C, d); P[f"input_sequence_embed_linear.{j}.bias"] = (C,)
    return P


def has_seqgen(cfg: dict) -> bool:
    """Configs whose UNet reads ``crossattn_audiomae_generated`` (context 0 of width 768 next to a Flan-T5 context):
    audioldm2-full and audioldm2-full-large.  audioldm_48k (FiLM only), the *_t5 models (T5 only) and the speech models
    (phoneme-conditioned 512-token generation, not built here) have no such stage."""
    dims = [c for c in (cfg["unet"].get("context_dim") or []) if c is not None]
    return dims[:2] == [768, 1024] and "-speech-" not in cfg.get("name", "")


# --------------------------------------------------------------------------------------
# Flan-T5-large text encoder (FlanT5HiddenState, encoders/modules.py:113-198: T5EncoderModel(T5Config.from_pretrained(
# "google/flan-t5-large")), run in fp32): 24 blocks, width 1024, 16 heads of 64, gated-GELU feed-forward of 2816 with
# gelu_new, RMSNorm eps 1e-6, 32 bidirectional relative-position buckets up to distance 128 (layer 0's table, shared by
# every layer), no biases, unscaled embedding.  The tokenizer (max_length 128, pad id 0, "" -> [1]) stays on the host.
# --------------------------------------------------------------------------------------

T5 = dict(d_model=1024, n_head=16, d_kv=64, d_ff=2816, n_layer=24, vocab=32128, eps=1e-6, num_buckets=32,
          max_distance=128, max_len=128, pad_id=0, eos_id=1)


def t5_param_shapes(n_layer: int = 24, with_embed_tokens: bool = True) -> Dict[str, Tuple[int, ...]]:
    """name -> shape of HF ``T5EncoderModel``'s state dict (relative to ``cond_stage_models.<i>.model.``).
    ``encoder.embed_tokens.weight`` is tied to ``shared.weight``."""
    C, F, H, V = T5["d_model"], T5["d_ff"], T5["n_head"], T5["vocab"]
    P: Dict[str, Tuple[int, ...]] = {"shared.weight": (V, C)}
    if with_embed_tokens:
        P["encoder.embed_tokens.weight"] = (V, C)
    for i in range(n_layer):
        b = f"encoder.block.{i}.layer"
        for n in ("q", "k", "v", "o"):
            P[f"{b}.0.SelfAttention.{n}.weight"] = (C, C)
        if i == 0:
            P[f"{b}.0.SelfAttention.relative_attention_bias.weight"] = (T5["num_buckets"], H)
        P[f"{b}.0.layer_norm.weight"] = (C,)
        P[f"{b}.1.DenseReluDense.wi_0.weight"] = (F, C)
        P[f"{b}.1.DenseReluDense.wi_1.weight"] = (F, C)
        P[f"{b}.1.DenseReluDense.wo.weight"] = (C, F)
        P[f"{b}.1.layer_norm.weight"] = (C,)
    P["encoder.final_layer_norm.weight"] = (C,)
    return P


def has_t5(cfg: dict) -> bool:
    """Configs whose UNet reads Flan-T5 states (a 1024-wide context): audioldm2-full / -large (next to the AudioMAE
    tokens) and the *_t5 models."""
    return 1024 in [c for c in (cfg["unet"].get("context_dim") or []) if c is not None]


# --------------------------------------------------------------------------------------
# CLAP text branch (CLAPAudioEmbeddingClassifierFreev2 with embed_mode "text", encoders/modules.py:546-745, and
# CLAP.get_text_embedding, clap/open_clip/model.py:656-663, 730-750): HF RobertaModel(RobertaConfig("roberta-base")) --
# 12 post-LN blocks, width 768, 12 heads of 64, erf-GELU feed-forward of 3072, LayerNorm eps 1e-5, learned positions
# offset by the pad id -- then the tanh pooler on token 0, text_projection (Linear 768 -> 512, ReLU, Linear 512 -> 512)
# and F.normalize.  The tokenizer (RobertaTokenizer, padding="max_length", max_length 512; "" -> [0, 2]) stays on the host.
# --------------------------------------------------------------------------------------

CLAP_TEXT = dict(d_model=768, n_head=12, d_head=64, d_ff=3072, n_layer=12, vocab=50265, max_positions=514, type_vocab=1,
                 pad_id=1, bos_id=0, eos_id=2, eps=1e-5, joint_dim=512, max_len=512)


def clap_text_param_shapes(n_layer: int = 12) -> Dict[str, Tuple[int, ...]]:
    """name -> shape of the CLAP text branch's state dict (relative to the CLAP model, e.g. ``cond_stage_models.0.model.``):
    HF ``RobertaModel`` keys under ``text_branch.`` and ``text_projection.{0,2}``."""
    C, F, P = CLAP_TEXT["d_model"], CLAP_TEXT["d_ff"], CLAP_TEXT["joint_dim"]
    e = "text_branch.embeddings"
    S: Dict[str, Tuple[int, ...]] = {
        f"{e}.word_embeddings.weight": (CLAP_TEXT["vocab"], C),
        f"{e}.position_embeddings.weight": (CLAP_TEXT["max_positions"], C),
        f"{e}.token_type_embeddings.weight": (CLAP_TEXT["type_vocab"], C),
        f"{e}.LayerNorm.weight": (C,), f"{e}.LayerNorm.bias": (C,),
    }
    for i in range(n_layer):
        b = f"text_branch.encoder.layer.{i}"
        for n in ("query", "key", "value"):
            S[f"{b}.attention.self.{n}.weight"] = (C, C)
            S[f"{b}.attention.self.{n}.bias"] = (C,)
        S[f"{b}.attention.output.dense.weight"] = (C, C)
        S[f"{b}.attention.output.dense.bias"] = (C,)
        S[f"{b}.attention.output.LayerNorm.weight"] = (C,)
        S[f"{b}.attention.output.LayerNorm.bias"] = (C,)
        S[f"{b}.intermediate.dense.weight"] = (F, C)
        S[f"{b}.intermediate.dense.bias"] = (F,)
        S[f"{b}.output.dense.weight"] = (C, F)
        S[f"{b}.output.dense.bias"] = (C,)
        S[f"{b}.output.LayerNorm.weight"] = (C,)
        S[f"{b}.output.LayerNorm.bias"] = (C,)
    S["text_branch.pooler.dense.weight"] = (C, C)
    S["text_branch.pooler.dense.bias"] = (C,)
    S["text_projection.0.weight"] = (P, C)
    S["text_projection.0.bias"] = (P,)
    S["text_projection.2.weight"] = (P, P)
    S["text_projection.2.bias"] = (P,)
    return S


def has_clap(cfg: dict) -> bool:
    """Configs conditioned on the CLAP text embedding: audioldm2-full / -large (GPT-2's first input) and audioldm_48k (the
    FiLM vector, 512 wide).  The tiny FiLM test configs (dim 24) are not."""
    return has_seqgen(cfg) or cfg["unet"].get("extra_film_condition_dim") == CLAP_TEXT["joint_dim"]


# --------------------------------------------------------------------------------------
# CLAP audio branch (CLAPAudioEmbeddingClassifierFreev2 with embed_mode "audio", encoders/modules.py:689-716, and
# CLAP.get_audio_embedding, clap/open_clip/model.py:752-777): HTSAT-base (HTSAT_Swin_Transformer, clap/open_clip/htsat.py,
# config :1271-1284 and model_configs/HTSAT-base.json) without fusion -- torchlibrosa's Spectrogram (n_fft 1024, hop 480,
# periodic Hann, reflect-centred) and LogmelFilterBank (64 mel bins, 50 Hz - 14 kHz, 10 log10, ref 1, no top_db), bn0,
# reshape_wav2img to a 256 x 256 image, a 4 x 4 patch embedding to a 64 x 64 grid of 128 channels, four pre-LN Swin stages
# (depths 2, 2, 12, 2; heads 4, 8, 16, 32 of 32 dims; 8 x 8 windows, odd blocks shifted by 4 where the grid is larger than
# a window) joined by PatchMerging, the final LayerNorm(1024) and the mean over tokens -- then audio_projection (Linear
# 1024 -> 512, ReLU, Linear 512 -> 512) and F.normalize.  Input: 48 kHz audio, resampled from 16 kHz by torchaudio first,
# truncated to 480 000 samples.
# --------------------------------------------------------------------------------------

CLAP_AUDIO = dict(sample_rate=48000, n_fft=1024, hop=480, n_mels=64, fmin=50.0, fmax=14000.0, max_samples=480000,
                  spec_size=256, freq_ratio=4, frames=1024, patch=4, embed_dim=128, depths=(2, 2, 12, 2),
                  heads=(4, 8, 16, 32), head_dim=32, window=8, mlp_ratio=4, eps=1e-5, joint_dim=512, bn_eps=1e-5)


def clap_audio_param_shapes(depths=CLAP_AUDIO["depths"]) -> Dict[str, Tuple[int, ...]]:
    """name -> shape of the CLAP audio branch's parameters and the running statistics of bn0 (relative to the CLAP model,
    e.g. ``clap.model.``): ``audio_branch.`` (HTSAT_Swin_Transformer, torchlibrosa's extractors included) and
    ``audio_projection.{0,2}``.  The relative_position_index / attn_mask buffers, tscam_conv and head are not read."""
    A = CLAP_AUDIO
    nb, E, M = A["n_fft"] // 2 + 1, A["embed_dim"], A["n_mels"]
    a = "audio_branch"
    S: Dict[str, Tuple[int, ...]] = {
        f"{a}.spectrogram_extractor.stft.conv_real.weight": (nb, 1, A["n_fft"]),
        f"{a}.spectrogram_extractor.stft.conv_imag.weight": (nb, 1, A["n_fft"]),
        f"{a}.logmel_extractor.melW": (nb, M),
        f"{a}.bn0.weight": (M,), f"{a}.bn0.bias": (M,), f"{a}.bn0.running_mean": (M,), f"{a}.bn0.running_var": (M,),
        f"{a}.patch_embed.proj.weight": (E, 1, A["patch"], A["patch"]), f"{a}.patch_embed.proj.bias": (E,),
        f"{a}.patch_embed.norm.weight": (E,), f"{a}.patch_embed.norm.bias": (E,),
    }
    nrel = (2 * A["window"] - 1) ** 2
    for i, depth in enumerate(depths):
        C, H = E * 2 ** i, A["heads"][i]
        for j in range(depth):
            b = f"{a}.layers.{i}.blocks.{j}"
            S[f"{b}.norm1.weight"] = (C,); S[f"{b}.norm1.bias"] = (C,)
            S[f"{b}.attn.relative_position_bias_table"] = (nrel, H)
            S[f"{b}.attn.qkv.weight"] = (3 * C, C); S[f"{b}.attn.qkv.bias"] = (3 * C,)
            S[f"{b}.attn.proj.weight"] = (C, C); S[f"{b}.attn.proj.bias"] = (C,)
            S[f"{b}.norm2.weight"] = (C,); S[f"{b}.norm2.bias"] = (C,)
            S[f"{b}.mlp.fc1.weight"] = (A["mlp_ratio"] * C, C); S[f"{b}.mlp.fc1.bias"] = (A["mlp_ratio"] * C,)
            S[f"{b}.mlp.fc2.weight"] = (C, A["mlp_ratio"] * C); S[f"{b}.mlp.fc2.bias"] = (C,)
        if i < len(depths) - 1:
            d = f"{a}.layers.{i}.downsample"
            S[f"{d}.norm.weight"] = (4 * C,); S[f"{d}.norm.bias"] = (4 * C,)
            S[f"{d}.reduction.weight"] = (2 * C, 4 * C)
    F = E * 2 ** (len(depths) - 1)
    S[f"{a}.norm.weight"] = (F,); S[f"{a}.norm.bias"] = (F,)
    P = A["joint_dim"]
    S["audio_projection.0.weight"] = (P, F); S["audio_projection.0.bias"] = (P,)
    S["audio_projection.2.weight"] = (P, P); S["audio_projection.2.bias"] = (P,)
    return S


def clap_audio_frames(n_samples: int, sampling_rate: int) -> int:
    """Frames T of the spectrogram of an n-sample clip at ``sampling_rate`` (16 000 or 48 000): the 48 kHz length
    (3 n at 16 kHz, torchaudio's ceil(3 n / 1)) truncated to 480 000 samples, // 480 + 1."""
    L48 = min(n_samples * (48000 // sampling_rate), CLAP_AUDIO["max_samples"])
    return L48 // CLAP_AUDIO["hop"] + 1
