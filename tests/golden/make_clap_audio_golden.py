"""Generate tests/golden/clap_audio.pt by running the UNMODIFIED reference CLAP audio branch and re-ranker.

    ALDM_REFERENCE_ROOT=<checkout of the reference> python tests/golden/make_clap_audio_golden.py

The reference's own ``HTSAT_Swin_Transformer`` (clap/open_clip/htsat.py) is built with the HTSAT-base audio config (and
with depths (2, 2, 2, 2) for the small cases) and loaded from synth.clap_audio_state_dict; ``CLAP.encode_audio`` and
``CLAP.get_audio_embedding`` (clap/open_clip/model.py:614-617, 752-777) are bound to a CLAP stand-in holding it and
``audio_projection``.  ``CLAPAudioEmbeddingClassifierFreev2.forward`` and ``cos_similarity`` (encoders/modules.py:639-735)
run on a stub ``self`` holding that stand-in, with the real ``torchaudio.functional.resample`` and the real
``get_audio_features`` (clap/training/data.py:421-450); the text side is HF RobertaModel with 2 layers (as in
tests/golden/make_clap_golden.py) and its tokenizer synth.clap_tokenize.  In this script only:
  * torchlibrosa (not installed) is a stand-in with the same parameter names: Spectrogram (STFT as conv1d with
    conv_real / conv_imag over reflect-padded input, power re^2 + im^2), LogmelFilterBank (input @ melW, 10 log10(max(x,
    1e-10)) - 10 log10(max(1e-10, 1)), no top_db) and a no-op SpecAugmentation (training only);
  * the absent imports of data.py and open_clip/utils.py (pandas, PIL, torchvision, soundfile, the open_clip package
    __init__) are stubbed in sys.modules.
Stored: the embedding of every case of clap_audio_cases.CASES, the seeded cos_similarity call (similarity, chosen
indices, replaced rows, seed, CPU generator state after the call), the reference's relative_position_index and attn_mask
buffers, and the parameter names and shapes of the HTSAT-base branch.
"""
from __future__ import annotations

import importlib
import os
import sys
import types

os.environ["HF_HUB_OFFLINE"] = "1"
os.environ["TRANSFORMERS_OFFLINE"] = "1"

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import numpy as np                              # noqa: E402
import torch                                    # noqa: E402
import torch.nn as nn                           # noqa: E402
import torch.nn.functional as F                 # noqa: E402

from audioldm2_b200 import synth                # noqa: E402
from oracle import ref_loader                   # noqa: E402
from tests.golden import clap_audio_cases as CA  # noqa: E402


def _module(name: str, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


class _STFT(nn.Module):
    def __init__(self, n_fft, hop_length, center, pad_mode):
        super().__init__()
        self.n_fft, self.hop, self.center, self.pad_mode = n_fft, hop_length, center, pad_mode
        self.conv_real = nn.Conv1d(1, n_fft // 2 + 1, n_fft, stride=hop_length, bias=False)
        self.conv_imag = nn.Conv1d(1, n_fft // 2 + 1, n_fft, stride=hop_length, bias=False)

    def forward(self, x):
        x = x[:, None, :]
        if self.center:
            x = F.pad(x, (self.n_fft // 2, self.n_fft // 2), mode=self.pad_mode)
        return self.conv_real(x)[:, None].transpose(2, 3), self.conv_imag(x)[:, None].transpose(2, 3)


class Spectrogram(nn.Module):
    def __init__(self, n_fft=2048, hop_length=None, win_length=None, window="hann", center=True, pad_mode="reflect",
                 power=2.0, freeze_parameters=True):
        super().__init__()
        assert window == "hann" and power == 2.0
        self.stft = _STFT(n_fft, hop_length, center, pad_mode)

    def forward(self, x):
        re, im = self.stft(x)
        return re ** 2 + im ** 2


class LogmelFilterBank(nn.Module):
    def __init__(self, sr=22050, n_fft=2048, n_mels=64, fmin=0.0, fmax=None, is_log=True, ref=1.0, amin=1e-10,
                 top_db=80.0, freeze_parameters=True):
        super().__init__()
        assert is_log and top_db is None
        self.ref, self.amin = ref, amin
        self.melW = nn.Parameter(torch.zeros(n_fft // 2 + 1, n_mels))

    def forward(self, x):
        mel = torch.matmul(x, self.melW)
        return 10.0 * torch.log10(torch.clamp(mel, min=self.amin)) - 10.0 * np.log10(np.maximum(self.amin, self.ref))


class SpecAugmentation(nn.Module):
    def __init__(self, *a, **k):
        super().__init__()

    def forward(self, x):
        raise AssertionError("SpecAugmentation runs in training mode only")


def reference():
    """-> (HTSAT_Swin_Transformer, CLAP, CLAPAudioEmbeddingClassifierFreev2), from the reference's own files."""
    root = ref_loader.REF_ROOT
    if root not in sys.path:
        sys.path.insert(0, root)
    base = os.path.join(root, "audioldm2")
    for name, sub in (("audioldm2", ""), ("audioldm2.clap", "clap"), ("audioldm2.clap.open_clip", "clap/open_clip"),
                      ("audioldm2.clap.training", "clap/training"), ("audioldm2.latent_diffusion", "latent_diffusion"),
                      ("audioldm2.latent_diffusion.modules", "latent_diffusion/modules"),
                      ("audioldm2.latent_diffusion.modules.encoders", "latent_diffusion/modules/encoders")):
        ref_loader._stub_pkg(name, os.path.join(base, sub))
    import transformers
    for name in ("BertModel", "RobertaModel", "BartModel", "RobertaConfig"):     # loaded before any stub below
        getattr(transformers, name)
    _module("torchlibrosa")
    _module("torchlibrosa.stft", Spectrogram=Spectrogram, LogmelFilterBank=LogmelFilterBank)
    _module("torchlibrosa.augmentation", SpecAugmentation=SpecAugmentation)
    absent = dict(pandas={}, soundfile={}, tqdm=dict(tqdm=lambda x, *a, **k: x), torchvision={},
                  **{"torchvision.datasets": {}, "torchvision.ops": {}, "torchvision.ops.misc": dict(FrozenBatchNorm2d=nn.Module),
                     "PIL": {}, "PIL.Image": dict(Image=object)})
    for name, attrs in absent.items():
        try:
            importlib.import_module(name)
        except ImportError:
            _module(name, **attrs)
    oc = sys.modules["audioldm2.clap.open_clip"]
    oc.tokenize, oc.create_model = None, None
    htsat = importlib.import_module("audioldm2.clap.open_clip.htsat")
    _module("audioldm2.clap.open_clip.pann_model", create_pann_model=None)
    clap_model = importlib.import_module("audioldm2.clap.open_clip.model").CLAP
    importlib.import_module("audioldm2.clap.training.data")

    class _Unused(nn.Module):
        pass

    _module("audioldm2.latent_diffusion.modules.audiomae.AudioMAE", Vanilla_AudioMAE=_Unused)
    _module("audioldm2.latent_diffusion.modules.phoneme_encoder.encoder", TextEncoder=_Unused)
    _module("audioldm2.audiomae_gen.sequence_input", Sequence2AudioMAE=_Unused)
    cond = importlib.import_module("audioldm2.latent_diffusion.modules.encoders.modules").CLAPAudioEmbeddingClassifierFreev2
    return htsat.HTSAT_Swin_Transformer, clap_model, cond


AUDIO_CFG = dict(audio_length=1024, clip_samples=480000, mel_bins=64, sample_rate=48000, window_size=1024, hop_size=480,
                 fmin=50, fmax=14000, class_num=527, model_type="HTSAT", model_name="base")


def audio_model(htsat_cls, clap_cls, depths, text=None):
    """A CLAP stand-in holding the reference HTSAT (the audio branch create_htsat_model builds for "base", with ``depths``)
    and audio_projection, loaded from the synthetic weights; plus the text branch of ``text`` when given."""
    cfg = types.SimpleNamespace(**AUDIO_CFG)
    m = nn.Module()
    m.audio_branch = htsat_cls(spec_size=256, patch_size=4, patch_stride=(4, 4), num_classes=527, embed_dim=128,
                               depths=list(depths), num_heads=[4, 8, 16, 32], window_size=8, config=cfg,
                               enable_fusion=False, fusion_type="None")
    m.audio_projection = nn.Sequential(nn.Linear(1024, 512), nn.ReLU(), nn.Linear(512, 512))
    missing, unexpected = m.load_state_dict(CA.weights(depths), strict=False)
    assert not unexpected, unexpected
    assert all(k.endswith(("relative_position_index", "attn_mask", "num_batches_tracked")) or ".tscam_conv." in k or
               ".head." in k for k in missing), missing
    if text is not None:
        m.text_branch, m.text_projection, m.text_branch_type = text.text_branch, text.text_projection, "roberta"
        for name in ("encode_text", "get_text_embedding"):
            setattr(m, name, types.MethodType(getattr(clap_cls, name), m))
    m.eval()
    for p in m.parameters():
        p.requires_grad = False
    for name in ("encode_audio", "get_audio_embedding"):
        setattr(m, name, types.MethodType(getattr(clap_cls, name), m))
    return m


class Tokenize:
    """The RoBERTa tokenizer's call signature over synth.clap_tokenize."""

    def __call__(self, text, padding, truncation, max_length, return_tensors):
        assert (padding, truncation, max_length, return_tensors) == ("max_length", True, 512, "pt")
        ids, mask = synth.clap_tokenize([text] if isinstance(text, str) else list(text))
        return {"input_ids": ids, "attention_mask": mask.long()}


class _NoMel(nn.Module):
    """Stands for torchaudio's MelSpectrogram: its output only feeds mel_fusion, which the non-fusion HTSAT never reads."""

    def forward(self, x):
        return torch.zeros(x.shape[0], 64, 1)


def ranker_stub(cond_cls, model, sr):
    """The attributes CLAPAudioEmbeddingClassifierFreev2.__init__ sets (encoders/modules.py:547-605) that cos_similarity
    and forward read."""

    class Stub:
        def __call__(self, batch):
            return cond_cls.forward(self, batch)

    s = Stub()
    s.model, s.tokenize, s.device, s.cuda = model, Tokenize(), "cpu", False
    s.embed_mode, s.sampling_rate, s.unconditional_prob, s.unconditional_token = "audio", sr, 0.1, None
    s.training, s.training_mode = False, False
    s.model_cfg = {"audio_cfg": AUDIO_CFG}
    s.mel_transform = _NoMel()
    for name in ("forward", "tokenizer", "make_decision", "build_unconditional_emb", "cos_similarity"):
        setattr(s, name, types.MethodType(getattr(cond_cls, name), s))
    return s


def main():
    htsat_cls, clap_cls, cond_cls = reference()
    import torchaudio.functional as AF
    out = {}
    for depths in (CA.SMALL, CA.BASE):
        m = audio_model(htsat_cls, clap_cls, depths)
        if depths == CA.BASE:
            out["param_shapes"] = {k: list(v.shape) for k, v in m.state_dict().items()}
            blocks = m.audio_branch.layers
            out["relative_position_index"] = blocks[0].blocks[0].attn.relative_position_index.to(torch.int16)
            for layer in blocks:
                b = layer.blocks[1]
                if b.attn_mask is not None:
                    am = b.attn_mask
                    assert bool(((am == 0) | (am == -100)).all())
                    out[f"attn_mask_bits.{layer.input_resolution[0]}"] = torch.from_numpy(
                        np.packbits((am != 0).numpy().reshape(-1)))
        for name, (dep, sr, L, n, _) in CA.CASES.items():
            if dep != depths:
                continue
            wav = CA.inputs(name)
            x = AF.resample(wav, orig_freq=sr, new_freq=48000) if sr != 48000 else wav
            from audioldm2.clap.training.data import get_audio_features
            d = get_audio_features(x, torch.zeros(1, 64), 480000, data_truncating="fusion", data_filling="repeatpad",
                                   audio_cfg=AUDIO_CFG)
            with torch.no_grad():
                e = m.get_audio_embedding(d)
            out[name] = e.float().contiguous()
            print(name, tuple(e.shape))
    # the seeded cos_similarity call: audio and text replaced at least once each
    from transformers import RobertaConfig, RobertaModel
    rcfg = RobertaConfig(vocab_size=50265, hidden_size=768, num_hidden_layers=CA.TEXT_LAYERS, num_attention_heads=12,
                         intermediate_size=3072, hidden_act="gelu", max_position_embeddings=514, type_vocab_size=1,
                         layer_norm_eps=1e-5, pad_token_id=1, bos_token_id=0, eos_token_id=2)
    text = nn.Module()
    text.text_branch = RobertaModel(rcfg)
    text.text_projection = nn.Sequential(nn.Linear(768, 512), nn.ReLU(), nn.Linear(512, 512))
    missing, unexpected = text.load_state_dict(CA.text_weights(), strict=False)
    assert not unexpected and all(k.endswith(("position_ids", "token_type_ids")) for k in missing), (missing, unexpected)
    m = audio_model(htsat_cls, clap_cls, CA.SMALL, text=text)
    s = ranker_stub(cond_cls, m, 16000)
    wav, texts, B = CA.rank_inputs()
    s.build_unconditional_emb()
    for seed in range(CA.RANK_SEED, CA.RANK_SEED + 1000):
        torch.manual_seed(seed)
        sim = s.cos_similarity(wav, texts)
        st = torch.get_rng_state()
        torch.manual_seed(seed)
        ra = [i for i in range(len(texts)) if float(torch.rand(1)) < 0.1]
        rt = [i for i in range(len(texts)) if float(torch.rand(1)) < 0.1]
        if ra and rt:
            break
    best = [i + int(torch.argmax(sim[i::B]).item()) * B for i in range(B)]
    out.update(rank_similarity=sim.float().contiguous(), rank_best=torch.tensor(best), rank_seed=torch.tensor(seed),
               rank_audio_replaced=torch.tensor(ra), rank_text_replaced=torch.tensor(rt), rank_rng_state=st)
    print("rank", seed, ra, rt, best, sim.tolist())
    torch.save(out, CA.PATH)
    print(f"wrote {CA.PATH} ({os.path.getsize(CA.PATH) / 1e3:.0f} KB)")


if __name__ == "__main__":
    main()
