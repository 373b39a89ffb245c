"""Generate tests/golden/t5.pt by running the UNMODIFIED reference Flan-T5 encoder wrapper.

    ALDM_REFERENCE_ROOT=<checkout of the reference> python tests/golden/make_t5_golden.py

``FlanT5HiddenState.encode_text``, ``forward`` and ``get_unconditional_condition`` (encoders/modules.py:113-198) are
called as they are, on a stub ``self`` that holds what the constructor would have built: HF
``T5EncoderModel(T5Config(<google/flan-t5-large values>, num_layers=n))`` loaded strict from synth.t5_state_dict, and a
tokenizer stand-in that returns the case's ids and mask (the sentencepiece model is a hub asset; "" tokenizes to [1]).
The constructor itself is never run: it downloads the tokenizer and the config.  ``encoders/modules.py`` imports the
CLAP, AudioMAE, phoneme-encoder and GPT-2 modules at module level; those are replaced by empty stand-ins in
``sys.modules`` here, in this script only.
Stored: the hidden states of every case in t5_cases.CASES, T5("") of t5_cases.UNCOND, and the reference's parameter names
and shapes.  The larger hidden states are kept as evenly spaced samples of their elements (``cases.Sampled``, the layout
of make_golden.py's fixtures), so that the file stays under 1 MB.
"""
from __future__ import annotations

import os
import sys
import types

os.environ["HF_HUB_OFFLINE"] = "1"
os.environ["TRANSFORMERS_OFFLINE"] = "1"

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import torch                                    # noqa: E402
import torch.nn as nn                           # noqa: E402

from oracle import ref_loader                   # noqa: E402
from tests.golden import cases, t5_cases        # noqa: E402

SAMPLE_BUDGET = 150_000      # float32 elements kept in the file: it stays well under 1 MB


def _module(name: str, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m


def reference_class():
    root = ref_loader.REF_ROOT
    if root not in sys.path:
        sys.path.insert(0, root)
    base = os.path.join(root, "audioldm2")
    ref_loader._stub_pkg("audioldm2", base)
    ref_loader._stub_pkg("audioldm2.latent_diffusion", os.path.join(base, "latent_diffusion"))
    ref_loader._stub_pkg("audioldm2.latent_diffusion.modules", os.path.join(base, "latent_diffusion", "modules"))
    ref_loader._stub_pkg("audioldm2.latent_diffusion.modules.encoders", os.path.join(base, "latent_diffusion", "modules", "encoders"))

    class _Unused(nn.Module):
        pass

    _module("audioldm2.clap.open_clip", create_model=None)
    _module("audioldm2.clap.training.data", get_audio_features=None)
    if "torchaudio" not in sys.modules:
        try:
            import torchaudio  # noqa: F401
        except ImportError:
            _module("torchaudio")
    _module("audioldm2.latent_diffusion.modules.audiomae.AudioMAE", Vanilla_AudioMAE=_Unused)
    _module("audioldm2.latent_diffusion.modules.phoneme_encoder.encoder", TextEncoder=_Unused)
    _module("audioldm2.audiomae_gen.sequence_input", Sequence2AudioMAE=_Unused)
    import importlib
    return importlib.import_module("audioldm2.latent_diffusion.modules.encoders.modules").FlanT5HiddenState


class FakeTokenizer:
    """What ``AutoTokenizer.from_pretrained("google/flan-t5-large")(prompt, max_length=128, padding=True,
    truncation=True, return_tensors="pt")`` returns, for prompts that are keys of ``table`` (ids, mask)."""

    def __init__(self, table):
        self.table = table

    def __call__(self, prompt, max_length, padding, truncation, return_tensors):
        assert (max_length, padding, truncation, return_tensors) == (128, True, True, "pt")
        ids, mask = self.table[tuple(prompt)]
        return types.SimpleNamespace(input_ids=ids, attention_mask=mask.long())


def stub(cls, n_layer: int, table):
    """The attributes FlanT5HiddenState.__init__ sets (encoders/modules.py:121-136); forward, encode_text and
    get_unconditional_condition are the reference's, bound to it."""
    from transformers import T5Config, T5EncoderModel
    cfg = T5Config(vocab_size=32128, d_model=1024, d_kv=64, d_ff=2816, num_layers=n_layer, num_heads=16,
                   relative_attention_num_buckets=32, relative_attention_max_distance=128, dropout_rate=0.1,
                   layer_norm_epsilon=1e-6, feed_forward_proj="gated-gelu", tie_word_embeddings=False, pad_token_id=0,
                   eos_token_id=1, decoder_start_token_id=0)
    assert cfg.dense_act_fn == "gelu_new"

    class Stub:
        def __call__(self, batch):
            return cls.forward(self, batch)

    s = Stub()
    s.model = T5EncoderModel(cfg)
    s.model.load_state_dict(t5_cases.weights(n_layer), strict=True)
    s.model.eval()
    for p in s.model.parameters():
        p.requires_grad = False
    s.tokenizer = FakeTokenizer(table)
    s.freeze_text_encoder = True
    s.empty_hidden_state_cfg = None
    s.device = None
    for name in ("forward", "encode_text", "get_unconditional_condition"):
        setattr(s, name, types.MethodType(getattr(cls, name), s))
    return s


def main():
    cls = reference_class()
    out = {}
    for n_layer in sorted({c[0] for c in t5_cases.CASES.values()}):
        table = {("",): (torch.tensor([[1]]), torch.tensor([[1]]))}
        names = [n for n, c in t5_cases.CASES.items() if c[0] == n_layer]
        for name in names:
            ids, mask = t5_cases.inputs(name)
            table[(name,) * ids.shape[0]] = (ids, mask)
        s = stub(cls, n_layer, table)
        if n_layer == 24:
            out["param_shapes"] = {k: list(v.shape) for k, v in s.model.state_dict().items()}
        for name in names:
            ids, _ = t5_cases.inputs(name)
            h, m = s.encode_text([name] * ids.shape[0])
            out[name] = h.float().contiguous()
            print(name, tuple(h.shape), float(h.abs().max()))
        for name, nl in t5_cases.UNCOND.items():
            if nl == n_layer:
                h, m = s.get_unconditional_condition(2)
                assert h.shape == (2, 1, 1024) and torch.equal(m, torch.ones(2, 1)) and torch.equal(h[0], h[1])
                out[name] = h[:1].float().contiguous()
                print(name, tuple(h.shape))
    big = {k: v for k, v in out.items() if torch.is_tensor(v) and v.numel() > 4096}
    total = sum(v.numel() for v in big.values())
    for k, v in big.items():
        n = min(v.numel(), max(4096, SAMPLE_BUDGET * v.numel() // total))
        del out[k]
        out[k + ".sample"] = v.reshape(-1)[cases.sample_index(v.numel(), n)].clone()
        out[k + ".shape"] = torch.tensor(list(v.shape), dtype=torch.int64)
    torch.save(out, t5_cases.PATH)
    print(f"wrote {t5_cases.PATH} ({os.path.getsize(t5_cases.PATH) / 1e3:.0f} KB)")


if __name__ == "__main__":
    main()
