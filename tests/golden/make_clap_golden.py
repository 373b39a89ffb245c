"""Generate tests/golden/clap.pt by running the UNMODIFIED reference CLAP text conditioner.

    ALDM_REFERENCE_ROOT=<checkout of the reference> python tests/golden/make_clap_golden.py

``CLAPAudioEmbeddingClassifierFreev2.forward``, ``tokenizer``, ``make_decision``, ``build_unconditional_emb`` and
``get_unconditional_condition`` (encoders/modules.py:546-745) are called as they are, on a stub ``self`` that holds what
the constructor would have built: a CLAP stand-in (an ``nn.Module``) with HF ``RobertaModel(RobertaConfig(<roberta-base
values>, num_hidden_layers=n))`` as ``text_branch`` and the ``text_projection`` Sequential, loaded strict from
synth.clap_text_state_dict, on which the reference's own ``CLAP.encode_text`` and ``get_text_embedding``
(clap/open_clip/model.py:629-663, 730-750) are bound; and a ``tokenize`` stand-in that returns the case's ids and mask
padded to 512 (the BPE vocabulary is a hub asset; "" tokenizes to [0, 2]).  The constructors themselves are never run:
they download the tokenizer and the pretrained model.  ``torchlibrosa`` and the HTSAT / PANN audio modules are replaced by
empty stand-ins in ``sys.modules`` here, in this script only.
Stored: the embedding of every case in clap_cases.CASES, CLAP("") of clap_cases.UNCOND, a seeded ``forward`` call at B = 8
(its output, the seed -- the first one for which at least one row is replaced by CLAP("") --, the replaced rows and the
CPU generator state after the call), and the reference's parameter names and shapes.
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

import torch                                    # noqa: E402
import torch.nn as nn                           # noqa: E402

from oracle import ref_loader                   # noqa: E402
from tests.golden import clap_cases             # noqa: E402


def _module(name: str, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


def reference_classes():
    """-> (CLAPAudioEmbeddingClassifierFreev2, CLAP), imported from the reference's own files."""
    root = ref_loader.REF_ROOT
    if root not in sys.path:
        sys.path.insert(0, root)
    base = os.path.join(root, "audioldm2")
    ref_loader._stub_pkg("audioldm2", base)
    ref_loader._stub_pkg("audioldm2.clap", os.path.join(base, "clap"))
    ref_loader._stub_pkg("audioldm2.clap.open_clip", os.path.join(base, "clap", "open_clip"))
    ref_loader._stub_pkg("audioldm2.latent_diffusion", os.path.join(base, "latent_diffusion"))
    ref_loader._stub_pkg("audioldm2.latent_diffusion.modules", os.path.join(base, "latent_diffusion", "modules"))
    ref_loader._stub_pkg("audioldm2.latent_diffusion.modules.encoders", os.path.join(base, "latent_diffusion", "modules", "encoders"))

    class _Unused(nn.Module):
        pass

    sys.modules["audioldm2.clap.open_clip"].create_model = None
    _module("torchlibrosa")
    _module("audioldm2.clap.open_clip.pann_model", create_pann_model=None)
    _module("audioldm2.clap.open_clip.htsat", create_htsat_model=None)
    _module("audioldm2.clap.open_clip.utils", freeze_batch_norm_2d=None)
    _module("audioldm2.clap.training")
    _module("audioldm2.clap.training.data", get_audio_features=None)
    if "torchaudio" not in sys.modules:
        try:
            import torchaudio  # noqa: F401
        except ImportError:
            _module("torchaudio")
    _module("audioldm2.latent_diffusion.modules.audiomae.AudioMAE", Vanilla_AudioMAE=_Unused)
    _module("audioldm2.latent_diffusion.modules.phoneme_encoder.encoder", TextEncoder=_Unused)
    _module("audioldm2.audiomae_gen.sequence_input", Sequence2AudioMAE=_Unused)
    clap_model = importlib.import_module("audioldm2.clap.open_clip.model").CLAP
    cond = importlib.import_module("audioldm2.latent_diffusion.modules.encoders.modules").CLAPAudioEmbeddingClassifierFreev2
    return cond, clap_model


class FakeTokenize:
    """What ``RobertaTokenizer.from_pretrained("roberta-base")(text, padding="max_length", truncation=True,
    max_length=512, return_tensors="pt")`` returns (input_ids, attention_mask), for prompt lists that are keys of
    ``table``."""

    def __init__(self, table):
        self.table = table

    def __call__(self, text, padding, truncation, max_length, return_tensors):
        assert (padding, truncation, max_length, return_tensors) == ("max_length", True, 512, "pt")
        ids, mask = self.table[tuple([text] if isinstance(text, str) else text)]
        return {"input_ids": ids.clone(), "attention_mask": mask.long()}


def stub(cond_cls, clap_cls, n_layer: int, table):
    """The attributes CLAPAudioEmbeddingClassifierFreev2.__init__ sets (encoders/modules.py:547-605) that the text path
    reads; the model is a CLAP stand-in holding the text branch (clap/open_clip/model.py:513-529)."""
    from transformers import RobertaConfig, RobertaModel
    cfg = RobertaConfig(vocab_size=50265, hidden_size=768, num_hidden_layers=n_layer, num_attention_heads=12,
                        intermediate_size=3072, hidden_act="gelu", hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1,
                        max_position_embeddings=514, type_vocab_size=1, initializer_range=0.02, layer_norm_eps=1e-5,
                        pad_token_id=1, bos_token_id=0, eos_token_id=2)

    class CLAPText(nn.Module):
        def __init__(self):
            super().__init__()
            self.text_branch = RobertaModel(cfg)
            self.text_projection = nn.Sequential(nn.Linear(768, 512), nn.ReLU(), nn.Linear(512, 512))
            self.text_branch_type = "roberta"

    m = CLAPText()
    missing, unexpected = m.load_state_dict(clap_cases.weights(n_layer), strict=False)
    assert not unexpected and all(k.endswith(("position_ids", "token_type_ids")) for k in missing), (missing, unexpected)
    m.eval()
    for p in m.parameters():
        p.requires_grad = False
    for name in ("encode_text", "get_text_embedding"):
        setattr(m, name, types.MethodType(getattr(clap_cls, name), m))

    class Stub:
        def __call__(self, batch):
            return cond_cls.forward(self, batch)

    s = Stub()
    s.model = m
    s.tokenize = FakeTokenize(table)
    s.device = "cpu"
    s.embed_mode = "text"
    s.unconditional_prob = 0.1
    s.unconditional_token = None
    s.training = False
    s.training_mode = False
    for name in ("forward", "tokenizer", "make_decision", "build_unconditional_emb", "get_unconditional_condition"):
        setattr(s, name, types.MethodType(getattr(cond_cls, name), s))
    return s


def _empty(n):
    ids, mask = torch.ones(n, 512, dtype=torch.int64), torch.zeros(n, 512)
    ids[:, 0], ids[:, 1] = 0, 2
    mask[:, :2] = 1
    return ids, mask


def main():
    cond_cls, clap_cls = reference_classes()
    out = {}
    for n_layer in sorted({c[0] for c in clap_cases.CASES.values()}):
        table = {("", ""): _empty(2)}
        names = [n for n, c in clap_cases.CASES.items() if c[0] == n_layer]
        for name in names:
            ids, mask = clap_cases.inputs(name)
            table[tuple(f"{name}.{i}" for i in range(ids.shape[0]))] = (ids, mask)
        s = stub(cond_cls, clap_cls, n_layer, table)
        if n_layer == 12:
            out["param_shapes"] = {k: list(v.shape) for k, v in s.model.state_dict().items()}
        for name in names:
            ids, mask = clap_cases.inputs(name)
            texts = [f"{name}.{i}" for i in range(ids.shape[0])]
            if ids.shape[0] == 1:        # forward's single-prompt path: the tokenizer squeezes, forward unsqueezes
                s.tokenize.table[(texts[0],)] = (ids, mask)
            with torch.no_grad():
                e = s.model.get_text_embedding(s.tokenizer(texts) if ids.shape[0] > 1 else
                                               {k: v.unsqueeze(0) for k, v in s.tokenizer(texts).items()})
            out[name] = e.float().contiguous()
            print(name, tuple(e.shape))
        for name, nl in clap_cases.UNCOND.items():
            if nl == n_layer:
                u = s.get_unconditional_condition(2)
                assert u.shape == (2, 1, 512) and torch.equal(u[0], u[1])
                out[name] = u[0].float().contiguous()
                print(name, tuple(u.shape))
        if n_layer == clap_cases.FORWARD[0]:
            name = clap_cases.FORWARD[1]
            texts = [f"{name}.{i}" for i in range(clap_cases.CASES[name][1].__len__())]
            s.build_unconditional_emb()
            assert not any(torch.equal(out[name][i:i + 1], s.unconditional_token) for i in range(len(texts)))
            for seed in range(1000):
                torch.manual_seed(seed)
                e = s(texts)
                replaced = [i for i in range(e.shape[0]) if torch.equal(e[i], s.unconditional_token)]
                if replaced:
                    break
            out.update(forward=e.float().contiguous(), forward_seed=torch.tensor(seed),
                       forward_replaced=torch.tensor(replaced, dtype=torch.int64), forward_rng_state=torch.get_rng_state())
            print("forward", seed, replaced)
    torch.save(out, clap_cases.PATH)
    print(f"wrote {clap_cases.PATH} ({os.path.getsize(clap_cases.PATH) / 1e3:.0f} KB)")


if __name__ == "__main__":
    main()
