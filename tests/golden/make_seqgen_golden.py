"""Generate tests/golden/seqgen.pt by running the UNMODIFIED reference AudioMAE token generator.

    ALDM_REFERENCE_ROOT=<checkout of the reference> python tests/golden/make_seqgen_golden.py

``Sequence2AudioMAE.generate``, ``get_input_sequence_and_mask``, ``add_sos_eos_tokens`` and
``truncate_sequence_and_mask`` (audiomae_gen/sequence_input.py) are called as they are, on a stub ``self`` that holds
what the constructor would have built: HF ``GPT2Model(GPT2Config(n_layer=n, attn_implementation="eager"))`` (the
reference reads ``GPT2Config.from_pretrained("gpt2")``, which is GPT-2 small: the same values as the GPT2Config()
defaults), the SOS / EOS embeddings and the two input projections, all loaded strict from synth.seqgen_state_dict.  The
constructor itself is never run: it downloads the GPT-2 config and instantiates the CLAP, T5 and AudioMAE encoders.
Stored: the generated tokens of every case in seqgen_cases.CASES and the reference's parameter names and shapes.
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
from tests.golden import seqgen_cases           # noqa: E402


def reference_class():
    root = ref_loader.REF_ROOT
    if root not in sys.path:
        sys.path.insert(0, root)
    base = os.path.join(root, "audioldm2")
    ref_loader._stub_pkg("audioldm2", base)
    ref_loader._stub_pkg("audioldm2.latent_diffusion", os.path.join(base, "latent_diffusion"))
    ref_loader._stub_pkg("audioldm2.audiomae_gen", os.path.join(base, "audiomae_gen"))
    import importlib
    return importlib.import_module("audioldm2.audiomae_gen.sequence_input").Sequence2AudioMAE


def stub(cls, n_layer: int):
    """The attributes Sequence2AudioMAE.__init__ sets that generate() reads (sequence_input.py:27-60), as a Module so that
    load_state_dict checks every key; the four methods are the reference's, bound to it."""
    from transformers import GPT2Config, GPT2Model
    m = nn.Module()
    m.model = GPT2Model(GPT2Config(n_layer=n_layer, attn_implementation="eager"))
    m.start_of_sequence_tokens = nn.Embedding(32, 768)
    m.end_of_sequence_tokens = nn.Embedding(32, 768)
    m.input_sequence_embed_linear = nn.ModuleList([nn.Linear(512, 768), nn.Linear(1024, 768)])
    m.sequence_input_key = ["film_clap_cond1", "crossattn_flan_t5"]        # utils.py:362-368
    m.mae_token_num = 8
    for name in ("generate", "get_input_sequence_and_mask", "add_sos_eos_tokens", "truncate_sequence_and_mask"):
        setattr(m, name, types.MethodType(getattr(cls, name), m))
    return m


def main():
    cls = reference_class()
    out = {}
    for n_layer in sorted({c[0] for c in seqgen_cases.CASES.values()}):
        m = stub(cls, n_layer).eval()
        sd = seqgen_cases.weights(n_layer)
        m.load_state_dict(sd, strict=True)
        if n_layer == 12:
            out["param_shapes"] = {k: list(v.shape) for k, v in m.state_dict().items()}
        for name, (nl, lens, _) in seqgen_cases.CASES.items():
            if nl != n_layer:
                continue
            clap, t5, mask = seqgen_cases.inputs(name)
            with torch.no_grad():
                tokens, _ = m.generate(None, cond_dict={"film_clap_cond1": clap, "crossattn_flan_t5": [t5, mask]})
            out[name] = tokens.float().contiguous()
            print(name, tuple(tokens.shape), float(tokens.abs().max()))
    torch.save(out, seqgen_cases.PATH)
    print("wrote", seqgen_cases.PATH)


if __name__ == "__main__":
    main()
