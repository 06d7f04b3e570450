"""Record what the drop-in reads from the reference's own modules as tests/golden/dropin_modules.json.

    IDX_REFERENCE=<reference checkout> python -m oracle.make_goldens_dropin

The reference's classes are instantiated (random init, small dims) through oracle/refimport.py, exactly as an
IndexTTS2 / IndexTTS object holds them: UnifiedVoice v2.5 and v1, the s2mel MyModel, the semantic codec, BigVGAN v2 and
the v1 BigVGAN.  For each module the file keeps the floating-point state-dict names and shapes and the plain attributes
`dropin.load_reference_weights` / `attach` / `attach_v1` read, plus the hyper-parameters the modules were built with.
tests/test_dropin_cpu.py rebuilds shape-only stand-ins from it."""
import json
import os

import torch

from oracle import refimport

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "dropin_modules.json")


def _shapes(module):
    return {k: list(v.shape) for k, v in module.state_dict().items() if torch.is_floating_point(v)}


def build():
    """The reference modules of the drop-in tests and the configurations they were built with."""
    from indextts_b200 import synth
    from oracle.gpt import make_gpt_weights
    from oracle.make_goldens_v1 import reference_module
    from oracle.validate_gpt_vs_hf import small_case

    cfg, _, _, _ = small_case()
    cfg = dict(cfg, n_langs=106)
    gpt = refimport.gpt_module(cfg, make_gpt_weights(cfg, seed=1, bf16=False))
    s2 = refimport.s2mel_module(refimport.s2mel_args(hidden=64, heads=1, depth=3, wn_hidden=64, wn_layers=2,
                                                     content_dim=64, lr_in=96, style_dim=24))
    codec = refimport.codec_module(codebook_size=64, hidden_size=96, codebook_dim=8, vocos_dim=48,
                                   vocos_intermediate_dim=64, vocos_num_layers=2)
    h = synth.small_config()
    bv = refimport.bigvgan_module(h)
    ccfg = synth.small_v1_cond_cfg(cfg["model_dim"])
    gpt1 = refimport.gpt_module_v1(cfg, ccfg, synth.make_gpt_v1_weights(cfg, ccfg, seed=3), kv_cache=False)
    h1 = synth.small_v1_config()
    bv1 = reference_module(h1, synth.make_bigvgan_v1_weights(h1, seed=5))
    return dict(cfg=cfg, ccfg=ccfg, h=h, h1=h1, gpt=gpt, s2mel=s2, codec=codec, bigvgan=bv, gpt_v1=gpt1, bigvgan_v1=bv1)


def _gpt_attrs(g):
    d = {k: getattr(g, k) for k in ("model_dim", "heads", "number_mel_codes", "start_mel_token", "stop_mel_token")}
    d["layers"] = len(g.gpt.h)
    if hasattr(g, "emo_perceiver_encoder"):
        d["emo_perceiver_heads"] = int(getattr(g.emo_perceiver_encoder, "heads", 0))
    if hasattr(g, "emo_input_size"):
        d["emo_input_size"] = int(g.emo_input_size)
    d["kv_cache"] = bool(getattr(getattr(g, "inference_model", None), "kv_cache", False))
    return d


def main():
    m = build()
    d = {"cfg": m["cfg"], "ccfg": m["ccfg"], "h": dict(m["h"]), "h1": dict(m["h1"]),
         "gpt": {"state_dict": _shapes(m["gpt"]), "attrs": _gpt_attrs(m["gpt"])},
         "gpt_v1": {"state_dict": _shapes(m["gpt_v1"]), "attrs": _gpt_attrs(m["gpt_v1"])},
         "s2mel": {"state_dict": _shapes(m["s2mel"])},
         "codec": {"state_dict": _shapes(m["codec"])},
         "bigvgan": {"state_dict": _shapes(m["bigvgan"]), "attrs": {"h": dict(m["bigvgan"].h)}},
         "bigvgan_v1": {"state_dict": _shapes(m["bigvgan_v1"]), "attrs": {"h": dict(m["bigvgan_v1"].h)}}}
    with open(OUT, "w") as f:
        json.dump(d, f, sort_keys=True, default=lambda o: list(o) if isinstance(o, tuple) else str(o))
        f.write("\n")
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
