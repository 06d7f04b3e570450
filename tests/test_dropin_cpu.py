"""CPU: `dropin.load_reference_weights`, `attach` and `attach_v1` against what the reference's own modules expose.  The
reference's classes were instantiated (random init, small dims) by oracle/make_goldens_dropin.py, which stored their
state-dict names and shapes and the attributes the drop-in reads (tests/golden/dropin_modules.json); the reference's seam
call sites are in tests/golden/reference_signatures.json (oracle/make_goldens_signatures.py).  Shape-only stand-ins are
rebuilt from them, a recording stand-in replaces the engine, and the tests check that every hyper-parameter the drop-in
derives from the modules' state dicts equals what the modules were constructed with, that every tensor name the engine
will ask for (`gpt.…`, `s2mel.…`, `codec.…`, `bigvgan.…`) is present, and that the reference's calls bind to the
callables the drop-in installs."""
import json
import os
import types

import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _golden(name):
    with open(os.path.join(GOLDEN, name)) as f:
        return json.load(f)


class StandIn(torch.nn.Module):
    """A module that has only the recorded state-dict entries (zeros of the recorded shapes)."""

    def __init__(self, shapes, **attrs):
        super().__init__()
        self._shapes = shapes
        for k, v in attrs.items():
            object.__setattr__(self, k, v)

    def state_dict(self, *a, **k):
        return {n: torch.zeros(s) for n, s in self._shapes.items()}


def _gpt(rec):
    a = rec["attrs"]
    sd = rec["state_dict"]
    extra = dict(gpt=types.SimpleNamespace(h=[None] * a["layers"]),
                 inference_model=types.SimpleNamespace(kv_cache=a["kv_cache"]))
    if "emo_perceiver_heads" in a:
        extra["emo_perceiver_encoder"] = types.SimpleNamespace(heads=a["emo_perceiver_heads"],
                                                               latents=torch.zeros(sd["emo_perceiver_encoder.latents"]))
    if "emo_input_size" in a:
        extra["emo_input_size"] = a["emo_input_size"]
    return StandIn(sd, **{k: a[k] for k in ("model_dim", "heads", "number_mel_codes", "start_mel_token", "stop_mel_token")},
                   **extra)


def _tts_v2_5():
    g = _golden("dropin_modules.json")
    gpt = _gpt(g["gpt"])
    s2 = StandIn(g["s2mel"]["state_dict"])
    s2.models = {"length_regulator": torch.nn.Module(), "cfm": types.SimpleNamespace(in_channels=80)}
    codec = StandIn(g["codec"]["state_dict"])
    bv = StandIn(g["bigvgan"]["state_dict"], h=g["bigvgan"]["attrs"]["h"])
    return g, types.SimpleNamespace(gpt=gpt, s2mel=s2, semantic_codec=codec, bigvgan=bv)


class RecordingEngine:
    device = 0

    def __init__(self):
        self.weights, self.calls = {}, {}

    def load_state_dict(self, prefix, sd):
        for k, v in sd.items():
            self.weights[prefix + k] = tuple(v.shape)

    def gpt_init(self, *a, **k):
        self.calls["gpt_init"] = (a, k)

    def emo_init(self, c):
        self.calls["emo_init"] = dict(c)
        self.emo_cfg = types.SimpleNamespace(**c)

    def s2mel_init(self, c):
        self.calls["s2mel_init"] = dict(c)

    def codec_init(self, c):
        self.calls["codec_init"] = dict(c)

    def bigvgan_init(self, h):
        self.calls["bigvgan_init"] = dict(h)


def test_config_derivation_from_real_reference_modules():
    from indextts_b200.dropin import load_reference_weights

    g, tts = _tts_v2_5()
    cfg, h = g["cfg"], g["h"]
    eng = RecordingEngine()
    load_reference_weights(eng, tts, max_batch=4)

    a, k = eng.calls["gpt_init"]
    assert a[:6] == (cfg["layers"], cfg["model_dim"], cfg["heads"], cfg["number_mel_codes"], cfg["start_mel_token"],
                     cfg["stop_mel_token"])
    assert a[6] == cfg["max_mel_tokens"] + 2 + 1            # mel_pos rows (model_v2.py:398-400)
    assert k["max_batch"] == 4 and k["weights_bf16"] is True
    emo = eng.calls["emo_init"]
    assert (emo["idim"], emo["odim"], emo["linear_units"], emo["heads"], emo["blocks"]) == (1024, 32, 48, 2, 1)
    assert emo["model_dim"] == cfg["model_dim"] and emo["p_dim"] == tts.gpt.emo_perceiver_encoder.latents.shape[-1]
    s = eng.calls["s2mel_init"]
    assert (s["hidden"], s["heads"], s["depth"], s["wn_hidden"], s["wn_layers"], s["wn_kernel"]) == (64, 1, 3, 64, 2, 5)
    assert (s["in_channels"], s["content_dim"], s["style_dim"], s["lr_in"], s["lr_convs"]) == (80, 64, 24, 96, 4)
    c = eng.calls["codec_init"]
    assert c == dict(codebook_size=64, hidden_size=96, codebook_dim=8, vocos_dim=48, vocos_intermediate_dim=64,
                     vocos_num_layers=2)
    assert eng.calls["bigvgan_init"]["upsample_rates"] == list(h["upsample_rates"])
    # the tensors the C++ side looks up by name exist under the names the reference uses
    need = ["gpt.gpt.h.0.attn.c_attn.weight", "gpt.mel_head.weight", "gpt.final_norm.weight", "gpt.spk_emb_proj.weight",
            "gpt.lang_embedding.weight", "gpt.text_pos_embedding.emb.weight", "gpt.emovec_layer.weight",
            "gpt.emo_conditioning_encoder.embed.out.0.weight", "gpt.emo_perceiver_encoder.latents",
            "s2mel.cfm.estimator.cond_projection.weight", "s2mel.cfm.estimator.wavenet.in_layers.0.conv.conv.weight",
            "s2mel.length_regulator.content_in_proj.weight", "codec.quantizer.quantizers.0.codebook.weight",
            "codec.decoder.1.weight", "bigvgan.conv_pre.weight", "bigvgan.ups.0.0.weight",
            "bigvgan.resblocks.0.convs1.0.weight", "bigvgan.conv_post.weight"]
    missing = [n for n in need if n not in eng.weights]
    assert not missing, missing
    assert not any(".weight_g" in n or ".weight_v" in n or "parametrizations" in n for n in eng.weights), \
        "weight-norm pairs must be folded before they reach the engine"


def _reference_call_sites():
    """(positional count, keyword names) of the calls `infer_generator` makes at the six seams (infer_v2_5.py:749-864)."""
    return _golden("reference_signatures.json")["call_sites_v2_5"]


def test_rebound_seams_accept_the_reference_call_sites():
    """Every call `infer_v2_5.py` makes at a seam binds to the callable `attach` installs there (same positional
    arity, same keyword names) — the drop-in claim of INTEGRATION.md, checked against the reference source."""
    import inspect

    from indextts_b200.dropin import attach

    _, tts = _tts_v2_5()
    gpt, bv = tts.gpt, tts.bigvgan
    eng = RecordingEngine()
    attach(tts, engine=eng)
    seams = {"merge_emovec": tts.gpt.merge_emovec, "inference_speech": tts.gpt.inference_speech,
             "codec_decode": tts.semantic_codec.decode, "length_regulator": tts.s2mel.models["length_regulator"].forward,
             "cfm_inference": tts.s2mel.models["cfm"].inference, "bigvgan": tts.bigvgan.forward}
    sites = _reference_call_sites()
    assert set(sites) == set(seams), (sorted(sites), sorted(seams))
    for name, calls in sites.items():
        sig = inspect.signature(seams[name])
        for npos, kws, star in calls:
            try:
                sig.bind(*([None] * npos), **{k: None for k in kws})
            except TypeError as e:
                raise AssertionError(f"{name}: reference call ({npos} positional, keywords {kws}) does not bind to {sig}: {e}")
    # the rebound objects are the reference's own module objects: infer_generator reaches them unchanged
    assert tts.gpt is gpt and tts.bigvgan is bv and tts._b200_engine is eng


def test_merge_emovec_refuses_lengths_below_the_feature_rows():
    """The reference's conformer masks feature rows at or beyond cond_lengths / emo_cond_lengths; the engine encodes every
    row.  The lengths infer_v2_5.py passes (the feature dim, 1024: trap P10) reach the engine unchanged; a length below
    the number of rows is refused rather than silently computing something else."""
    from indextts_b200.dropin import attach

    _, tts = _tts_v2_5()

    class Reached(Exception):
        """raised by the stand-in engine: the call got through to the engine (no device to return a tensor to here)"""

    class Rec(RecordingEngine):
        def merge_emovec(self, spk, emo, alpha):
            self.calls.setdefault("merge_emovec", []).append((tuple(spk.shape), tuple(emo.shape), alpha))
            raise Reached

    eng = Rec()
    attach(tts, engine=eng)
    spk, emo = torch.zeros(1, 64, 1024), torch.zeros(1, 90, 1024)
    full = torch.tensor([1024])
    for cl, el, alpha in ((full, full, 0.6), (torch.tensor([64]), torch.tensor([90]), 1.0), (None, None, 1.0)):
        with pytest.raises(Reached):     # the .infer() lengths, exactly the rows, no lengths: nothing is masked
            tts.gpt.merge_emovec(spk, emo, cl, el, alpha=alpha)
    assert eng.calls["merge_emovec"] == [((64, 1024), (90, 1024), 0.6), ((64, 1024), (90, 1024), 1.0),
                                         ((64, 1024), (90, 1024), 1.0)]
    for cl, el, what in ((torch.tensor([63]), full, "cond_lengths"), (full, torch.tensor([89]), "emo_cond_lengths")):
        with pytest.raises(RuntimeError, match=what):
            tts.gpt.merge_emovec(spk, emo, cl, el)
    assert len(eng.calls["merge_emovec"]) == 3


def test_attach_v1_on_real_reference_v1_modules():
    """v1 / v1.5 drop-in (row a13): `attach_v1` on the reference's own v1 `UnifiedVoice` and `BigVGAN` classes — the derived
    prompt-encoder / vocoder configuration equals what the modules were built with, and the calls `indextts/infer.py` makes
    at the three seams bind to the rebound callables."""
    import inspect

    from indextts_b200.dropin import attach_v1

    g = _golden("dropin_modules.json")
    cfg, ccfg, h = g["cfg"], g["ccfg"], g["h1"]
    gpt = _gpt(g["gpt_v1"])
    bv = StandIn(g["bigvgan_v1"]["state_dict"], h=g["bigvgan_v1"]["attrs"]["h"])
    tts = types.SimpleNamespace(gpt=gpt, bigvgan=bv)

    class Rec(RecordingEngine):
        def v1_cond_init(self, c, n):
            self.calls["v1_cond_init"] = (dict(c), n)

        def v1_vocoder_init(self, hh):
            self.calls["v1_vocoder_init"] = dict(hh)

    eng = Rec()
    attach_v1(tts, engine=eng)
    c, n = eng.calls["v1_cond_init"]
    assert n == 32
    for k in ("idim", "odim", "linear_units", "heads", "blocks", "cnn_kernel", "p_dim", "p_heads", "p_dim_head", "p_depth", "p_ff_mult"):
        assert c[k] == ccfg[k], (k, c[k], ccfg[k])
    a, kw = eng.calls["gpt_init"]
    assert a[:3] == (cfg["layers"], cfg["model_dim"], cfg["heads"]) and kw["weights_bf16"] is False
    assert eng.calls["v1_vocoder_init"]["gpt_dim"] == h["gpt_dim"]
    assert "bigvgan_v1.speaker_encoder.blocks.0.conv.conv.weight" in eng.weights and "bigvgan_v1.cond_layer.weight" in eng.weights
    assert "gpt.conditioning_encoder.embed.out.0.weight" in eng.weights and "gpt.perceiver_encoder.latents" in eng.weights
    # call sites of indextts/infer.py
    sites = _golden("reference_signatures.json")["call_sites_v1"]
    want = {"inference_speech": tts.gpt.inference_speech, "gpt_forward": tts.gpt.forward, "bigvgan": tts.bigvgan.forward}
    for name, calls in sites.items():
        for npos, kws, _ in calls:
            inspect.signature(want[name]).bind(*([None] * npos), **{k: None for k in kws})
    assert set(sites) == set(want)
