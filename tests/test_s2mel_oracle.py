"""CPU: s2mel / codec restatement against goldens minted from the reference modules."""
import os

import numpy as np
import torch

from oracle.s2mel import (cfm_inference, codec_decode, dit_forward, fold_weight_norm, length_regulate,
                          make_codec_weights, make_s2mel_weights, small_codec_cfg, small_s2mel_cfg)

GOLD = os.path.join(os.path.dirname(__file__), "golden", "s2mel_small.npz")


def test_small_pipeline_matches_reference_golden():
    g = np.load(GOLD)
    c, cc = small_s2mel_cfg(), small_codec_cfg()
    w = fold_weight_norm(make_s2mel_weights(c, seed=int(g["seed_s2mel"])))
    wc = fold_weight_norm(make_codec_weights(cc, seed=int(g["seed_codec"])))
    S = codec_decode(wc, torch.from_numpy(g["codes"]))
    assert np.abs(S.numpy() - g["S_infer"]).max() < 1e-5
    cond = length_regulate(w, torch.from_numpy(g["lr_in"]), int(g["ylen"]))
    assert np.abs(cond.numpy() - g["cond"]).max() < 1e-5
    mu, prompt, style, z = (torch.from_numpy(g[k]) for k in ("mu", "prompt", "style", "z"))
    T, P = mu.shape[1], prompt.shape[-1]
    px = torch.zeros(1, 80, T)
    px[..., :P] = prompt
    d = dit_forward(w, c, z, px, torch.LongTensor([T]), torch.from_numpy(g["t"]), style, mu)
    assert np.abs(d.numpy() - g["dit"]).max() < 2e-4
    mel = cfm_inference(w, c, mu, torch.LongTensor([T]), prompt, style, z, int(g["n_steps"]), 0.7)
    assert np.abs(mel.numpy() - g["mel"]).max() < 1e-3
    assert np.all(mel.numpy()[:, :, :P] == 0)


def test_weight_norm_fold():
    v = torch.randn(6, 4, 3)
    gg = torch.rand(6, 1, 1) + 0.5
    w = fold_weight_norm({"c.weight_g": gg, "c.weight_v": v, "c.bias": torch.zeros(6)})
    ref = torch._weight_norm(v, gg, 0)
    assert torch.allclose(w["c.weight"], ref, atol=1e-6) and "c.bias" in w and "c.weight_v" not in w


def test_short_sequences_match_reference_golden():
    """1- and 2-frame inputs, where the WaveNet's reflect padding (encodec.py pad1d) zero-extends before it reflects:
    the oracle's SConv1d and one small-dims DiT evaluation against the reference modules."""
    from oracle.s2mel import _reflect_conv
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "s2mel_short.npz"))
    w, b = torch.from_numpy(g["sconv_weight"]), torch.from_numpy(g["sconv_bias"])
    for T in (1, 2, 3):
        y = _reflect_conv(torch.from_numpy(g[f"sconv_x{T}"]), w, b, 5)
        assert np.abs(y.numpy() - g[f"sconv_y{T}"]).max() < 1e-5
    c = small_s2mel_cfg()
    wd = fold_weight_norm(make_s2mel_weights(c, seed=int(g["seed_s2mel"])))
    for T in (1, 2):
        mu, style, z, t = (torch.from_numpy(g[f"dit{T}_{k}"]) for k in ("mu", "style", "z", "t"))
        d = dit_forward(wd, c, z, torch.zeros(1, 80, T), torch.LongTensor([T]), t, style, mu)
        assert np.abs(d.numpy() - g[f"dit{T}"]).max() < 2e-4
