"""Emotion-vector path (row a7): CPU oracle vs goldens from the reference modules; GPU engine vs both."""
import os

import numpy as np
import pytest
import torch

from oracle.emo import (EMO_CFG, conformer_encode, get_emovec, make_emo_weights, merge_emovec, perceiver_resample,
                        small_emo_cfg)

GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("name,cfg", [("emo_small", small_emo_cfg()), ("emo_full", dict(EMO_CFG))])
def test_oracle_matches_reference_golden(name, cfg):
    g = np.load(os.path.join(GOLD, name + ".npz"))
    w = make_emo_weights(cfg, seed=int(g["seed"]))
    ev = get_emovec(w, cfg, torch.from_numpy(g["feats"]))
    assert np.abs(ev.numpy() - g["emovec"]).max() < 5e-4


def test_oracle_matches_reference_golden_at_a_15s_prompt():
    """The oracle at T = 750 feature rows (T' = 374), where it is the yardstick of tests/test_emo_lengths_gpu.py: the
    reference modules' ctx, latent and emo_vec, the features re-drawn from the stored seed."""
    g = np.load(os.path.join(GOLD, "emo_full_t750.npz"))
    cfg = dict(EMO_CFG)
    w = make_emo_weights(cfg, seed=int(g["seed"]))
    feats = torch.randn(int(g["T"]), cfg["idim"], generator=torch.Generator().manual_seed(int(g["feats_seed"])))
    ctx = conformer_encode(w, cfg, feats)
    lat = perceiver_resample(w, cfg, ctx)
    ev = get_emovec(w, cfg, feats)
    assert ctx.shape == g["ctx"].shape == (374, cfg["odim"])
    assert np.abs(ctx.numpy() - g["ctx"]).max() < 2e-4 and np.abs(lat.numpy() - g["latent"]).max() < 2e-4
    assert np.abs(ev.numpy() - g["emovec"]).max() < 5e-4


@pytest.mark.gpu
@pytest.mark.parametrize("name,cfg", [("emo_small", small_emo_cfg()), ("emo_full", dict(EMO_CFG))])
def test_engine_emovec_vs_golden_and_merge(engine, name, cfg):
    """tf32 GEMMs (default): emo_vec within 2e-2 of the reference golden on values of std ~1;
    strict fp32 back end within 2e-3."""
    g = np.load(os.path.join(GOLD, name + ".npz"))
    w = make_emo_weights(cfg, seed=int(g["seed"]))
    engine.load_state_dict("gpt.", w)
    engine.emo_init(cfg)
    ev = engine.merge_emovec(g["feats"])
    err = np.abs(ev - g["emovec"]).max()
    print(f"{name}: emovec max err (tf32) {err:.2e}, ref std {g['emovec'].std():.2f}")
    assert err < 2e-2
    engine.set_option("gemm_backend", 1)
    try:
        ev32 = engine.merge_emovec(g["feats"])
    finally:
        engine.set_option("gemm_backend", 0)
    err32 = np.abs(ev32 - g["emovec"]).max()
    print(f"{name}: emovec max err (fp32) {err32:.2e}")
    assert err32 < 2e-3
    # merge with a different emotion reference and alpha (model_v2.py:837)
    gen = torch.Generator().manual_seed(4)
    emo_feats = torch.randn(g["feats"].shape[0] + 9, cfg["idim"], generator=gen)
    ref = merge_emovec(w, cfg, torch.from_numpy(g["feats"]), emo_feats, alpha=0.6).numpy()
    got = engine.merge_emovec(g["feats"], emo_feats.numpy(), alpha=0.6)
    assert np.abs(got - ref).max() < 2e-2


REF_WRAPPER_GOLD = os.path.join(GOLD, "gpt_ref_wrapper.npz")


def _ref_emo_feats(g):
    ge = torch.Generator().manual_seed(int(g["emo_feats_seed"]))
    return torch.randn(1, 23, 1024, generator=ge)[0], torch.randn(1, 31, 1024, generator=ge)[0]


REF_ECFG = dict(idim=1024, odim=32, linear_units=48, heads=2, blocks=1, cnn_kernel=15, p_dim=1024, p_heads=2, p_dim_head=64,
                p_depth=2, p_ff_mult=2, model_dim=256)


def test_oracle_merge_emovec_vs_reference_wrapper_golden():
    """`UnifiedVoice.merge_emovec` of the reference itself (model_v2.py:827-838 through get_emo_conditioning :588-593),
    run by oracle/make_goldens_gpt_ref.py with these seeded weights."""
    g = np.load(REF_WRAPPER_GOLD)
    w = make_emo_weights(REF_ECFG, seed=int(g["emo_seed"]))
    spk_f, emo_f = _ref_emo_feats(g)
    ev = merge_emovec(w, REF_ECFG, spk_f, emo_f, 0.6).numpy()
    assert np.abs(ev - g["emo_vec"]).max() < 1e-5


@pytest.mark.gpu
def test_engine_merge_emovec_vs_reference_wrapper_golden(engine):
    g = np.load(REF_WRAPPER_GOLD)
    w = make_emo_weights(REF_ECFG, seed=int(g["emo_seed"]))
    engine.load_state_dict("gpt.", w)
    engine.emo_init(REF_ECFG)
    spk_f, emo_f = (t.numpy() for t in _ref_emo_feats(g))
    engine.set_option("gemm_backend", 1)
    try:
        ev32 = engine.merge_emovec(spk_f, emo_f, alpha=0.6)
    finally:
        engine.set_option("gemm_backend", 0)
    ev = engine.merge_emovec(spk_f, emo_f, alpha=0.6)
    e32, e = float(np.abs(ev32 - g["emo_vec"]).max()), float(np.abs(ev - g["emo_vec"]).max())
    print(f"merge_emovec vs the reference wrapper: fp32 back end {e32:.2e}, tf32 {e:.2e}")
    assert e32 < 2e-3 and e < 2e-2
