"""CPU: the v1 / v1.5 vocoder-side restatement (oracle/v1.py: ECAPA-TDNN speaker encoder + latent-conditioned BigVGAN,
SURVEY section 8 row a13) against outputs of the reference's own `indextts.BigVGAN.models.BigVGAN`
(tests/golden/v1_vocoder_small.npz and, at the IndexTTS-1.5 geometry, v1_vocoder_full.npz; oracle/make_goldens_v1.py)
and of the v1 UnifiedVoice (v1_gpt_small.npz).  The CUDA side is checked against this restatement by tests/test_v1_gpu.py
and tests/test_v1_full_gpu.py."""
import os

import numpy as np
import torch

from indextts_b200 import synth
from oracle import v1

GOLD = os.path.join(os.path.dirname(__file__), "golden", "v1_vocoder_small.npz")


def test_ecapa_and_bigvgan_v1_match_reference_module():
    g = np.load(GOLD)
    h = synth.small_v1_config()
    w = synth.make_bigvgan_v1_weights(h, seed=int(g["seed"]))
    latent, mel_ref = torch.from_numpy(g["latent"]), torch.from_numpy(g["mel_ref"])
    spk = v1.ecapa_tdnn(w, mel_ref).numpy()
    assert spk.shape == g["spk"].shape == (1, 1, h["speaker_embedding_dim"])
    assert np.abs(spk - g["spk"]).max() <= 1e-4 * max(1.0, float(np.abs(g["spk"]).max()))
    wav = v1.bigvgan_v1_forward(h, w, latent, mel_ref).numpy()
    assert wav.shape == g["wav"].shape == (1, 1, latent.shape[1] * 8)
    assert np.abs(wav - g["wav"]).max() <= 1e-5
    assert np.abs(wav).max() <= 1.0                      # tanh output (models.py:247)
    # the speaker embedding really conditions the waveform
    wav2 = v1.bigvgan_v1_forward(h, w, latent, mel_ref.flip(1) * 0.5).numpy()
    assert np.abs(wav2 - wav).max() > 1e-3


def test_bigvgan_v1_5_geometry_matches_reference_module():
    """The real v1.5 generator (synth.v1_5_config: 1280 -> 1536 channels, six upsamples, x1024, kernels 3/7/11, speaker
    embedding folded in after conv_pre and after each upsample) on 4 latents and a 61-frame reference mel."""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "v1_vocoder_full.npz"))
    h = synth.v1_5_config()
    w = synth.make_bigvgan_v1_weights(h, seed=int(g["seed"]), post_gain=synth.V1_5_POST_GAIN)
    latent, mel_ref = torch.from_numpy(g["latent"]), torch.from_numpy(g["mel_ref"])
    assert latent.shape == (1, 4, 1280) and mel_ref.shape == (1, 61, 100)
    spk = v1.ecapa_tdnn(w, mel_ref).numpy()
    assert spk.shape == g["spk"].shape == (1, 1, 512)
    assert np.abs(spk - g["spk"]).max() <= 1e-4 * max(1.0, float(np.abs(g["spk"]).max()))
    wav = v1.bigvgan_v1_forward(h, w, latent, mel_ref).numpy()
    assert wav.shape == g["wav"].shape == (1, 1, 4 * 1024)
    assert np.abs(wav - g["wav"]).max() <= 1e-5
    assert np.abs(wav).max() < 1.0


def test_v1_gpt_side_matches_reference_unifiedvoice():
    """v1 UnifiedVoice (indextts/gpt/model.py) — 32-latent conformer-perceiver prompt, v1 prompt assembly, greedy decode
    without the KV cache (infer.py:101) and the latent pass for the vocoder — against outputs of the reference class
    (tests/golden/v1_gpt_small.npz, oracle/make_goldens_v1.py:main_gpt)."""
    from oracle.gpt import GptOracle
    from oracle.validate_gpt_vs_hf import small_case
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "v1_gpt_small.npz"))
    cfg, _, _, _ = small_case()
    ccfg = synth.small_v1_cond_cfg(cfg["model_dim"])
    w = synth.make_gpt_v1_weights(cfg, ccfg, seed=int(g["seed"]))
    mel, text = torch.from_numpy(g["mel"]), torch.from_numpy(g["text"])
    conds = v1.get_conditioning_v1(w, ccfg, mel[0].t())
    assert conds.shape == (32, cfg["model_dim"]) and np.abs(conds.numpy() - g["conds"]).max() < 2e-4
    prompt = v1.prepare_inputs_v1(w, conds, text)
    assert prompt.shape[0] == 32 + len(text) + 2
    n = len(g["codes"])
    codes, logits = v1.generate_v1(GptOracle(cfg, w, bf16=False), prompt, n, 10.0, kv_cache=False)
    assert codes.tolist() == g["codes"].tolist()
    assert np.abs(logits - g["logits"]).max() < 5e-4
    lat = v1.latents_v1(GptOracle(cfg, w, bf16=False), conds, text, codes[codes != cfg["stop_mel_token"]]).numpy()
    assert lat.shape == g["latents"].shape and np.abs(lat - g["latents"]).max() < 5e-4
    # the cached path sits one mel position later from step 1 on (trap P1): it is a different function
    c2, _ = v1.generate_v1(GptOracle(cfg, w, bf16=False), prompt, n, 10.0, kv_cache=True)
    assert c2[0] == codes[0]
