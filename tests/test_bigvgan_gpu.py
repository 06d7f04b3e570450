"""GPU parity of the BigVGAN path (C-ABI) against goldens from the reference module and the CPU
oracle.  Tolerances: Activation1d <= 1e-5 max-abs (fp32, SURVEY §8c); waveform RMS error <= 1e-3
(north-star) with the default wgmma tf32 convolutions — measured value is printed; max-abs
<= 2e-2 guards against localised garbage; with the strict fp32 back end the error is ~1e-6."""
import os

import numpy as np
import pytest
import torch

from oracle.bigvgan import (BIGVGAN_V2_22K, activation1d, bigvgan_forward, kaiser_sinc_filter1d,
                            make_bigvgan_weights, small_config, synthetic_mel, wav_rms_err)

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def test_activation1d_kat_and_random(engine):
    g = np.load(os.path.join(GOLD, "activation1d_kat.npz"))
    y = engine.antialias_snake(g["x"], g["alpha"], g["beta"])
    assert np.abs(y - g["y"]).max() <= 1e-5
    yr = engine.antialias_snake(g["xr"], g["alpha_r"], g["beta_r"])
    assert np.abs(yr - g["yr"]).max() <= 1e-5


@pytest.mark.parametrize("B,C,T", [(1, 24, 1000), (2, 48, 333), (1, 96, 7), (3, 1536, 65), (1, 5, 1)])
def test_activation1d_shapes_vs_oracle(engine, B, C, T):
    g = torch.Generator().manual_seed(B * 1000 + C + T)
    x = torch.randn(B, C, T, generator=g) * 2.0
    alpha = torch.randn(C, generator=g) * 0.3
    beta = torch.randn(C, generator=g) * 0.3
    ref = activation1d(x, alpha, beta, kaiser_sinc_filter1d()).numpy()
    got = engine.antialias_snake(x.numpy(), alpha.numpy(), beta.numpy())
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() <= 2e-5


def _load(engine, h, seed):
    w = make_bigvgan_weights(h, seed=seed)
    engine.load_state_dict("bigvgan.", w)
    engine.bigvgan_init(h)
    return w


def test_small_generator_vs_reference_golden(engine):
    g = np.load(os.path.join(GOLD, "bigvgan_small.npz"))
    h = small_config()
    _load(engine, h, int(g["seed"]))
    wav = engine.bigvgan_forward(g["mel"])
    assert wav.shape == g["wav"].shape
    err = wav_rms_err(wav, g["wav"])
    print(f"small generator (tf32): rms err {err:.2e}, max abs {np.abs(wav - g['wav']).max():.2e}")
    assert err <= 1e-3 and np.abs(wav - g["wav"]).max() <= 2e-2
    engine.set_option("gemm_backend", 1)
    try:
        wav = engine.bigvgan_forward(g["mel"])
    finally:
        engine.set_option("gemm_backend", 0)
    err = wav_rms_err(wav, g["wav"])
    print(f"small generator (strict fp32): rms err {err:.2e}")
    assert err <= 1e-5


def test_full_generator_vs_reference_golden(engine):
    g = np.load(os.path.join(GOLD, "bigvgan_full_f12.npz"))
    h = dict(BIGVGAN_V2_22K)
    w = _load(engine, h, int(g["seed"]))
    wav = engine.bigvgan_forward(g["mel"])
    err = wav_rms_err(wav, g["wav"])
    print(f"full generator F=12: rms err {err:.2e}, max abs {np.abs(wav - g['wav']).max():.2e}, "
          f"device ms {engine.bigvgan_last_ms():.3f}")
    assert err <= 1e-3 and np.abs(wav - g["wav"]).max() <= 2e-2
    # longer, batched, ragged-free input against the CPU oracle (seconds on the host cores)
    mel = synthetic_mel(2, 48, seed=9)
    ref = bigvgan_forward(h, w, mel).numpy()
    wav = engine.bigvgan_forward(mel.numpy())
    err = wav_rms_err(wav, ref)
    print(f"full generator B=2 F=48: rms err {err:.2e}, device ms {engine.bigvgan_last_ms():.3f}")
    assert err <= 1e-3 and np.abs(wav - ref).max() <= 2e-2


def test_full_size_properties(engine):
    """Size-independent properties at a BASELINE-size input (F=880 = 256 tokens): output shape,
    finiteness, clamp range, batch independence and time-locality (receptive field) — a change in
    the last mel frames must not alter the early samples."""
    h = dict(BIGVGAN_V2_22K)
    _load(engine, h, 1234)
    mel = synthetic_mel(2, 880, seed=4).numpy()
    wav = engine.bigvgan_forward(mel)
    assert wav.shape == (2, 1, 880 * 256) and np.isfinite(wav).all()
    assert wav.min() >= -1.0 and wav.max() <= 1.0
    single = engine.bigvgan_forward(mel[1:2])
    assert np.abs(single[0] - wav[1]).max() <= 1e-5
    mel2 = mel.copy()
    mel2[:, :, -40:] += 0.5
    wav2 = engine.bigvgan_forward(mel2)
    assert np.array_equal(wav2[:, :, : 700 * 256], wav[:, :, : 700 * 256])
    assert np.abs(wav2[:, :, -20 * 256:] - wav[:, :, -20 * 256:]).max() > 1e-4
    print(f"full generator B=2 F=880: device ms {engine.bigvgan_last_ms():.2f}")
