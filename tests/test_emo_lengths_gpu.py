"""GPU: the prompt encoders end to end at real prompt lengths, against their oracles run in float64 on the GPU.

* `merge_emovec` at the full emotion config for feature lengths T on both sides of the points where the conformer's attention
  GEMMs move to the tensor cores (T2 = (T - 3) // 2 + 1 = 31 / 32 for the scores, 44 / 45 for P V), up to T = 750 (a 15 s
  prompt after the w2v-BERT front end, T2 = 374), on the default tf32 path and on the strict fp32 one.
* The merge itself: speaker and emotion features of different lengths in both orders (the second encoder pass re-uses the
  arena), alpha in {0, 0.6, 1} against the fp32 lerp of the two single-input vectors, bitwise repeatability.
* The v1 / v1.5 speaker conformer (SURVEY section 8: 512 dims, 2048 FF units, 8 heads, 6 blocks, 100 mels, 32 latents at
  p_dim = model_dim = 1280) up to T = 1406 mel frames (15 s at 24 kHz, hop 256).
* The v1 ECAPA-TDNN speaker embedding at 5 .. 9 frames (fewer than 8 rows per statistics thread row) and at 1406."""
import numpy as np
import pytest
import torch

from indextts_b200 import synth
from indextts_b200.synth import V1_COND_CFG
from oracle import v1
from oracle.emo import EMO_CFG, get_emovec, make_emo_weights

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
LENGTHS = [3, 4, 64, 65, 91, 129, 750]


def _on_gpu(w):
    return {k: v.double().cuda() for k, v in w.items()}


def _feats(T, seed, dim):
    return torch.randn(T, dim, generator=torch.Generator().manual_seed(seed))


@pytest.fixture(scope="module")
def emo_full(engine):
    cfg = dict(EMO_CFG)
    w = make_emo_weights(cfg, seed=777)
    engine.load_state_dict("gpt.", w)
    engine.emo_init(cfg)
    return cfg, _on_gpu(w)


def _strict(engine, fn):
    engine.set_option("gemm_backend", 1)
    try:
        return fn()
    finally:
        engine.set_option("gemm_backend", 0)


@pytest.mark.parametrize("T", LENGTHS)
def test_merge_emovec_at_prompt_lengths(engine, emo_full, T):
    cfg, wd = emo_full
    x = _feats(T, T, cfg["idim"])
    ref = get_emovec(wd, cfg, x.double().cuda()).cpu().numpy()
    got = engine.merge_emovec(x.numpy())
    got32 = _strict(engine, lambda: engine.merge_emovec(x.numpy()))
    e, e32 = float(np.abs(got - ref).max()), float(np.abs(got32 - ref).max())
    print(f"merge_emovec T={T} (T2={(T - 3) // 2 + 1}): max err tf32 {e:.2e}, fp32 {e32:.2e} (ref std {ref.std():.2f})")
    assert np.all(np.isfinite(got)) and np.all(np.isfinite(got32))
    assert e < 2e-2 and e32 < 2e-3


@pytest.mark.parametrize("Ts,Te", [(65, 750), (750, 65), (3, 129)])
def test_merge_semantics(engine, emo_full, Ts, Te):
    cfg, _ = emo_full
    spk, emo = _feats(Ts, 100 + Ts, cfg["idim"]).numpy(), _feats(Te, 200 + Te, cfg["idim"]).numpy()
    base, ev = engine.merge_emovec(spk), engine.merge_emovec(emo)
    first = {}
    for alpha in (0.0, 0.6, 1.0):
        got = engine.merge_emovec(spk, emo, alpha)
        a = float(np.float32(alpha))
        d = ev.astype(np.float64) - base
        want = base + a * d
        # lerp_kernel: base + alpha * (emo - base) in fp32, one rounding per operation
        bound = 2.001 * U * np.abs(a * d) + U * np.abs(want) + U * 2.001 * U * np.abs(a * d)
        err = np.abs(got - want)
        print(f"merge Ts={Ts} Te={Te} alpha={alpha}: max |merge - lerp| {err.max():.2e}, max err / bound "
              f"{(err / np.maximum(bound, 1e-45)).max():.3f}")
        assert np.all(err <= bound)
        if alpha == 0.0:
            assert np.array_equal(got.view(np.uint32), base.view(np.uint32))
        first[alpha] = got
    again = engine.merge_emovec(spk, emo, 0.6)
    assert np.array_equal(again.view(np.uint32), first[0.6].view(np.uint32))


@pytest.fixture(scope="module")
def v1_cond(engine):
    w = make_emo_weights(V1_COND_CFG, seed=4242, enc_prefix="conditioning_encoder.", per_prefix="perceiver_encoder.",
                         n_latents=32, heads_out=False)
    engine.load_state_dict("gpt.", w)
    engine.v1_cond_init(V1_COND_CFG, 32)
    return _on_gpu(w)


@pytest.mark.parametrize("T", [3, 61, 1406])
def test_v1_conditioning_at_prompt_lengths(engine, v1_cond, T):
    mel = _feats(T, 300 + T, V1_COND_CFG["idim"])
    ref = v1.get_conditioning_v1(v1_cond, V1_COND_CFG, mel.double().cuda()).cpu().numpy()
    got = engine.v1_get_conditioning(mel.numpy())
    got32 = _strict(engine, lambda: engine.v1_get_conditioning(mel.numpy()))
    e, e32 = float(np.abs(got - ref).max()), float(np.abs(got32 - ref).max())
    print(f"v1 get_conditioning T={T} (T2={(T - 3) // 2 + 1}): max err tf32 {e:.2e}, fp32 {e32:.2e} "
          f"(ref std {ref.std():.2f})")
    assert got.shape == (32, V1_COND_CFG["model_dim"])
    assert e < 2e-2 and e32 < 2e-3


@pytest.fixture(scope="module")
def v1_vocoder(engine):
    h = synth.small_v1_config()
    w = synth.make_bigvgan_v1_weights(h, seed=4321)
    engine.load_state_dict("bigvgan_v1.", {k: v for k, v in w.items() if v.is_floating_point()})
    engine.v1_vocoder_init(h)
    return h, _on_gpu({k: v for k, v in w.items() if k.startswith("speaker_encoder.")})


@pytest.mark.parametrize("Tm", [5, 6, 7, 8, 9, 1406])
def test_v1_speaker_embedding_at_prompt_lengths(engine, v1_vocoder, Tm):
    h, wd = v1_vocoder
    mel = _feats(Tm, 400 + Tm, h["num_mels"]) * 1.5 - 4.0
    ref = v1.ecapa_tdnn(wd, mel[None].double().cuda())[0, 0].cpu().numpy()
    scale = float(np.abs(ref).max())
    got = engine.v1_speaker_embedding(mel.numpy())
    got32 = _strict(engine, lambda: engine.v1_speaker_embedding(mel.numpy()))
    e, e32 = float(np.abs(got - ref).max()) / scale, float(np.abs(got32 - ref).max()) / scale
    print(f"ECAPA embedding Tm={Tm}: relative max err tf32 {e:.2e}, fp32 {e32:.2e}")
    assert e < 5e-3 and e32 < 1e-4
