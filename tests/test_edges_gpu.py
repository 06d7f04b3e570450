"""GPU: edge cases of the path against the oracle — minimal and ragged sizes, limits, error behaviour.
(The reference's own tests only exercise whole-file outputs; these are the degenerate shapes its code paths accept:
one speech token, an empty text, a prompt of one mel frame, a single mel frame through the vocoder.)"""
import numpy as np
import pytest
import torch

from indextts_b200 import synth
from indextts_b200.engine import fold_weight_norm
from oracle import bigvgan as obv
from oracle.s2mel import cfm_inference, codec_decode, length_regulate
from oracle.s2mel import fold_weight_norm as oracle_fold
from oracle.validate_gpt_vs_hf import small_case
from tests.gpt_common import GptOracle, load_gpt, make_gpt_weights, prepare_gpt_inputs, r16

pytestmark = pytest.mark.gpu


def test_gpt_minimal_prompt_and_limits(engine):
    cfg, style, emo, text = small_case()
    w = make_gpt_weights(cfg, seed=1234, bf16=True)
    load_gpt(engine, cfg, w, max_batch=2)
    # empty text: prompt = [cond, 0, 0, start_text, stop_text] (model_v2.py:648-714)
    empty = torch.zeros(0, dtype=torch.long)
    ref = prepare_gpt_inputs(w, style, r16(emo), empty, lang=1, bf16=True).numpy()
    got = engine.gpt_prepare_inputs(style.numpy(), r16(emo).numpy(), empty.numpy(), 1)
    assert got.shape == ref.shape == (5, cfg["model_dim"]) and np.array_equal(got[1:], ref[1:])
    o_codes, _ = GptOracle(cfg, w, bf16=True).generate(ref, 6, 10.0, 6)
    (codes,) = engine.gpt_generate([got], 6, 10.0, forbid_stop_before=6)
    assert len(codes) == 6 and int((codes == o_codes).sum()) >= 5
    # a single new token
    (one,) = engine.gpt_generate([got], 1, 10.0, forbid_stop_before=1)
    assert one.tolist() == codes[:1].tolist()
    # limits are errors, not silent truncation: max_new_tokens beyond the mel position table, too many requests,
    # a prompt longer than max_prompt, an unsupported beam width
    with pytest.raises(RuntimeError):
        engine.gpt_generate([got], cfg["max_mel_positions"], 10.0)
    # more requests than max_batch run as consecutive decode groups: same tokens as one request at a time
    three = engine.gpt_generate([got, ref[:4], got], 6, 10.0, forbid_stop_before=6)
    (alone,) = engine.gpt_generate([ref[:4]], 6, 10.0, forbid_stop_before=6)
    assert np.array_equal(three[0], codes) and np.array_equal(three[2], codes) and np.array_equal(three[1], alone)
    # ... and the sampler's stream follows the request's global index, not its place in a group
    kw = dict(do_sample=True, top_k=20, top_p=0.9, temperature=1.3, seed=17, forbid_stop_before=6)
    grouped = engine.gpt_generate([got] * 5, 6, 10.0, **kw)
    load_gpt(engine, cfg, w, max_batch=8)
    whole = engine.gpt_generate([got] * 5, 6, 10.0, **kw)
    load_gpt(engine, cfg, w, max_batch=2)
    assert all(np.array_equal(a, b) for a, b in zip(grouped, whole))
    assert any(not np.array_equal(grouped[0], g) for g in grouped[1:])
    with pytest.raises(RuntimeError):
        engine.gpt_generate([np.zeros((129 + 64, cfg["model_dim"]), np.float32)], 4, 10.0)
    with pytest.raises(RuntimeError):
        engine.gpt_generate([got], 4, 10.0, num_beams=5, do_sample=True)
    with pytest.raises(RuntimeError, match="text token id"):
        engine.gpt_prepare_inputs(style.numpy(), r16(emo).numpy(), np.array([5, 10 ** 6], dtype=np.int32), 1)
    assert engine.gpt_prepare_inputs(style.numpy(), r16(emo).numpy(), empty.numpy(), 1).shape == (5, cfg["model_dim"])
    with pytest.raises(RuntimeError):          # 3 beams need 3 rows, max_batch is 2 here
        engine.gpt_generate([got], 4, 10.0, num_beams=3, do_sample=True)


def test_tail_minimal_sizes_vs_oracle(engine):
    c, cc, h = synth.small_s2mel_cfg(), synth.small_codec_cfg(), synth.small_config()
    ws, wc, wb = synth.make_s2mel_weights(c, 11), synth.make_codec_weights(cc, 12), synth.make_bigvgan_weights(h, 13)
    engine.load_state_dict("s2mel.", {k: v for k, v in fold_weight_norm(ws).items() if v.is_floating_point()})
    engine.load_state_dict("codec.", fold_weight_norm(wc))
    engine.load_state_dict("bigvgan.", wb)
    engine.s2mel_init(c); engine.codec_init(cc); engine.bigvgan_init(h)
    wsf, wcf = oracle_fold(ws), oracle_fold(wc)
    engine.set_option("gemm_backend", 1)          # strict fp32: the comparison is about shapes and borders
    try:
        # one speech token → 2 frames → ylen 3 → T = P + 3 with a one-frame prompt
        codes = np.array([5], dtype=np.int32)
        S = engine.codec_decode(codes)
        S_ref = codec_decode(wcf, torch.from_numpy(codes.astype(np.int64))[None])[0].numpy()
        assert S.shape == S_ref.shape == (2, S_ref.shape[1]) and np.abs(S - S_ref).max() < 1e-4
        lr_in = S[:, : c["lr_in"]] if S.shape[1] >= c["lr_in"] else np.pad(S, ((0, 0), (0, c["lr_in"] - S.shape[1])))
        cond = engine.length_regulate(lr_in, 3)
        cond_ref = length_regulate(wsf, torch.from_numpy(lr_in)[None], 3)[0].numpy()
        assert cond.shape == (3, cond_ref.shape[1]) and np.abs(cond - cond_ref).max() < 1e-4
        g = torch.Generator().manual_seed(3)
        P = 1
        pc = torch.randn(P, c["content_dim"], generator=g)
        ref_mel = torch.randn(80, P, generator=g) - 4.0
        sty = torch.randn(c["style_dim"], generator=g)
        mu = torch.cat([pc, torch.from_numpy(cond)], 0)
        z = torch.randn(80, mu.shape[0], generator=g)
        mel = engine.cfm_solve(mu.numpy(), ref_mel.numpy(), sty.numpy(), z.numpy(), 3, 0.7)
        mel_ref = cfm_inference(wsf, c, mu[None], torch.LongTensor([mu.shape[0]]), ref_mel[None], sty[None], z[None], 3, 0.7)[0].numpy()
        assert mel.shape == (80, 4) and np.abs(mel - mel_ref).max() < 1e-3 and np.all(mel[:, :P] == 0)
        # n_timesteps = 1: a single Euler step
        mel1 = engine.cfm_solve(mu.numpy(), ref_mel.numpy(), sty.numpy(), z.numpy(), 1, 0.7)
        mel1_ref = cfm_inference(wsf, c, mu[None], torch.LongTensor([mu.shape[0]]), ref_mel[None], sty[None], z[None], 1, 0.7)[0].numpy()
        assert np.abs(mel1 - mel1_ref).max() < 1e-3
        # a single mel frame through the vocoder; and a ragged batch dimension (B = 3)
        for B, F in ((1, 1), (3, 2)):
            m = synth.synthetic_mel(B, F, seed=B)
            wav = engine.bigvgan_forward(m.numpy())
            wav_ref = obv.bigvgan_forward(h, wb, m).numpy()
            assert wav.shape == wav_ref.shape and np.abs(wav - wav_ref).max() < 1e-4
    finally:
        engine.set_option("gemm_backend", 0)
    # argument errors surface as RuntimeError with a message (no silent fallback)
    with pytest.raises(RuntimeError):
        engine.cfm_solve(mu.numpy(), ref_mel.numpy(), sty.numpy(), z.numpy(), 0, 0.7)
    with pytest.raises(RuntimeError, match="inference_cfg_rate"):      # only the CFG pair path is built (infer_v2_5.py:831)
        engine.cfm_solve(mu.numpy(), ref_mel.numpy(), sty.numpy(), z.numpy(), 2, 0.0)
    with pytest.raises(RuntimeError, match="outside the codebook"):
        engine.codec_decode(np.array([3, cc["codebook_size"] + 7], dtype=np.int32))
    assert engine.codec_decode(np.array([3], dtype=np.int32)).shape[0] == 2      # the engine stays usable afterwards


@pytest.mark.parametrize("backend,tol", [(1, 1e-4), (0, 1e-2)])
def test_dit_forward_one_to_three_frames(engine, backend, tol):
    """1, 2 and 3 frames, where the WaveNet's reflect padding (encodec.py pad1d) zero-extends a 1- or 2-frame input
    before it reflects: the DiT against the oracle, and at 1 and 2 frames against the reference golden."""
    import os
    from oracle.s2mel import dit_forward, small_codec_cfg, small_s2mel_cfg
    from tests.test_s2mel_gpu import _load
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "s2mel_short.npz"))
    c = small_s2mel_cfg()
    w, _ = _load(engine, c, small_codec_cfg(), int(g["seed_s2mel"]), 4321)
    engine.set_option("gemm_backend", backend)
    try:
        rng = np.random.default_rng(12)
        for T in (1, 2, 3):
            if T < 3:
                mu, style, z, t = (g[f"dit{T}_{k}"] for k in ("mu", "style", "z", "t"))
            else:
                mu = rng.standard_normal((1, T, c["content_dim"])).astype(np.float32)
                style = rng.standard_normal((1, c["style_dim"])).astype(np.float32)
                z = rng.standard_normal((1, 80, T)).astype(np.float32)
                t = np.array([0.45], np.float32)
            px = np.zeros((1, 80, T), np.float32)
            d = engine.dit_forward(z, px, t, style, mu)
            ref = dit_forward(w, c, *(torch.from_numpy(a) for a in (z, px)), torch.LongTensor([T]),
                              torch.from_numpy(t), torch.from_numpy(style), torch.from_numpy(mu)).numpy()
            err = np.abs(d - ref).max()
            print(f"[backend {backend}] DiT T={T}: max err vs oracle {err:.2e}")
            assert np.all(np.isfinite(d)) and err < tol
            if T < 3:
                assert np.abs(d - g[f"dit{T}"]).max() < tol
    finally:
        engine.set_option("gemm_backend", 0)
