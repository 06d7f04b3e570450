"""GPU parity tests of the fused GPT decode path (through the C-ABI) against the CPU oracle and
the golden vectors minted from stock transformers.GPT2Model.

Tolerances (bf16 path): logits are bf16 values (ulp 2^-6 = 0.0156 at |x| in [2,4), 0.031 in
[4,8), 0.0625 in [8,16)); the reference path itself is only defined up to its rounding noise
(HF autocast vs HF fp32 on the 2-layer golden case: rms 0.0185 at logit std 4.1, see
oracle/validate_gpt_vs_hf.py; the 24-layer geometry accumulates ~1.5x that).  Under teacher
forcing the engine must agree with the oracle per step to rms <= 0.035 and max-abs <= 0.16
(4.5 sigma of that noise over 8194 logits x 48 steps, plus the final bf16 quantisation of a logit
of magnitude up to 16) and its greedy pick must equal the oracle's except at near-ties
(processed-score gap <= 0.13 = 2 bf16 ulps at |logit| in [8,16))."""
import os

import numpy as np
import pytest
import torch

from tests.gpt_common import (GptOracle, check_teacher_forced, gpt_config, load_gpt,
                              make_gpt_weights, prepare_gpt_inputs, r16)
from oracle.validate_gpt_vs_hf import small_case

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "gpt_small.npz")
TOL = dict(max_abs=0.16, max_rms=0.035, tie_tol=0.13)


def test_prepare_inputs_matches_oracle(engine):
    cfg, style, emo, text = small_case()
    w = make_gpt_weights(cfg, seed=1234, bf16=True)
    load_gpt(engine, cfg, w)
    ref = prepare_gpt_inputs(w, style, r16(emo), text, lang=1, bf16=True).numpy()
    got = engine.gpt_prepare_inputs(style.numpy(), r16(emo).numpy(), text.numpy(), 1)
    assert got.shape == ref.shape
    # rows >= 1 are pure gathers + bf16 adds: bit exact; row 0 has a 192-term dot product
    assert np.array_equal(got[1:], ref[1:])
    assert np.abs(got[0] - ref[0]).max() <= 2.0 ** -6


def test_small_bf16_greedy_vs_hf_golden(engine):
    g = np.load(GOLD)
    cfg, style, emo, text = small_case()
    w = make_gpt_weights(cfg, seed=int(g["weight_seed"]), bf16=True)
    load_gpt(engine, cfg, w)
    n = int(g["n_steps"])
    prompt = g["prompt_bf16"]
    o_codes, o_logits = g["bf16_codes"], g["bf16_logits"]
    (e_codes,), (e_logits,) = engine.gpt_generate([prompt], n, 10.0, forbid_stop_before=n,
                                                  forced_codes=[o_codes], return_logits=True)
    ties = check_teacher_forced(cfg, o_codes, o_logits, e_codes, e_logits, 10.0, n, **TOL)
    # free running: identical tokens up to the first near-tie
    (f_codes,) = engine.gpt_generate([prompt], n, 10.0, forbid_stop_before=n)
    if ties == 0:
        assert np.array_equal(f_codes, o_codes)
    # and the engine is inside the bf16 noise of the real HF autocast path as well
    d = e_logits - g["hf_autocast_logits"]
    assert np.sqrt((d ** 2).mean()) < 0.035


def test_batched_ragged_prompts_equal_single(engine):
    """Mirror of the reference's only token-level check (tests/padding_test.py:83-108): the same
    utterance decoded alone, and inside a batch of ragged prompts, yields the same tokens."""
    cfg, style, emo, _ = small_case()
    w = make_gpt_weights(cfg, seed=99, bf16=True)
    load_gpt(engine, cfg, w, max_batch=4)
    g = torch.Generator().manual_seed(5)
    prompts = []
    for n_text in (3, 9, 17):
        text = torch.randint(2, 100, (n_text,), generator=g)
        prompts.append(prepare_gpt_inputs(w, style, r16(emo), text, lang=2, bf16=True).numpy())
    n = 16
    singles = [engine.gpt_generate([p], n, 10.0, forbid_stop_before=n, return_logits=True) for p in prompts]
    codes_b, logits_b = engine.gpt_generate(prompts, n, 10.0, forbid_stop_before=n, return_logits=True,
                                            forced_codes=[s[0][0] for s in singles])
    for i in range(3):
        sc, sl = singles[i][0][0], singles[i][1][0]
        check_teacher_forced(cfg, sc, sl, codes_b[i], logits_b[i], 10.0, n, **TOL)


def test_stop_token_and_lengths(engine):
    cfg, style, emo, text = small_case()
    w = make_gpt_weights(cfg, seed=5, bf16=True)
    w["mel_head.bias"] = w["mel_head.bias"].clone()
    w["mel_head.bias"][cfg["stop_mel_token"]] += 100.0
    load_gpt(engine, cfg, w)
    prompt = prepare_gpt_inputs(w, style, r16(emo), text, lang=0, bf16=True).numpy()
    (codes,) = engine.gpt_generate([prompt], 40, 10.0, forbid_stop_before=3)
    assert len(codes) == 4 and codes[-1] == cfg["stop_mel_token"]
    o_codes, _ = GptOracle(cfg, w, bf16=True).generate(prompt, 40, 10.0, 3)
    assert len(o_codes) == 4
    # max_new_tokens bound
    (codes,) = engine.gpt_generate([prompt], 5, 10.0, forbid_stop_before=100)
    assert len(codes) == 5


def test_full_size_v25_decode_vs_oracle(engine):
    """IndexTTS-2.5 geometry [ASSUMED 24 x 1280 x 20 heads, V=8194]: 48 greedy steps, S=37."""
    cfg = gpt_config()
    w = make_gpt_weights(cfg, seed=2025, bf16=True)
    load_gpt(engine, cfg, w, max_prompt=64)
    g = torch.Generator().manual_seed(11)
    style = torch.randn(192, generator=g)
    emo = r16(torch.randn(cfg["model_dim"], generator=g) * 0.5)
    text = torch.randint(2, 12000, (32,), generator=g)
    prompt = prepare_gpt_inputs(w, style, emo, text, lang=1, bf16=True).numpy()
    n = 48
    o_codes, o_logits = GptOracle(cfg, w, bf16=True).generate(prompt, n, 10.0, n)
    (e_codes,), (e_logits,) = engine.gpt_generate([prompt], n, 10.0, forbid_stop_before=n,
                                                  forced_codes=[o_codes], return_logits=True)
    ties = check_teacher_forced(cfg, o_codes, o_logits, e_codes, e_logits, 10.0, n, **TOL)
    (f_codes,) = engine.gpt_generate([prompt], n, 10.0, forbid_stop_before=n)
    agree = int((f_codes == o_codes).sum())
    print(f"full-size: teacher-forced near-tie disagreements {ties}/{n}; free-run agreement {agree}/{n}; "
          f"timing {engine.gpt_last_timing()}")
    if ties == 0:
        assert np.array_equal(f_codes, o_codes)
    # the batch-1 kernel's data-flow hand-overs between phases are race-free: repeated runs are bit-identical, and
    # gpt_fused_kernel (grid barriers between phases; IDX_GPT_V2=0 at init), teacher-forced on the same codes,
    # agrees within the bf16 noise of the path
    n2 = 96
    (r1,), (l1,) = engine.gpt_generate([prompt], n2, 10.0, forbid_stop_before=n2, return_logits=True)
    (r2,), (l2,) = engine.gpt_generate([prompt], n2, 10.0, forbid_stop_before=n2, return_logits=True)
    assert np.array_equal(r1, r2) and np.array_equal(l1, l2)
    os.environ["IDX_GPT_V2"] = "0"
    try:
        load_gpt(engine, cfg, w, max_prompt=64)
        (_,), (lb,) = engine.gpt_generate([prompt], n2, 10.0, forbid_stop_before=n2, forced_codes=[r1], return_logits=True)
    finally:
        del os.environ["IDX_GPT_V2"]
        load_gpt(engine, cfg, w, max_prompt=64)
    d = np.abs(lb - l1)
    print(f"gpt_decode1 vs gpt_fused_kernel over {n2} steps: max |dlogit| {d.max():.3f}, rms {np.sqrt((d ** 2).mean()):.4f}")
    assert d.max() <= TOL["max_abs"] and np.sqrt((d.astype(np.float64) ** 2).mean()) <= TOL["max_rms"]


def test_device_sampler_vs_oracle(engine):
    """do_sample=True, num_beams=1 (temperature → top-k → top-p → multinomial, HF warper order): the device
    sampler uses a documented Philox stream; with the same seed the oracle reproduces its picks except where a
    bf16-level logit difference moves a CDF boundary (teacher-forced, >= 90 % identical), every pick lies in
    the oracle's kept set, top_k=1 is greedy, and the stream is deterministic per seed."""
    cfg, style, emo, text = small_case()
    w = make_gpt_weights(cfg, seed=1234, bf16=True)
    load_gpt(engine, cfg, w)
    prompt = prepare_gpt_inputs(w, style, r16(emo), text, lang=1, bf16=True).numpy()
    n = 40
    kw = dict(do_sample=True, top_k=30, top_p=0.8, temperature=0.8, seed=2024)
    o_codes, o_logits = GptOracle(cfg, w, bf16=True).generate(prompt, n, 10.0, n, **kw)
    (e_codes,) = engine.gpt_generate([prompt], n, 10.0, forbid_stop_before=n, forced_codes=[o_codes], **kw)
    agree = int((e_codes == o_codes).sum())
    print(f"sampler: {agree}/{n} identical picks under teacher forcing")
    assert agree >= int(0.9 * n)
    (a,) = engine.gpt_generate([prompt], n, 10.0, forbid_stop_before=n, **kw)
    (b,) = engine.gpt_generate([prompt], n, 10.0, forbid_stop_before=n, **kw)
    assert np.array_equal(a, b)
    (c,) = engine.gpt_generate([prompt], n, 10.0, forbid_stop_before=n, **dict(kw, seed=99))
    assert not np.array_equal(a, c)
    (g1,) = engine.gpt_generate([prompt], n, 10.0, forbid_stop_before=n, do_sample=True, top_k=1, seed=5)
    (g0,) = engine.gpt_generate([prompt], n, 10.0, forbid_stop_before=n)
    assert np.array_equal(g1, g0)


def test_strict_fp32_small_vs_oracle(engine):
    """weights_bf16=False: the reference's default fp32 arithmetic (infer_v2_5.py:77 `use_bf16=False`) through the
    per-op fp32 kernels.  Teacher-forced logits within 1e-4 of the fp32 oracle (SURVEY section 8c tolerance) and the
    free-running greedy tokens identical."""
    cfg, style, emo, text = small_case()
    w = make_gpt_weights(cfg, seed=1234, bf16=False)
    load_gpt(engine, cfg, w, max_batch=2, bf16=False)
    prompt = prepare_gpt_inputs(w, style, emo, text, lang=1, bf16=False).numpy()
    got_prompt = engine.gpt_prepare_inputs(style.numpy(), emo.numpy(), text.numpy(), 1)
    assert np.abs(got_prompt - prompt).max() <= 1e-5
    n = 32
    o_codes, o_logits = GptOracle(cfg, w, bf16=False).generate(prompt, n, 10.0, n)
    (e_codes,), (e_logits,) = engine.gpt_generate([prompt], n, 10.0, forbid_stop_before=n,
                                                  forced_codes=[o_codes], return_logits=True)
    err = float(np.abs(e_logits - o_logits).max())
    print(f"strict fp32 small: max |logit err| {err:.2e} at logit std {o_logits.std():.2f}")
    assert err <= 1e-4
    assert np.array_equal(e_codes, o_codes)
    (f_codes,) = engine.gpt_generate([prompt], n, 10.0, forbid_stop_before=n)
    assert np.array_equal(f_codes, o_codes)
    # stop handling and sampling run through the same contract as the fused path
    (s1,) = engine.gpt_generate([prompt], n, 10.0, forbid_stop_before=n, do_sample=True, top_k=1, seed=3)
    assert np.array_equal(s1, o_codes)
    two = engine.gpt_generate([prompt, prompt[:-2]], 6, 10.0, forbid_stop_before=6)
    assert np.array_equal(two[0], o_codes[:6]) and len(two[1]) == 6


def test_strict_fp32_full_size_256_tokens_token_for_token(engine):
    """BASELINE configs[1]: IndexTTS-2.5 geometry, S = 37 prompt rows, 256 greedy speech tokens, fp32 — the engine's
    free-running tokens equal the fp32 oracle's token for token (north-star parity statement)."""
    cfg = gpt_config()
    w = make_gpt_weights(cfg, seed=2025, bf16=False)
    load_gpt(engine, cfg, w, max_prompt=64, bf16=False)
    g = torch.Generator().manual_seed(11)
    style = torch.randn(192, generator=g)
    emo = torch.randn(cfg["model_dim"], generator=g) * 0.5
    text = torch.randint(2, 12000, (32,), generator=g)
    prompt = prepare_gpt_inputs(w, style, emo, text, lang=1, bf16=False).numpy()
    n = 256
    o_codes, o_logits = GptOracle(cfg, w, bf16=False).generate(prompt, n, 10.0, n)
    (e_codes,), (e_logits,) = engine.gpt_generate([prompt], n, 10.0, forbid_stop_before=n, return_logits=True)
    agree = int((e_codes == o_codes).sum())
    err = float(np.abs(e_logits - o_logits).max()) if agree == n else float("nan")
    print(f"strict fp32 full size: {agree}/{n} tokens identical, max |logit err| {err:.2e}, timing {engine.gpt_last_timing()}")
    assert np.array_equal(e_codes, o_codes)
    assert err <= 5e-4


def _beam_params(cfg, **kw):
    p = dict(num_beams=3, start=cfg["start_mel_token"], stop=cfg["stop_mel_token"], repetition_penalty=10.0,
             temperature=0.8, top_k=30, top_p=0.8, length_penalty=0.0, seed=7, forbid_stop_before=0, do_sample=True)
    p.update(kw)
    return p


def _check_beam_run(engine, cfg, prompt, n, p, utt=0, codes=None, lg=None):
    """Replay the logits the engine's beams saw through the oracle's beam-sample logic: every (parent, token) choice,
    the running scores, the termination step and the returned hypothesis must be identical."""
    from oracle import beam
    par, tok, sc, fs = engine.gpt_beam_trace(utt, num_beams=p["num_beams"])
    rep = beam.run_beam(lambda k, pa, tk: lg[k], p, n, utt=utt)
    # the host polls the done flags every 8 steps: after the scorer is done the engine may run a few pad steps
    assert rep["steps"] <= len(par) < rep["steps"] + 8 or len(par) == n, (rep["steps"], len(par))
    for k, (bp, bt, bs) in enumerate(rep["trace"]):
        assert bp == par[k].tolist() and bt == tok[k].tolist(), (k, bp, par[k], bt, tok[k])
        assert np.allclose(bs, sc[k], rtol=0, atol=2e-4), (k, bs, sc[k])
    assert rep["codes"].tolist() == codes.tolist()
    assert abs(rep["score"] - fs) <= 2e-4
    return par, tok


def test_beam_sample_default_mode_vs_oracle(engine):
    """num_beams=3, do_sample=True — the `.infer()` default (transformers_generation_utils.py:3325-3609).  The engine
    dumps the raw logits of every beam row at every step; (1) the oracle's restatement of log_softmax → processors →
    joint multinomial → BeamSearchScorer, fed with those logits and the same Philox stream, reproduces every choice;
    (2) the logits along the winning lineage equal the model's teacher-forced logits for that token sequence, i.e. the
    KV-cache lineage map (instead of HF's index_select) is right."""
    cfg, style, emo, text = small_case()
    w = make_gpt_weights(cfg, seed=1234, bf16=True)
    load_gpt(engine, cfg, w, max_batch=8)
    prompt = prepare_gpt_inputs(w, style, r16(emo), text, lang=1, bf16=True).numpy()
    n = 28
    p = _beam_params(cfg)
    kw = dict(do_sample=True, num_beams=3, top_k=30, top_p=0.8, temperature=0.8, seed=7, length_penalty=0.0)
    (codes,), (lg,) = engine.gpt_generate([prompt], n, 10.0, return_logits=True, **kw)
    par, tok = _check_beam_run(engine, cfg, prompt, n, p, 0, codes, lg)
    # lineage of final beam 0
    K = min(len(par), len(codes))
    i = 0
    toks, rows = [0] * K, [0] * K
    for k in range(K - 1, -1, -1):
        toks[k], rows[k] = int(tok[k][i]), int(par[k][i])
        i = rows[k]
    (tf_codes,), (tf_logits,) = engine.gpt_generate([prompt], K, 10.0, forbid_stop_before=K, forced_codes=[np.array(toks, np.int32)],
                                                     return_logits=True)
    err = max(float(np.abs(lg[k][rows[k]] - tf_logits[k]).max()) for k in range(K))
    print(f"beam-sample: {K} steps, returned {len(codes)} codes, lineage logits max err vs teacher-forced {err:.3f}")
    assert err <= 0.13
    # deterministic per seed; another seed explores differently
    (again,) = engine.gpt_generate([prompt], n, 10.0, **kw)
    assert np.array_equal(again, codes)
    engine.gpt_generate([prompt], n, 10.0, **dict(kw, seed=8))
    _, tok8, _, _ = engine.gpt_beam_trace(0, num_beams=3)
    assert not np.array_equal(tok8, tok)          # (the best hypothesis may well coincide; the explored beams do not)


def test_beam_search_variants_and_batch(engine):
    """Plain beam search (do_sample=False: topk of the union), length_penalty, two utterances in one call (rows 0-2 and
    3-5, ragged prompts) — each replayed through the oracle logic."""
    cfg, style, emo, text = small_case()
    w = make_gpt_weights(cfg, seed=1234, bf16=True)
    load_gpt(engine, cfg, w, max_batch=8)
    p0 = prepare_gpt_inputs(w, style, r16(emo), text, lang=1, bf16=True).numpy()
    p1 = prepare_gpt_inputs(w, style * 0.5, r16(emo), text[:-3], lang=0, bf16=True).numpy()
    n = 16
    (c,), (lg,) = engine.gpt_generate([p0], n, 10.0, return_logits=True, do_sample=False, num_beams=3, length_penalty=1.0)
    _check_beam_run(engine, cfg, p0, n, _beam_params(cfg, do_sample=False, length_penalty=1.0), 0, c, lg)
    (c2,), (lg2,) = engine.gpt_generate([p0], n, 10.0, return_logits=True, do_sample=True, num_beams=2, top_k=5, top_p=0.9,
                                        temperature=1.2, seed=3)
    _check_beam_run(engine, cfg, p0, n, _beam_params(cfg, num_beams=2, top_k=5, top_p=0.9, temperature=1.2, seed=3), 0, c2, lg2)
    kw = dict(do_sample=True, num_beams=3, top_k=30, top_p=0.8, temperature=0.8, seed=21)
    cs, lgs = engine.gpt_generate([p0, p1], n, 10.0, return_logits=True, **kw)
    for u, pr in enumerate([p0, p1]):
        _check_beam_run(engine, cfg, pr, n, _beam_params(cfg, seed=21), u, cs[u], lgs[u])
    # early termination: a stop token that is easy to sample ends hypotheses; the result still replays exactly
    # (top_k = 100 is the webui's maximum: more than the 64 candidate slots of round 1)
    (c3,), (lg3,) = engine.gpt_generate([p0], 40, 1.0, return_logits=True, do_sample=True, num_beams=3, top_k=100, top_p=1.0,
                                        temperature=3.0, seed=5)
    _check_beam_run(engine, cfg, p0, 40, _beam_params(cfg, repetition_penalty=1.0, top_k=100, top_p=1.0, temperature=3.0, seed=5),
                    0, c3, lg3)
    # HF semantics are kept exactly or refused, never silently capped
    for bad in (0, 129):
        with pytest.raises(RuntimeError, match="top_k"):
            engine.gpt_generate([p0], 4, 1.0, do_sample=True, num_beams=3, top_k=bad, seed=1)
        with pytest.raises(RuntimeError, match="top_k"):
            engine.gpt_generate([p0], 4, 1.0, do_sample=True, top_k=bad, seed=1)


def test_strict_fp32_engine_vs_reference_unifiedvoice_golden(engine):
    """The CUDA path (strict fp32) against outputs of the reference's own `UnifiedVoice.inference_speech`
    (tests/golden/gpt_ref_wrapper.npz, oracle/make_goldens_gpt_ref.py): prompt assembly, 24 greedy tokens, logits."""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "gpt_ref_wrapper.npz"))
    cfg, _, _, _ = small_case()
    cfg = dict(cfg, n_langs=106)
    w = make_gpt_weights(cfg, seed=int(g["seed"]), bf16=False)
    load_gpt(engine, cfg, w, bf16=False)
    prompt = engine.gpt_prepare_inputs(g["style"], g["emo"], g["text"], int(g["lang"]))
    assert prompt.shape == g["prompt"].shape and np.abs(prompt - g["prompt"]).max() <= 1e-5
    n = int(g["n_steps"])
    (codes,), (logits,) = engine.gpt_generate([prompt], n, 10.0, return_logits=True)
    assert codes.tolist() == g["greedy_codes"][: len(codes)].tolist()
    err = float(np.abs(logits - g["greedy_logits"][: len(codes)]).max())
    print(f"strict fp32 engine vs reference UnifiedVoice: {len(codes)} tokens identical, max |logit diff| {err:.2e}")
    assert err <= 1e-4
