"""GPU: beam search (plain and beam-sample) on the strict fp32 GPT path (weights_bf16 = 0), the decode IndexTTS v1 / v1.5
`.infer()` asks for by default (num_beams=3, do_sample=True, top_k=30, top_p=0.8).

* Every run is replayed step by step through oracle/beam.py from the logits the engine's beam rows saw: each step's
  (parent, token, score), the termination step and the returned hypothesis.
* Numerics contract: a beam row computes exactly what the one-sequence strict path computes for that row's token history.
  Each final beam's lineage is rebuilt from the trace and teacher-forced through the one-row path (forced_codes); the beam
  row's logits must be bitwise equal to the forced run's at every step.  At the v1.5 geometry the lineage is also held to
  the fp32 oracle (the strict path's 5e-4 bound).
* Early termination (a raised stop-token bias): finished hypotheses, the scorer's done flag, the pad steps after it.
* The no-cache position rule (mel_pos_mode = 1 on W is mode 0 on the shifted table W'), two requests in one call, the
  refusals, and the drop-in `attach_v1` called with the kwargs infer.py passes.
The lineage check fails for each of these planted faults: a generated key read from the row's own slot instead of its
lineage slot, k / v written one position early (plen + k - 1), and rows >= 1 accumulating in another order."""
import types

import numpy as np
import pytest
import torch

from indextts_b200 import synth
from indextts_b200.dropin import attach_v1
from oracle import v1
from oracle.gpt import GptOracle
from tests.test_gpt_gpu import _beam_params, _check_beam_run
from tests.test_v1_full_gpu import (MAX_PROMPT, _check_pos_rule, _init, _set_pos, _shifted, small_v1,  # noqa: F401
                                    v15_gpt)

pytestmark = pytest.mark.gpu

REP = 10.0


def _run(engine, prompts, n, m, mode, do_sample=True, lp=0.0, seed=7, top_k=30, top_p=0.8, temperature=0.8):
    kw = dict(num_beams=m, do_sample=do_sample, top_k=top_k, top_p=top_p, temperature=temperature, length_penalty=lp,
              seed=seed, mel_pos_mode=mode, return_logits=True)
    return engine.gpt_generate(prompts, n, REP, **kw)


def _lineages(par, tok, K):
    """For every final beam: (tokens, rows) with rows[k] = the beam row whose logits chose tokens[k] at step k."""
    out = []
    for i0 in range(par.shape[1]):
        i, toks, rows = i0, [0] * K, [0] * K
        for k in range(K - 1, -1, -1):
            toks[k], rows[k] = int(tok[k][i]), int(par[k][i])
            i = rows[k]
        out.append((toks, rows))
    return out


def _check_lineages_bitwise(engine, prompt, par, tok, lg, K, mode):
    """Each final beam's lineage, teacher-forced through the one-row strict path: bitwise equal logits at every step."""
    for b, (toks, rows) in enumerate(_lineages(par, tok, K)):
        (_,), (tf,) = engine.gpt_generate([prompt], K, REP, forbid_stop_before=K, forced_codes=[np.array(toks, np.int32)],
                                          return_logits=True, mel_pos_mode=mode)
        assert tf.shape[0] == K
        for k in range(K):
            assert np.array_equal(lg[k][rows[k]].view(np.uint32), tf[k].view(np.uint32)), (b, k)
    return _lineages(par, tok, K)


def _replay_steps(engine, cfg, p, n, utt, codes, lg):
    from oracle import beam
    par, tok = _check_beam_run(engine, cfg, None, n, p, utt, codes, lg)
    steps = beam.run_beam(lambda k, pa, tk: lg[k], p, n, utt=utt)["steps"]
    return par, tok, steps


@pytest.mark.parametrize("m", [2, 3, 4])
@pytest.mark.parametrize("do_sample", [True, False], ids=["sample", "plain"])
@pytest.mark.parametrize("lp", [0.0, 1.0])
@pytest.mark.parametrize("mode", [0, 1])
def test_strict_beams_small_replay_and_lineage(engine, small_v1, m, do_sample, lp, mode):
    cfg, w, prompts = small_v1
    engine.load_state_dict("gpt.", w)
    _init(engine, cfg, False, 128, 4)
    n = 24
    (codes,), (lg,) = _run(engine, prompts[:1], n, m, mode, do_sample, lp)
    assert lg.shape[1:] == (m, cfg["number_mel_codes"])
    p = _beam_params(cfg, num_beams=m, do_sample=do_sample, length_penalty=lp)
    par, tok, K = _replay_steps(engine, cfg, p, n, 0, codes, lg)
    _check_lineages_bitwise(engine, prompts[0], par, tok, lg, K, mode)
    print(f"strict beams m={m} {'sample' if do_sample else 'plain'} lp={lp} mode={mode}: {K} steps replayed, "
          f"{len(codes)} codes returned, {m} lineages bitwise equal to the one-row path")


def _stop_biased(w, cfg, bias=9.0):
    """mel_head.bias[stop] raised: hypotheses finish well before max_new and the scorer ends the search early."""
    w = dict(w)
    w["mel_head.bias"] = w["mel_head.bias"].clone()
    w["mel_head.bias"][cfg["stop_mel_token"]] += bias
    return w


@pytest.mark.parametrize("m,do_sample", [(3, True), (2, False)], ids=["sample-3", "plain-2"])
@pytest.mark.parametrize("mode", [0, 1])
def test_strict_beams_small_early_termination(engine, small_v1, m, do_sample, mode):
    """Finished hypotheses, the done flag, the identity-reorder pad steps after it and finalize with a finished best
    hypothesis: the termination step and the returned hypothesis replay exactly, the lineages are bitwise the one-row
    path, and the logits dump holds every beam step the search ran (gpt_last_timing()["steps"])."""
    cfg, w, prompts = small_v1
    engine.load_state_dict("gpt.", _stop_biased(w, cfg))
    _init(engine, cfg, False, 128, 4)
    n = 48
    (codes,), (lg,) = _run(engine, prompts[:1], n, m, mode, do_sample)
    p = _beam_params(cfg, num_beams=m, do_sample=do_sample)
    par, tok, K = _replay_steps(engine, cfg, p, n, 0, codes, lg)
    steps = engine.gpt_last_timing()["steps"]
    assert K < n and steps == len(par) == lg.shape[0], (K, steps, len(par), lg.shape)
    assert codes[-1] == cfg["stop_mel_token"] and len(codes) <= K
    _check_lineages_bitwise(engine, prompts[0], par, tok, lg, K, mode)
    print(f"strict beams early stop m={m} {'sample' if do_sample else 'plain'} mode={mode}: done after {K} of {n} steps, "
          f"{steps} run, finished hypothesis of {len(codes)} codes")


def test_strict_beams_two_requests_stop_at_their_own_steps(engine, small_v1):
    """Two requests that end at different steps: each replays with its own step count, and each logits dump has as many
    rows as the longest search ran."""
    cfg, w, prompts = small_v1
    engine.load_state_dict("gpt.", _stop_biased(w, cfg))
    _init(engine, cfg, False, 128, 4)
    n = 48
    cs, lgs = _run(engine, prompts[:2], n, 3, 0)
    steps = engine.gpt_last_timing()["steps"]
    Ks, runs = [], []
    for u in range(2):
        par, tok, K = _replay_steps(engine, cfg, _beam_params(cfg), n, u, cs[u], lgs[u])
        _check_lineages_bitwise(engine, prompts[u], par, tok, lgs[u], K, 0)
        assert lgs[u].shape[0] == steps
        Ks.append(K)
        runs.append(len(par))
    assert max(runs) == steps and min(Ks) < n, (Ks, runs, steps)
    print(f"strict beams, two requests: done after {Ks} steps, {runs} run, dumps of {steps} rows")


def test_strict_beams_no_cache_rule_small(engine, small_v1):
    cfg, w, prompts = small_v1
    engine.load_state_dict("gpt.", w)
    _check_pos_rule(engine, cfg, w, prompts[:2], 40, False, 128, 4, {}, 3, "strict beam search, 3 beams")


def test_strict_beams_two_requests_in_one_call(engine, small_v1):
    cfg, w, prompts = small_v1
    engine.load_state_dict("gpt.", w)
    _init(engine, cfg, False, 128, 4)
    n = 32
    cs, lgs = _run(engine, prompts[:2], n, 3, 1, seed=21)
    toks = []
    for u in range(2):
        par, tok, K = _replay_steps(engine, cfg, _beam_params(cfg, seed=21), n, u, cs[u], lgs[u])
        _check_lineages_bitwise(engine, prompts[u], par, tok, lgs[u], K, 1)
        toks.append(tok)
        print(f"strict beams, request {u} of 2: {K} steps replayed with utt = {u}")
    assert not np.array_equal(toks[0], toks[1][: len(toks[0])])
    # the second request's Philox stream is its global index: alone it is request 0 and explores other beams
    _run(engine, prompts[1:2], n, 3, 1, seed=21)
    _, alone, _, _ = engine.gpt_beam_trace(0, num_beams=3)
    assert not np.array_equal(alone, toks[1])


def test_strict_beams_refused_before_launch(engine, small_v1):
    cfg, w, prompts = small_v1
    engine.load_state_dict("gpt.", w)
    _init(engine, cfg, False, 128, 2)
    _run(engine, prompts[:1], 8, 2, 0)
    before = engine.gpt_last_timing()
    assert before["launches"] > 0
    with pytest.raises(RuntimeError, match="max_batch"):
        _run(engine, prompts[:1], 8, 3, 0)
    assert engine.gpt_last_timing() == before
    with pytest.raises(RuntimeError, match="forced_codes"):
        engine.gpt_generate(prompts[:1], 8, REP, num_beams=2, forced_codes=[np.zeros(8, np.int32)])
    assert engine.gpt_last_timing() == before


def test_strict_beams_v1_5_geometry_infer_defaults(engine, v15_gpt):
    """24 x 1280, V = 8194, a prompt from the engine's own v1_get_conditioning: three-beam beam-sample with the `.infer()`
    defaults, 64 steps, mel_pos_mode = 1 (no KV cache on the reference's side)."""
    cfg, w = v15_gpt
    engine.load_state_dict("gpt.", w)
    _init(engine, cfg, False, MAX_PROMPT, 4)
    engine.v1_cond_init(synth.V1_COND_CFG, 32)
    mel = torch.randn(200, 100, generator=torch.Generator().manual_seed(15)).numpy() * 1.5 - 4.0
    conds = engine.v1_get_conditioning(mel)
    text = torch.randint(2, 100, (30,), generator=torch.Generator().manual_seed(30))
    prompt = v1.prepare_inputs_v1(w, torch.as_tensor(conds), text).numpy()
    n = 64
    (codes,), (lg,) = _run(engine, [prompt], n, 3, 1, seed=1234, temperature=1.0)
    p = _beam_params(cfg, seed=1234, temperature=1.0)
    par, tok, K = _replay_steps(engine, cfg, p, n, 0, codes, lg)
    lines = _check_lineages_bitwise(engine, prompt, par, tok, lg, K, 1)
    gw = {k: v.cuda() for k, v in w.items() if not k.startswith(("conditioning_encoder.", "perceiver_encoder."))}
    gw["mel_pos_embedding.emb.weight"] = _shifted(w).cuda()
    orc = GptOracle(cfg, gw, bf16=False)
    worst = 0.0
    for toks, rows in lines:
        _, ol = orc.generate(prompt, K, REP, K, forced=toks)
        worst = max(worst, max(float(np.abs(lg[k][rows[k]] - ol[k]).max()) for k in range(K)))
    del gw, orc
    torch.cuda.empty_cache()
    print(f"strict beams v1.5 geometry: {K} steps replayed, {len(codes)} codes, 3 lineages bitwise equal to the one-row "
          f"path, max |logit - fp32 oracle| {worst:.2e}, timing {engine.gpt_last_timing()}")
    assert worst <= 5e-4


class _Mod:
    def __init__(self, sd, **attrs):
        self._sd = sd
        self.__dict__.update(attrs)

    def state_dict(self):
        return self._sd


def test_attach_v1_default_infer_kwargs_decode(engine):
    """`attach_v1` on seeded v1 stand-ins; `inference_speech` with exactly the kwargs infer.py passes by default, then with
    a right-padded two-text batch as infer_fast builds it (v1.5: stop_text_token padding).  Each row equals a direct engine
    call on that text with the seed the drop-in draws from torch's generator."""
    from oracle.validate_gpt_vs_hf import small_case
    cfg = small_case()[0]
    wg = synth.make_gpt_v1_weights(cfg, synth.small_v1_cond_cfg(cfg["model_dim"]), seed=321)
    h = synth.small_v1_config()
    wb = synth.make_bigvgan_v1_weights(h, seed=4321)
    tts = types.SimpleNamespace()
    tts.gpt = _Mod(wg, model_dim=cfg["model_dim"], heads=cfg["heads"], number_mel_codes=cfg["number_mel_codes"],
                   start_mel_token=cfg["start_mel_token"], stop_mel_token=cfg["stop_mel_token"],
                   max_mel_tokens=cfg["max_mel_tokens"], gpt=types.SimpleNamespace(h=[None] * cfg["layers"]),
                   inference_model=types.SimpleNamespace(kv_cache=False))
    tts.bigvgan = _Mod({k: v for k, v in wb.items() if v.is_floating_point()}, h=h)
    attach_v1(tts, engine=engine)
    mel = torch.randn(1, 100, 120, generator=torch.Generator().manual_seed(4)) * 1.5 - 4.0
    conds = engine.v1_get_conditioning(mel[0].t().contiguous().numpy())
    g = torch.Generator().manual_seed(9)
    texts = [torch.randint(2, 100, (n,), generator=g, dtype=torch.int32) for n in (11, 6)]
    n = 40
    defaults = dict(do_sample=True, top_p=0.8, top_k=30, temperature=1.0, num_return_sequences=1, length_penalty=0.0,
                    num_beams=3, repetition_penalty=10.0, max_generate_length=n)
    padded = torch.nn.utils.rnn.pad_sequence(texts, batch_first=True, padding_value=1, padding_side="right")
    for batch in (texts[0][None], padded):
        torch.manual_seed(77)
        got = tts.gpt.inference_speech(mel, batch, cond_mel_lengths=torch.tensor([mel.shape[-1]]), **defaults)
        torch.manual_seed(77)
        seeds = [int(torch.randint(0, 2 ** 31 - 1, (1,)).item()) for _ in range(batch.shape[0])]
        for i in range(batch.shape[0]):
            (want,) = engine.gpt_generate([engine.gpt_prepare_inputs_v1(conds, texts[i].numpy())], n, 10.0, do_sample=True,
                                          top_k=30, top_p=0.8, temperature=1.0, num_beams=3, length_penalty=0.0,
                                          seed=seeds[i], mel_pos_mode=1)
            row = got[i].cpu().numpy()
            assert row[: len(want)].tolist() == want.tolist(), i
            assert np.all(row[len(want):] == cfg["stop_mel_token"])
        print(f"attach_v1, infer() defaults, batch of {batch.shape[0]}: codes of lengths "
              f"{[int((r != cfg['stop_mel_token']).sum()) for r in got.cpu()]} equal the direct engine calls")
