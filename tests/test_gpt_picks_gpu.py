"""Every GPT decode path's token pick, replayed in fp64 from the exact fp32 logits that path consumed.

The paths: gpt_decode1_kernel (one request), gpt_decode8_kernel (2-8 requests), gpt_fused_kernel at BT = 1 / 8
(IDX_GPT_V2=0 / IDX_GPT_V8=0 at init), the strict fp32 path (weights_bf16=False), and consecutive decode groups
(more requests than max_batch, so the Philox sequence index is the group base + row).  Each pick is checked against
tests/pick_refs.py with zero model noise: greedy picks exactly, sampled picks exactly except where a decision lies
within fp32 rounding of its boundary (counted, and bounded).  Rows of mel_head.weight set to zero with one bf16-exact
bias force exact logit ties on every path, whatever its accumulation order."""
import contextlib
import os

import numpy as np
import pytest
import torch

from oracle.validate_gpt_vs_hf import small_case
from tests.gpt_common import gpt_config, load_gpt, make_gpt_weights, prepare_gpt_inputs, r16
from tests.pick_refs import pick, replay_sequence

pytestmark = pytest.mark.gpu

N_SMALL = 40
SAMPLED = [(30, 0.8, 0.8), (1, 1.0, 1.0), (128, 1.0, 3.0), (5, 0.3, 0.5)]
PATHS = {                     # requests, max_batch, bf16 weights, environment at init
    "decode1": (1, 1, True, {}),
    "decode8_3": (3, 8, True, {}),
    "decode8_8": (8, 8, True, {}),
    "fused_bt1": (1, 1, True, {"IDX_GPT_V2": "0"}),
    "fused_bt8": (3, 8, True, {"IDX_GPT_V8": "0"}),
    "strict_1": (1, 1, False, {}),
    "strict_2": (2, 2, False, {}),
    "groups_5x2": (5, 2, True, {}),
}


@contextlib.contextmanager
def _env(env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _init(engine, cfg, w, path, max_prompt=128):
    _, max_batch, bf16, env = PATHS[path]
    with _env(env):
        load_gpt(engine, cfg, w, max_batch=max_batch, max_prompt=max_prompt, bf16=bf16)


def _prompts(cfg, w, n, bf16, seed=5):
    _, style, emo, _ = small_case()
    g = torch.Generator().manual_seed(seed)
    emo = r16(emo) if bf16 else emo
    texts = [torch.randint(2, 100, (int(3 + 5 * i % 17),), generator=g) for i in range(n)]
    return [prepare_gpt_inputs(w, style * (1 + 0.1 * i), emo, t, lang=i % 3, bf16=bf16).numpy()
            for i, t in enumerate(texts)]


def _tie(w, tokens, bias):
    """mel_head rows of `tokens` set to zero with one bf16-exact bias: their logit is exactly `bias` on every path."""
    w = dict(w)
    w["mel_head.weight"] = w["mel_head.weight"].clone()
    w["mel_head.bias"] = w["mel_head.bias"].clone()
    w["mel_head.weight"][tokens] = 0.0
    w["mel_head.bias"][tokens] = bias
    return w


class Stats:
    def __init__(self):
        self.sampled = self.margins = self.refused = self.refusals_checked = 0


def _run(engine, cfg, prompts, n, sp, forced=False, tie_tokens=None, stats=None, seed=0):
    """One generate call, every step of every sequence replayed.  Returns the replays."""
    kw = dict(forbid_stop_before=sp.get("forbid_stop_before", 0))
    if sp.get("do_sample"):
        kw.update(do_sample=True, top_k=sp["top_k"], top_p=sp["top_p"], temperature=sp["temperature"], seed=sp["seed"])
    fc = None
    if forced:
        rng = np.random.default_rng(seed)
        fc = [rng.integers(0, cfg["number_mel_codes"], n).astype(np.int32) for _ in prompts]
    try:
        codes, logits = engine.gpt_generate(prompts, n, sp["rep_penalty"], forced_codes=fc, return_logits=True, **kw)
    except RuntimeError as err:
        # bf16 logits tie often: top_k = 128 can meet a boundary tie wider than 128 candidates, which is refused
        if "more than 128 tokens tie" not in str(err) or stats is None:
            raise
        stats.refused += 1
        if fc is not None:
            # teacher forced, the logits do not depend on the picks: a greedy run yields them, and the reference must
            # refuse one of its steps (the first one reported, unless another sequence's step came first)
            step = int(str(err).rsplit(" ", 1)[1].rstrip(")"))
            _, logits = engine.gpt_generate(prompts, n, sp["rep_penalty"], forced_codes=fc, return_logits=True,
                                            forbid_stop_before=kw["forbid_stop_before"])
            assert any(pick(lg[step], {1, cfg["start_mel_token"]} | set(f[:step].tolist()), step, i,
                            stop_tok=cfg["stop_mel_token"], **sp).refuse for i, (lg, f) in enumerate(zip(logits, fc)))
            stats.refusals_checked += 1
        return []
    out = []
    for i in range(len(prompts)):
        rp = replay_sequence(codes[i], logits[i], seq=i, start_tok=cfg["start_mel_token"], stop_tok=cfg["stop_mel_token"],
                             max_new=n, forced=None if fc is None else fc[i], tie_tokens=tie_tokens, **sp)
        if stats is not None and sp.get("do_sample"):
            stats.sampled += rp.steps
            stats.margins += rp.margins
        out.append(rp)
    return out


def _modes(n):
    for rep in (10.0, 1.0, 0.5):
        yield dict(rep_penalty=rep)
    yield dict(rep_penalty=10.0, forbid_stop_before=n // 2)
    for top_k, top_p, t in SAMPLED:
        yield dict(rep_penalty=10.0, do_sample=True, top_k=top_k, top_p=top_p, temperature=t, seed=2024)


@pytest.mark.parametrize("path", list(PATHS))
def test_small_picks_replay_exactly(engine, path):
    nreq, _, bf16, _ = PATHS[path]
    cfg = small_case()[0]
    w = make_gpt_weights(cfg, seed=1234, bf16=bf16)
    _init(engine, cfg, w, path)
    prompts = _prompts(cfg, w, nreq, bf16)
    st = Stats()
    for sp in _modes(N_SMALL):
        for forced in (False, True):
            _run(engine, cfg, prompts, N_SMALL, sp, forced=forced, stats=st, seed=len(sp))
    print(f"{path}: {st.sampled} sampled picks, {st.margins} within an fp32 margin; {st.refused} calls refused a "
          f"top-k tie wider than 128 ({st.refusals_checked} of them checked against the reference)")
    assert st.sampled > 0 and st.margins <= 0.005 * st.sampled


@pytest.mark.parametrize("path", list(PATHS))
def test_small_forced_ties(engine, path):
    """Greedy: a group at stride 53 (with token 1, the start and stop tokens) ties on every step until the group is
    used up.  Sampling: 40 tied tokens with top_k 30 (the ties extend the kept set) and exactly 128 (accepted); top_p
    puts its boundary between multiples of 1/n.  129 tied tokens are refused, and the engine works on the next call."""
    nreq, _, bf16, _ = PATHS[path]
    cfg = small_case()[0]
    V, start, stop = cfg["number_mel_codes"], cfg["start_mel_token"], cfg["stop_mel_token"]
    base = make_gpt_weights(cfg, seed=77, bf16=bf16)
    prompts = _prompts(cfg, base, nreq, bf16, seed=9)

    grp = sorted(set(range(0, V, 53)) | {1, start, stop})
    w = _tie(base, grp, 48.0)
    _init(engine, cfg, w, path)
    n = len(grp) - 2          # 1 and start are seen from the start and stop is banned: the rest are picked in turn
    for rp in _run(engine, cfg, prompts, n, dict(rep_penalty=10.0, forbid_stop_before=n), tie_tokens=grp):
        assert rp.ties >= len(grp) - 4, rp

    for n_tied, stride, top_p in ((40, 7, 1 - 7.5 / 40), (128, 2, 1 - 12.5 / 128)):
        grp = list(range(1, 1 + stride * n_tied, stride))[:n_tied]
        assert len(grp) == n_tied and grp[-1] < V - 2
        w = _tie(base, grp, 32.0)
        _init(engine, cfg, w, path)
        sp = dict(rep_penalty=1.0, do_sample=True, top_k=30, top_p=top_p, temperature=0.8, seed=11)
        for forced in (False, True):
            for rp in _run(engine, cfg, prompts, 24, sp, forced=forced, tie_tokens=grp):
                assert rp.ties == rp.steps == 24, rp

    w = _tie(base, list(range(1, 259, 2)), 32.0)          # 129 tied tokens
    _init(engine, cfg, w, path)
    with pytest.raises(RuntimeError, match="more than 128 tokens tie"):
        engine.gpt_generate(prompts, 8, 1.0, do_sample=True, top_k=30, top_p=0.9, temperature=0.8, seed=3)
    for rp in _run(engine, cfg, prompts, 8, dict(rep_penalty=1.0)):
        assert rp.steps == 8


def test_beam_sample_tie_overflow_refused(engine):
    cfg = small_case()[0]
    base = make_gpt_weights(cfg, seed=77, bf16=True)
    prompts = _prompts(cfg, base, 1, True)
    kw = dict(do_sample=True, num_beams=3, top_k=30, top_p=1.0, temperature=0.8, seed=3)
    for n_tied, refused in ((129, True), (128, False)):
        w = _tie(base, list(range(1, 1 + 2 * n_tied, 2)), 32.0)
        load_gpt(engine, cfg, w, max_batch=8)
        if refused:
            with pytest.raises(RuntimeError, match="more than 128 tokens tie"):
                engine.gpt_generate(prompts, 6, 1.0, **kw)
        else:
            (codes,) = engine.gpt_generate(prompts, 6, 1.0, **kw)
            assert len(codes) >= 1
    # plain beam search keeps no ties and is not refused
    w = _tie(base, list(range(1, 259, 2)), 32.0)
    load_gpt(engine, cfg, w, max_batch=8)
    engine.gpt_generate(prompts, 6, 1.0, num_beams=3)


def test_sampling_parameters_refused_before_launch(engine):
    cfg = small_case()[0]
    w = make_gpt_weights(cfg, seed=1234, bf16=True)
    load_gpt(engine, cfg, w)
    prompts = _prompts(cfg, w, 1, True)
    engine.gpt_generate(prompts, 4, 10.0)
    before = engine.gpt_last_timing()
    nan, inf = float("nan"), float("inf")
    bad = [dict(repetition_penalty=x) for x in (0.0, -1.0, nan, inf)]
    bad += [dict(do_sample=True, top_k=30, temperature=x) for x in (0.0, -0.5, nan, inf)]
    bad += [dict(do_sample=True, top_k=30, top_p=x) for x in (-0.1, 1.5, nan)]
    for kw in bad:
        kw = dict(dict(repetition_penalty=10.0), **kw)
        with pytest.raises(RuntimeError, match="repetition_penalty|temperature|top_p"):
            engine.gpt_generate(prompts, 4, **kw)
        assert engine.gpt_last_timing() == before, kw
    # greedy ignores temperature and top_p, as HF does
    (a,) = engine.gpt_generate(prompts, 4, 10.0, temperature=0.0, top_p=5.0)
    (b,) = engine.gpt_generate(prompts, 4, 10.0)
    assert np.array_equal(a, b)


@pytest.fixture(scope="module")
def full():
    cfg = gpt_config()
    w = make_gpt_weights(cfg, seed=2025, bf16=True)
    g = torch.Generator().manual_seed(11)
    style = torch.randn(192, generator=g)
    emo = r16(torch.randn(cfg["model_dim"], generator=g) * 0.5)
    prompts = [prepare_gpt_inputs(w, style * (1 + 0.2 * i), emo, torch.randint(2, 12000, (20 + 4 * i,), generator=g),
                                  lang=1, bf16=True).numpy() for i in range(3)]
    return cfg, w, prompts


@pytest.mark.parametrize("path", ["decode1", "decode8_3", "fused_bt1"])
def test_full_size_picks_replay_exactly(engine, full, path):
    """24 x 1280, V = 8194 (NPL = 40): a greedy and a sampled run of 64 steps, and a greedy tie group at stride 53 over
    V (with 1, start, stop = the V tail) that ties on every step across CTA, warp and thread-slot boundaries."""
    cfg, w, prompts = full
    nreq = PATHS[path][0]
    prompts = prompts[:nreq]
    _init(engine, cfg, w, path, max_prompt=64)
    n = 64
    _run(engine, cfg, prompts, n, dict(rep_penalty=10.0, forbid_stop_before=n))
    st = Stats()
    _run(engine, cfg, prompts, n, dict(rep_penalty=10.0, do_sample=True, top_k=30, top_p=0.8, temperature=0.8, seed=7),
         stats=st)
    V = cfg["number_mel_codes"]
    grp = sorted(set(range(0, V, 53)) | {1, cfg["start_mel_token"], cfg["stop_mel_token"]})
    _init(engine, cfg, _tie(w, grp, 48.0), path, max_prompt=64)
    n = len(grp) - 2
    for rp in _run(engine, cfg, prompts, n, dict(rep_penalty=10.0, forbid_stop_before=n), tie_tokens=grp):
        assert rp.ties >= len(grp) - 4, rp
    print(f"{path} full size: {st.sampled} sampled picks, {st.margins} within an fp32 margin; tie group of {len(grp)}")
    assert st.margins <= max(1, 0.005 * st.sampled)
