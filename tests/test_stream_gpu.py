"""Chunked streaming on the H100 at the real geometry (synthetic weights: GPT 24 x 1280, the config-2 tail of synth):
the resumable decode idx_gpt_stream_* against idx_gpt_generate, the beam commit against the beam buffers, tail calls
between two decode calls, and the device join of idx_stream_vocode against idx_codes_to_wav and the host model of the
reference's StreamingDecoder join (tests/stream_refs.py)."""
import numpy as np
import pytest
import torch

from indextts_b200 import synth
from indextts_b200.engine import fold_weight_norm
from tests.stream_refs import HostJoin

MAX_NEW = 160
P = 200                       # prompt frames of the tail (a 10 s prompt has 861; the join does not depend on P)
STOP = 8193


@pytest.fixture(scope="module")
def rig(engine):
    cfg = synth.gpt_config()
    engine.load_state_dict("gpt.", synth.make_gpt_weights(cfg, seed=2025, bf16=True))
    engine.gpt_init(cfg["layers"], cfg["model_dim"], cfg["heads"], cfg["number_mel_codes"], cfg["start_mel_token"],
                    cfg["stop_mel_token"], cfg["max_mel_positions"], max_prompt=64, max_batch=4, weights_bf16=True)
    c, cc, h = dict(synth.S2MEL_CFG), dict(synth.CODEC_CFG), dict(synth.BIGVGAN_V2_22K)
    ws = fold_weight_norm(synth.make_s2mel_weights(c, seed=1234))
    engine.load_state_dict("s2mel.", {k: v for k, v in ws.items() if v.is_floating_point()})
    engine.load_state_dict("codec.", fold_weight_norm(synth.make_codec_weights(cc, seed=4321)))
    engine.load_state_dict("bigvgan.", synth.make_bigvgan_weights(h, seed=1234))
    engine.s2mel_init(c)
    engine.codec_init(cc)
    engine.bigvgan_init(h)
    g = torch.Generator().manual_seed(7)
    style = torch.randn(192, generator=g).numpy()
    emo = synth.r16(torch.randn(cfg["model_dim"], generator=g) * 0.5).numpy()
    text = torch.randint(2, 12000, (32,), generator=g).numpy()
    prompt = engine.gpt_prepare_inputs(style, emo, text, 1)
    tail = dict(prompt_condition=torch.randn(P, 512, generator=g).numpy(),
                ref_mel=(torch.randn(80, P, generator=g) * 1.5 - 4.0).numpy(), style=style)
    return dict(cfg=cfg, prompt=prompt, tail=tail)


def _stream(engine, prompt, step, between=None, **kw):
    """Every code of a stream whose `until` grows by `step`, checking the commit contract of num_beams = 1."""
    out = []
    with engine.gpt_stream(prompt, MAX_NEW, **kw) as st:
        until = 0
        while not st.finished:
            until += step
            new, fin = st.next(until)
            out.append(new)
            if not fin and kw.get("num_beams", 1) == 1:
                assert st.n_committed == until          # the launches end exactly at `until`
            if between is not None:
                between()
    return np.concatenate(out)


SAMPLE = dict(do_sample=True, top_k=30, top_p=0.8, temperature=0.8, repetition_penalty=10.0, seed=11)
GREEDY = dict(do_sample=False, repetition_penalty=10.0)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("name,kw", [("greedy", GREEDY), ("sample", SAMPLE), ("greedy_forbid", dict(GREEDY, forbid_stop_before=MAX_NEW))])
def test_stream_codes_equal_generate(engine, rig, name, kw, mode):
    ref = engine.gpt_generate([rig["prompt"]], MAX_NEW, mel_pos_mode=mode, **kw)[0]
    for step in (1, 7, 64, 100, MAX_NEW):
        got = _stream(engine, rig["prompt"], step, mel_pos_mode=mode, **kw)
        np.testing.assert_array_equal(got, ref, err_msg=f"{name} mel_pos_mode {mode} until step {step}")
    print(f"{name} mode {mode}: {len(ref)} codes, stop token {'produced' if ref[-1] == STOP else 'not produced'}")


def _host_lcp(bs, m):
    cands = [] if bs["done"] else [bs["hist"][j][:bs["steps"]] for j in range(m)]
    for q in range(bs["nhyp"]):
        s = bs["hyp_order"][q]
        cands.append(bs["hyp_tok"][s][:bs["hyp_len"][s]])
    n = min(len(c) for c in cands)
    for t in range(n):
        if any(c[t] != cands[0][t] for c in cands[1:]):
            return t, cands[0]
    return n, cands[0]


@pytest.mark.gpu
@pytest.mark.parametrize("do_sample", [0, 1])
@pytest.mark.parametrize("m", [2, 3, 4])
def test_beam_stream_commits_only_what_cannot_change(engine, rig, m, do_sample):
    kw = dict(SAMPLE if do_sample else GREEDY, num_beams=m, length_penalty=1.0)
    ref = engine.gpt_generate([rig["prompt"]], MAX_NEW, **kw)[0]
    for step in (1, 7, 64, 100, MAX_NEW):
        trail, prefixes = [], []
        with engine.gpt_stream(rig["prompt"], MAX_NEW, **kw) as st:
            until = 0
            while not st.finished:
                until += step
                st.next(until)
                if not st.finished:
                    assert st.n_committed >= until
                    bs = st.beam_state()
                    lcp, c0 = _host_lcp(bs, m)
                    assert st.n_committed == lcp, (step, bs["steps"])
                    np.testing.assert_array_equal(st.codes, c0[:lcp])
                    trail.append(bs["steps"] - lcp)
                    prefixes.append(st.codes.copy())
            got = st.codes.copy()
        np.testing.assert_array_equal(got, ref, err_msg=f"num_beams {m} do_sample {do_sample} until step {step}")
        for pfx in prefixes:
            np.testing.assert_array_equal(ref[:len(pfx)], pfx)
        if step == 1:
            print(f"num_beams {m} do_sample {do_sample}: {len(ref)} codes; the commit trails the decode by "
                  f"{min(trail, default=0)}..{max(trail, default=0)} steps (mean {np.mean(trail) if trail else 0:.1f}) "
                  "-- random weights say little about how real beams agree")


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [GREEDY, dict(SAMPLE, num_beams=3)])
def test_tail_calls_between_next_calls_change_nothing(engine, rig, kw):
    rng = np.random.default_rng(3)
    codes = rng.integers(0, 8192, 10).astype(np.int32)
    F = int(2 * 10 * 1.72)
    z = rng.standard_normal((80, P + F)).astype(np.float32)
    t = rig["tail"]

    def tail():
        engine.codes_to_wav(codes, t["prompt_condition"], t["ref_mel"], t["style"], z, F, want_wav=True)

    quiet = _stream(engine, rig["prompt"], 7, **kw)
    busy = _stream(engine, rig["prompt"], 7, between=tail, **kw)
    np.testing.assert_array_equal(busy, quiet)
    np.testing.assert_array_equal(quiet, engine.gpt_generate([rig["prompt"]], MAX_NEW, **kw)[0])


JOIN_CASES = {
    "three windows, overlap 20 codes": (20, [100, 100, 60], True),
    "overlap 0 (concatenation), then the flush": (0, [50, 50], False),
    "a single window": (20, [70], True),
    "no last window: the flush fades the kept tail out": (20, [100, 100], False),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(JOIN_CASES))
@pytest.mark.parametrize("device", [False, True])
def test_stream_vocode_join(engine, rig, case, device):
    from indextts_b200.streaming import overlap_samples, window_frames
    ov, sizes, ends_last = JOIN_CASES[case]
    ovlp = overlap_samples(ov)
    rng = np.random.default_rng(len(sizes) * 100 + ov)
    t = rig["tail"]
    hj, total, want_total = HostJoin(), 0, 0
    for i, n in enumerate(sizes):
        codes = rng.integers(0, 8192, n).astype(np.int32)
        F = window_frames(n)
        z = rng.standard_normal((80, P + F)).astype(np.float32)
        last = ends_last and i == len(sizes) - 1
        wav = np.asarray(engine.codes_to_wav(codes, t["prompt_condition"], t["ref_mel"], t["style"], z, F)["wav"])
        args = (codes, t["prompt_condition"], t["ref_mel"], t["style"], z)
        if device:
            args = tuple(torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in args)
        res = engine.stream_vocode(*args, F, overlap_samples=ovlp, first=i == 0, last=last, want_wav=True)
        got_wav = res["wav"].cpu().numpy() if device else res["wav"]
        assert got_wav.view(np.uint32).tobytes() == wav.view(np.uint32).tobytes(), f"window {i}: waveform differs"
        pcm = res["pcm"].cpu().numpy() if device else res["pcm"]
        want = hj.push(wav, ovlp, first=i == 0, last=last)
        assert pcm.dtype == np.int16 and len(pcm) == len(want), (i, len(pcm), len(want))
        assert int(np.abs(pcm.astype(np.int32) - want.astype(np.int32)).max(initial=0)) <= 1, f"window {i}"
        total += len(pcm)
        want_total += len(want)
    if not ends_last:
        pcm = engine.stream_vocode(None, last=True)["pcm"]
        want = hj.flush()
        assert len(pcm) == len(want) and int(np.abs(pcm.astype(np.int32) - want.astype(np.int32)).max(initial=0)) <= 1
        total += len(pcm)
        want_total += len(want)
    assert total == want_total
    # after the last window nothing is kept: a flush emits nothing
    assert len(engine.stream_vocode(None, last=True)["pcm"]) == 0


def _rc(fn, *a, **k):
    with pytest.raises(RuntimeError) as ex:
        fn(*a, **k)
    return int(str(ex.value).split("failed (")[1].split(")")[0])


@pytest.mark.gpu
def test_refusals_and_states(engine, rig):
    import ctypes as C
    lib, h, prompt = engine.lib, engine.h, rig["prompt"]
    ref = engine.gpt_generate([prompt], 40, **GREEDY)[0]
    buf = np.zeros(64, np.int32)
    n, fin = C.c_int32(0), C.c_int32(0)
    assert lib.idx_gpt_stream_next(h, 1, buf.ctypes.data, C.byref(n), C.byref(fin)) == 3       # next without begin
    assert lib.idx_gpt_stream_end(h) == 3                                                     # end without begin
    assert _rc(engine.gpt_stream, prompt, 40, forced_codes=[[1, 2, 3]]) == 2
    st = engine.gpt_stream(prompt, 40, **GREEDY)
    try:
        assert lib.idx_gpt_stream_next(h, 0, buf.ctypes.data, C.byref(n), C.byref(fin)) == 2  # until < 1
        assert _rc(engine.gpt_stream, prompt, 40) == 3                                        # a second begin
        assert _rc(engine.gpt_generate, [prompt], 40) == 3
        assert _rc(engine.gpt_latents_v1, np.zeros((32, 1280), np.float32), [5, 6], [7, 8]) == 3
        assert _rc(engine.gpt_probe_attention, 0, 40) == 3
        assert _rc(engine.gpt_probe_prefill, 0, 64) == 3
        assert _rc(engine.gpt_kv, 0, 0, 0, 4) == 3
        cfg = rig["cfg"]
        assert _rc(engine.gpt_init, cfg["layers"], cfg["model_dim"], cfg["heads"]) == 3
        # the tail runs while the stream is open
        codes = np.arange(1, 11, dtype=np.int32)
        F = int(2 * 10 * 1.72)
        z = np.zeros((80, P + F), np.float32)
        t = rig["tail"]
        engine.codes_to_wav(codes, t["prompt_condition"], t["ref_mel"], t["style"], z, F)
        st.next(40)
        np.testing.assert_array_equal(st.codes, ref)
    finally:
        st.close()
    np.testing.assert_array_equal(engine.gpt_generate([prompt], 40, **GREEDY)[0], ref)

    # idx_stream_vocode refusals: nothing is emitted and the kept tail stays
    t = rig["tail"]
    codes = np.arange(1, 21, dtype=np.int32)
    F = int(2 * 20 * 1.72)
    z = np.zeros((80, P + F), np.float32)
    args = (codes, t["prompt_condition"], t["ref_mel"], t["style"], z, F)
    assert _rc(engine.stream_vocode, *args, overlap_samples=-1, first=True) == 2
    assert _rc(engine.stream_vocode, *args, overlap_samples=F * 256 // 2 + 1, first=True) == 2    # len < 2 ovlp, not last
    engine.stream_vocode(*args, overlap_samples=F * 256 // 2, first=True, last=True)              # a last window may be short
    r, _, keep = engine._vocode_request(*args, False, False, False)
    pcm = np.zeros(F * 256, np.int16)
    cap = C.c_int32(F * 256 - 1)
    assert lib.idx_stream_vocode(h, C.byref(r), 25, C.c_float(0.7), 0, 1, pcm.ctypes.data, C.byref(cap)) == 2
    assert lib.idx_stream_vocode(h, None, 25, C.c_float(0.7), 0, 0, pcm.ctypes.data, C.byref(cap)) == 2   # flush w/o LAST


@pytest.mark.gpu
def test_strict_path_refuses_a_stream(engine, rig):
    cfg = synth.gpt_config(layers=2, model_dim=256, heads=4)
    engine.load_state_dict("gpt.", synth.make_gpt_weights(cfg, seed=5, bf16=False))
    engine.gpt_init(cfg["layers"], cfg["model_dim"], cfg["heads"], cfg["number_mel_codes"], cfg["start_mel_token"],
                    cfg["stop_mel_token"], cfg["max_mel_positions"], max_prompt=64, max_batch=1, weights_bf16=False)
    prompt = np.random.default_rng(1).standard_normal((20, 256)).astype(np.float32) * 0.1
    assert _rc(engine.gpt_stream, prompt, 20) == 2
