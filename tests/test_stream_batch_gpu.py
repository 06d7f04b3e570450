"""Batched chunked streaming on the H100 at the real geometry (synthetic weights: GPT 24 x 1280, the config-2 tail of
synth), one decode group of up to 8 requests with prompts of different lengths: the resumable group decode
idx_gpt_stream_*_batch against idx_gpt_generate, every request's beam commit against its beam buffers, tail calls between
two decode calls, the multi-slot join of idx_stream_vocode_batch against idx_codes_to_wav and the host model of the
reference's join (tests/stream_refs.py), the stream_segments generator replayed on the host, and the refusals."""
import ctypes as C

import numpy as np
import pytest
import torch

from indextts_b200 import synth
from indextts_b200.engine import fold_weight_norm
from tests.stream_refs import HostJoin

MAX_NEW = 160
P = 200
P2 = 120                      # a second speaker prompt of another length
STOP = 8193
SAMPLE = dict(do_sample=True, top_k=30, top_p=0.8, temperature=0.8, repetition_penalty=10.0, seed=11)
GREEDY = dict(do_sample=False, repetition_penalty=10.0)


def _lengths(engine, prompts):
    return [len(c) for c in engine.gpt_generate(prompts, MAX_NEW, **GREEDY)]


@pytest.fixture(scope="module")
def rig(engine):
    cfg = synth.gpt_config()
    w = synth.make_gpt_weights(cfg, seed=2025, bf16=True)
    engine.load_state_dict("gpt.", w)

    def init():
        engine.gpt_init(cfg["layers"], cfg["model_dim"], cfg["heads"], cfg["number_mel_codes"], cfg["start_mel_token"],
                        cfg["stop_mel_token"], cfg["max_mel_positions"], max_prompt=96, max_batch=8, weights_bf16=True)
    init()
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
    prompts = []
    for i in range(8):                      # text lengths 16..51: prompts of different lengths
        emo = synth.r16(torch.randn(cfg["model_dim"], generator=g) * 0.5).numpy()
        text = torch.randint(2, 12000, (16 + 5 * i,), generator=g).numpy()
        prompts.append(engine.gpt_prepare_inputs(style, emo, text, 1))
    # the random weights may never pick the stop code: raise its head bias until requests end at different lengths
    bias = w["mel_head.bias"].clone()
    for add in (0.0, 4.0, 6.0, 8.0, 10.0, 12.0):
        b = bias.clone()
        b[STOP] += add
        engine.load_weight("gpt.mel_head.bias", b)
        init()
        lens = _lengths(engine, prompts)
        if len({n for n in lens if n < MAX_NEW}) >= 2:
            break
    print(f"stop-code bias +{add}: greedy lengths {lens}")
    tail = dict(prompt_condition=torch.randn(P, 512, generator=g).numpy(),
                ref_mel=(torch.randn(80, P, generator=g) * 1.5 - 4.0).numpy(), style=style)
    tail2 = dict(prompt_condition=torch.randn(P2, 512, generator=g).numpy(),
                 ref_mel=(torch.randn(80, P2, generator=g) * 1.5 - 4.0).numpy(), style=torch.randn(192, generator=g).numpy())
    return dict(cfg=cfg, prompts=prompts, tail=tail, tail2=tail2, lens=lens)


@pytest.mark.gpu
def test_requests_end_at_different_lengths(engine, rig):
    ended = {n for n in rig["lens"] if n < MAX_NEW}
    assert len(ended) >= 2, rig["lens"]


def _stream_batch(engine, prompts, step, between=None, **kw):
    """Every request's codes of a group stream whose `until` grows by step (odd requests) or 2 step (even ones), checking
    the return and launch rules of num_beams = 1."""
    n = len(prompts)
    m = kw.get("num_beams", 1)
    out = [[] for _ in range(n)]
    with engine.gpt_stream_batch(prompts, MAX_NEW, **kw) as st:
        while not all(st.finished):
            fin0 = list(st.finished)
            until = [st.n_committed[i] + step * (1 + i % 2) for i in range(n)]
            new, fin = st.next(until)
            for i in range(n):
                out[i].append(new[i])
            live = [i for i in range(n) if not fin[i]]
            newly = any(fin[i] and not fin0[i] for i in range(n))
            if m == 1 and live:
                target = min(until[i] for i in live)
                assert len({st.n_committed[i] for i in live}) == 1          # the rows advance in lockstep
                if not newly:
                    assert st.n_committed[live[0]] == target                # the launch ends at the smallest until
                else:
                    assert st.n_committed[live[0]] <= target
            if between is not None:
                between()
    return [np.concatenate(o) for o in out]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("name,kw", [("greedy", GREEDY), ("sample", SAMPLE)])
@pytest.mark.parametrize("nreq", [2, 3, 8])
def test_group_stream_codes_equal_generate(engine, rig, nreq, name, kw, mode):
    prompts = rig["prompts"][:nreq]
    ref = engine.gpt_generate(prompts, MAX_NEW, mel_pos_mode=mode, **kw)
    for step in (1, 7, 32, 100, MAX_NEW):
        got = _stream_batch(engine, prompts, step, mel_pos_mode=mode, **kw)
        for i in range(nreq):
            np.testing.assert_array_equal(got[i], ref[i], err_msg=f"{name} mode {mode} nreq {nreq} step {step} request {i}")
    print(f"nreq {nreq} {name} mode {mode}: lengths {[len(r) for r in ref]}")


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [GREEDY, SAMPLE, dict(SAMPLE, num_beams=3)])
def test_one_request_group_equals_gpt_stream(engine, rig, kw):
    p = rig["prompts"][3]
    for step in (1, 7, 64):
        a, b = [], []
        with engine.gpt_stream_batch([p], MAX_NEW, **kw) as sb:
            while not sb.finished[0]:
                new, _ = sb.next([sb.n_committed[0] + step])
                a.append((new[0].copy(), sb.n_committed[0], sb.finished[0]))
        with engine.gpt_stream(p, MAX_NEW, **kw) as s1:
            while not s1.finished:
                new, _ = s1.next(s1.n_committed + step)
                b.append((new.copy(), s1.n_committed, s1.finished))
        assert len(a) == len(b)
        for x, y in zip(a, b):
            np.testing.assert_array_equal(x[0], y[0])
            assert x[1:] == y[1:]


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
def test_group_beam_stream(engine, rig, m, do_sample):
    nreq = 8 // m
    prompts = rig["prompts"][:nreq]
    kw = dict(SAMPLE if do_sample else GREEDY, num_beams=m, length_penalty=1.0)
    ref = engine.gpt_generate(prompts, MAX_NEW, **kw)
    early = 0
    for step in (1, 7, MAX_NEW):
        with engine.gpt_stream_batch(prompts, MAX_NEW, **kw) as st:
            prev = [np.zeros(0, np.int32)] * nreq
            while not all(st.finished):
                st.next([st.n_committed[i] + step for i in range(nreq)])
                group_open = not all(st.finished)
                for i in range(nreq):
                    codes = st.codes[i].copy()
                    assert len(codes) >= len(prev[i])
                    np.testing.assert_array_equal(codes[:len(prev[i])], prev[i])     # prefixes never shrink
                    np.testing.assert_array_equal(ref[i][:len(codes)], codes)
                    prev[i] = codes
                    if st.finished[i]:
                        if group_open:
                            np.testing.assert_array_equal(codes, ref[i])             # finished before the group
                            early += 1
                        continue
                    bs = st.beam_state(i)
                    lcp, c0 = _host_lcp(bs, m)
                    assert st.n_committed[i] == lcp, (i, bs["steps"])
                    np.testing.assert_array_equal(codes, c0[:lcp])
            for i in range(nreq):
                np.testing.assert_array_equal(st.codes[i], ref[i], err_msg=f"m {m} sample {do_sample} step {step} req {i}")
    print(f"num_beams {m} x {nreq} requests, do_sample {do_sample}: lengths {[len(r) for r in ref]}, "
          f"{early} request reports finished before the group ended")


def _window(rng, t, n):
    from indextts_b200.streaming import window_frames
    codes = rng.integers(0, 8192, n).astype(np.int32)
    F = window_frames(n)
    z = rng.standard_normal((80, t["ref_mel"].shape[-1] + F)).astype(np.float32)
    return dict(codes=codes, prompt_condition=t["prompt_condition"], ref_mel=t["ref_mel"], style=t["style"], z=z, F=F)


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [GREEDY, dict(SAMPLE, num_beams=2)])
def test_tail_calls_between_next_calls_change_nothing(engine, rig, kw):
    from indextts_b200.streaming import overlap_samples
    rng = np.random.default_rng(3)
    t, t2 = rig["tail"], rig["tail2"]
    w0, w1 = _window(rng, t, 30), _window(rng, t2, 30)

    def tail():
        engine.codes_to_wav(**w0, want_wav=True)
        engine.stream_vocode_batch([dict(w0, slot=0, first=True, overlap_samples=overlap_samples(5)),
                                    dict(w1, slot=1, first=True, last=True)])

    prompts = rig["prompts"][:3]
    quiet = _stream_batch(engine, prompts, 7, **kw)
    busy = _stream_batch(engine, prompts, 7, between=tail, **kw)
    ref = engine.gpt_generate(prompts, MAX_NEW, **kw)
    for i in range(3):
        np.testing.assert_array_equal(busy[i], quiet[i])
        np.testing.assert_array_equal(quiet[i], ref[i])


def _np(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _close(got, want, what):
    got = _np(got)
    assert got.dtype == np.int16 and len(got) == len(want), (what, len(got), len(want))
    assert int(np.abs(got.astype(np.int32) - want.astype(np.int32)).max(initial=0)) <= 1, what


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True])
def test_stream_vocode_batch_join(engine, rig, device):
    from indextts_b200.streaming import overlap_samples
    rng = np.random.default_rng(11)
    t, t2 = rig["tail"], rig["tail2"]
    ovlp = overlap_samples(10)

    def dev(w):
        if not device:
            return w
        return {k: (torch.from_numpy(np.ascontiguousarray(v)).cuda() if isinstance(v, np.ndarray) else v) for k, v in w.items()}

    # per call: slot -> (window size in codes or None for the flush, first, last, speaker)
    calls = [
        {0: (40, True, False, t), 1: (40, True, False, t2), 2: (25, True, True, t2), 5: (30, True, False, t)},
        {0: (40, False, False, t), 1: (None, False, True, None), 5: (12, False, True, t2)},
        {0: (9, False, True, t2), 3: (40, True, False, t)},
        {3: (None, False, True, None)},
    ]
    joins = {s: HostJoin() for s in range(8)}
    for ci, call in enumerate(calls):
        ws, wavs = [], []
        for slot, (n, first, last, tt) in call.items():
            if n is None:
                ws.append(dict(slot=slot, codes=None, last=True))
                wavs.append(None)
                continue
            w = _window(rng, tt, n)
            wavs.append(np.asarray(engine.codes_to_wav(**w)["wav"]))             # the solo tail of the window
            ws.append(dict(dev(w), slot=slot, first=first, last=last, overlap_samples=ovlp, want_wav=True))
        res = engine.stream_vocode_batch(ws)
        for w, r, wav in zip(ws, res, wavs):
            slot = w["slot"]
            if wav is None:
                want = joins[slot].flush()
                _close(r["pcm"], np.zeros(0, np.int16) if want is None else want, f"call {ci} flush of slot {slot}")
                continue
            got_wav = _np(r["wav"])
            assert got_wav.view(np.uint32).tobytes() == wav.view(np.uint32).tobytes(), f"call {ci} slot {slot}: waveform"
            _close(r["pcm"], joins[slot].push(wav, ovlp, first=w["first"], last=w["last"]), f"call {ci} slot {slot}")
    # a one-window call on slot 0 equals stream_vocode (its one-window, slot-0 case)
    w = _window(rng, t2, 40)
    a = engine.stream_vocode_batch([dict(w, slot=0, first=True, overlap_samples=ovlp)])[0]["pcm"]
    b = engine.stream_vocode(**w, overlap_samples=ovlp, first=True)["pcm"]
    np.testing.assert_array_equal(_np(a), _np(b))
    engine.stream_vocode(None, last=True)


@pytest.mark.gpu
@pytest.mark.parametrize("shared", [True, False])
def test_stream_segments_replays_on_the_host(engine, rig, shared):
    from indextts_b200 import streaming
    prompts = [rig["prompts"][i] for i in (0, 4, 7)]
    chunk, ov = 40, 10
    ovlp = streaming.overlap_samples(ov)
    t, t2 = rig["tail"], rig["tail2"]
    spk = [t, t2, t] if not shared else [t] * 3
    pc = t["prompt_condition"] if shared else [s["prompt_condition"] for s in spk]
    mel = t["ref_mel"] if shared else [s["ref_mel"] for s in spk]
    sty = t["style"] if shared else [s["style"] for s in spk]
    ref = engine.gpt_generate(prompts, MAX_NEW, **SAMPLE)
    calls, orig = [], engine.stream_vocode_batch

    def spy(windows, *a, **k):
        calls.append([dict(slot=w["slot"], z=None if w.get("codes") is None else np.array(w["z"]), F=w.get("F"),
                           codes=None if w.get("codes") is None else np.array(w["codes"])) for w in windows])
        return orig(windows, *a, **k)
    engine.stream_vocode_batch = spy
    try:
        torch.manual_seed(1234)
        got, n_done = [[] for _ in range(3)], [0, 0, 0]
        for audio, done in streaming.stream_segments(engine, prompts, pc, mel, sty, chunk_codes=chunk, overlap_codes=ov,
                                                     max_new_tokens=MAX_NEW, **SAMPLE):
            for i in range(3):
                if audio[i] is not None:
                    assert n_done[i] == 0, "audio after done"
                    got[i].append(_np(audio[i]))
                n_done[i] += done[i]
    finally:
        del engine.stream_vocode_batch
    assert n_done == [1, 1, 1]
    # the noise: torch.randn(80, P_i + F) per window, in call order and request order within a call
    torch.manual_seed(1234)
    for call in calls:
        for w in call:
            if w["z"] is not None:
                z = torch.randn(80, int(spk[w["slot"]]["ref_mel"].shape[-1]) + w["F"]).numpy()
                assert z.tobytes() == w["z"].tobytes()
    # each request's windows: its own schedule over its streamed codes, joined on the host
    for i in range(3):
        codes = ref[i]
        n = int(np.flatnonzero(codes == STOP)[0]) if (codes == STOP).any() else len(codes)
        sched = streaming.schedule(n, chunk, ov)
        mine = [w for call in calls for w in call if w["slot"] == i]
        hj, want = HostJoin(), []
        for k, w in enumerate(mine):
            if w["codes"] is None:
                assert k == len(sched) and (not sched or not sched[-1][2])
                want.append(hj.flush())
                continue
            a, b, last = sched[k]
            np.testing.assert_array_equal(w["codes"], codes[a:b])
            s = spk[i]
            wav = np.asarray(engine.codes_to_wav(w["codes"], s["prompt_condition"], s["ref_mel"], s["style"], w["z"],
                                                 w["F"])["wav"])
            want.append(hj.push(wav, ovlp, first=k == 0, last=last))
        want = np.concatenate(want) if want else np.zeros(0, np.int16)
        _close(np.concatenate(got[i]) if got[i] else np.zeros(0, np.int16), want, f"request {i}")
        print(f"request {i}: {n} codes, {len(mine)} windows, {len(want)} samples")


def _rc(fn, *a, **k):
    with pytest.raises(RuntimeError) as ex:
        fn(*a, **k)
    return int(str(ex.value).split("failed (")[1].split(")")[0])


@pytest.mark.gpu
def test_refusals_leave_everything_as_it_was(engine, rig):
    from indextts_b200.engine import StreamWindow
    from indextts_b200.streaming import overlap_samples
    lib, h, prompts = engine.lib, engine.h, rig["prompts"]
    assert _rc(engine.gpt_stream_batch, prompts[:3], 40, **dict(SAMPLE, num_beams=3)) == 2     # 9 rows > max_batch 8
    ref = engine.gpt_generate(prompts[:3], 40, **GREEDY)
    st = engine.gpt_stream_batch(prompts[:3], 40, **GREEDY)
    try:
        u = (C.c_int32 * 3)(5, 0, 5)
        outs = (C.c_void_p * 3)(*[b.ctypes.data for b in st._bufs])
        n, fin = (C.c_int32 * 3)(), (C.c_int32 * 3)()
        assert lib.idx_gpt_stream_next_batch(h, u, outs, n, fin) == 2                           # until < 1
        assert st.n_committed == [0, 0, 0]
        assert _rc(engine.gpt_stream_batch, prompts[:2], 40) == 3                              # a second begin
        assert _rc(engine.gpt_stream, prompts[0], 40) == 3
        assert _rc(engine.gpt_generate, [prompts[0]], 40) == 3
        while not all(st.finished):
            st.next([40] * 3)
        for i in range(3):
            np.testing.assert_array_equal(st.codes[i], ref[i])
    finally:
        st.close()

    # idx_stream_vocode_batch: slots 0 and 1 keep tails; each refused call emits nothing and keeps them
    rng = np.random.default_rng(5)
    t, t2 = rig["tail"], rig["tail2"]
    ovlp = overlap_samples(10)
    w0, w1 = _window(rng, t, 40), _window(rng, t2, 40)
    hj = [HostJoin(), HostJoin()]
    res = engine.stream_vocode_batch([dict(w0, slot=0, first=True, overlap_samples=ovlp),
                                      dict(w1, slot=1, first=True, overlap_samples=ovlp)])
    for k, w in enumerate((w0, w1)):
        _close(res[k]["pcm"], hj[k].push(np.asarray(engine.codes_to_wav(**w)["wav"]), ovlp, first=True), f"slot {k}")
    keep = []

    def win(slot, w=None, flags=0, cap=None):
        r = None
        if w is not None:
            r, _, k = engine._vocode_request(w["codes"], w["prompt_condition"], w["ref_mel"], w["style"], w["z"], w["F"],
                                             False, False, False)
            keep.append((r, k))
        pcm = np.full(w["F"] * 256 + ovlp if w is not None else ovlp, 777, np.int16)
        cnt = C.c_int32(len(pcm) if cap is None else cap)
        keep.append((pcm, cnt))
        return StreamWindow(slot, None if r is None else C.pointer(r), ovlp, flags, pcm.ctypes.data, C.pointer(cnt)), pcm, cnt

    w2 = _window(rng, t, 40)
    bad = {
        "slot 8": [win(8, w2)],
        "slot -1": [win(-1, w2)],
        "duplicate slots": [win(2, w2), win(2, w2)],
        "flush without LAST": [win(3, None, 0)],
        "capacity too small": [win(2, w2), win(0, w2, cap=w2["F"] * 256)],
        "unknown flags": [win(2, w2, 4)],
    }
    for what, ws in bad.items():
        arr = (StreamWindow * len(ws))(*[x[0] for x in ws])
        assert lib.idx_stream_vocode_batch(h, arr, len(ws), 25, C.c_float(0.7)) == 2, what
        for _, pcm, cnt in ws:
            assert (pcm == 777).all(), f"{what}: something was emitted"
    flushed = engine.stream_vocode_batch([dict(slot=0, codes=None, last=True), dict(slot=1, codes=None, last=True)])
    for k in range(2):
        _close(flushed[k]["pcm"], hj[k].flush(), f"kept tail of slot {k} after the refusals")
