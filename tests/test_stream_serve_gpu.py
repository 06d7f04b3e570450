"""Serving groups on the H100 at the real geometry (synthetic weights: GPT 24 x 1280, the config-2 tail of synth):
requests admitted into a running idx_gpt_serve_* group at staggered steps against idx_gpt_generate of all of them, slot
reuse, cancels, tail calls between decode calls, StreamServer end to end against the host join of tests/stream_refs.py,
and the refusals."""
import ctypes as C
import os

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
N_REQ = 12                    # gpt_generate decodes them as groups of 8 and 4: both on gpt_decode8_kernel
SAMPLE = dict(do_sample=True, top_k=30, top_p=0.8, temperature=0.8, repetition_penalty=10.0, seed=11)
GREEDY = dict(do_sample=False, repetition_penalty=10.0)


@pytest.fixture(scope="module")
def rig(engine):
    cfg = synth.gpt_config()
    w = synth.make_gpt_weights(cfg, seed=2025, bf16=True)
    engine.load_state_dict("gpt.", w)

    def init(bf16=True):
        engine.gpt_init(cfg["layers"], cfg["model_dim"], cfg["heads"], cfg["number_mel_codes"], cfg["start_mel_token"],
                        cfg["stop_mel_token"], cfg["max_mel_positions"], max_prompt=96, max_batch=8, weights_bf16=bf16)
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
    for i in range(N_REQ):                  # text lengths 16..71: prompts of different lengths
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
        lens = [len(x) for x in engine.gpt_generate(prompts, MAX_NEW, **GREEDY)]
        if len({n for n in lens if n < MAX_NEW}) >= 2:
            break
    print(f"stop-code bias +{add}: greedy lengths {lens}")
    tail = dict(prompt_condition=torch.randn(P, 512, generator=g).numpy(),
                ref_mel=(torch.randn(80, P, generator=g) * 1.5 - 4.0).numpy(), style=style)
    tail2 = dict(prompt_condition=torch.randn(P2, 512, generator=g).numpy(),
                 ref_mel=(torch.randn(80, P2, generator=g) * 1.5 - 4.0).numpy(), style=torch.randn(192, generator=g).numpy())
    return dict(cfg=cfg, prompts=prompts, tail=tail, tail2=tail2, lens=lens, init=init)


STEPS = (1, 3, 7, 16, 40)


def _serve(engine, prompts, slots, order=None, between=None, cancel=None, **kw):
    """Serve the requests through one group: at each next return at most one waiting request (in `order`, sequence index =
    its position in `prompts`) is admitted into the lowest free slot, each live slot asks for a varied number of further
    codes, finished slots are released.  cancel: {request: codes after which it is released live}.  Returns each
    request's codes."""
    order = list(range(len(prompts))) if order is None else list(order)
    out, who, rnd = {}, [None] * slots, 0
    with engine.gpt_serve(slots, MAX_NEW, **kw) as sv:
        while order or any(w is not None for w in who):
            free = [s for s in range(slots) if who[s] is None]
            if free and order:
                i = order.pop(0)
                sv.admit(free[0], prompts[i], i)
                who[free[0]] = i
            until = [sv.n_committed[s] + STEPS[(s + rnd) % len(STEPS)] if who[s] is not None else 0 for s in range(slots)]
            fin0 = list(sv.finished)
            new, fin = sv.next(until)
            rnd += 1
            live = [s for s in range(slots) if who[s] is not None and not fin[s]]
            newly = any(who[s] is not None and fin[s] and not fin0[s] for s in range(slots))
            if live and not newly:            # the call ends at the smallest until of the live slots
                assert min(until[s] - sv.n_committed[s] for s in live) == 0
            for s in range(slots):
                i = who[s]
                if i is None:
                    assert new[s] is None
                    continue
                if fin[s] or (cancel and i in cancel and sv.n_committed[s] >= cancel[i]):
                    out[i] = sv.codes[s].copy()
                    sv.release(s)
                    who[s] = None
            if between is not None:
                between()
    return [out[i] for i in range(len(prompts)) if i in out]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("name,kw", [("greedy", GREEDY), ("sample", SAMPLE)])
@pytest.mark.parametrize("slots", [4, 8])
def test_admitted_requests_decode_what_generate_decodes(engine, rig, slots, name, kw, mode):
    prompts = rig["prompts"]
    ref = engine.gpt_generate(prompts, MAX_NEW, mel_pos_mode=mode, **kw)
    got = _serve(engine, prompts, slots, mel_pos_mode=mode, **kw)
    for i in range(N_REQ):
        np.testing.assert_array_equal(got[i], ref[i], err_msg=f"{name} mode {mode} slots {slots} request {i}")
    print(f"slots {slots} {name} mode {mode}: lengths {[len(r) for r in ref]}")


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [GREEDY, SAMPLE])
def test_reused_slot_decodes_as_a_fresh_one(engine, rig, kw):
    prompts = rig["prompts"]
    ref = engine.gpt_generate(prompts, MAX_NEW, **kw)
    long_i = max(range(N_REQ), key=lambda i: (len(ref[i]), len(prompts[i])))
    short_i = min(i for i in range(N_REQ) if len(prompts[i]) < len(prompts[long_i]))
    with engine.gpt_serve(2, MAX_NEW, **kw) as sv:
        sv.admit(0, prompts[long_i], long_i)
        sv.admit(1, prompts[short_i], short_i)
        while not sv.finished[0]:
            sv.next([sv.n_committed[0] + 9, sv.n_committed[1] + 5 if not sv.finished[1] else 1])
        np.testing.assert_array_equal(sv.codes[0], ref[long_i])
        sv.release(0)                      # the longer request's prompt and codes stay in the slot's cache rows
        sv.admit(0, prompts[short_i], short_i)
        while not sv.finished[0]:
            sv.next([sv.n_committed[0] + 11, sv.n_committed[1] + 3 if not sv.finished[1] else 1])
        reused = sv.codes[0].copy()
    with engine.gpt_serve(2, MAX_NEW, **kw) as sv:
        sv.admit(1, prompts[short_i], short_i)
        while not sv.finished[1]:
            sv.next([1, MAX_NEW])
        fresh = sv.codes[1].copy()
    np.testing.assert_array_equal(reused, fresh)
    np.testing.assert_array_equal(reused, ref[short_i])


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [GREEDY, SAMPLE])
def test_cancel_leaves_the_other_rows_unchanged(engine, rig, kw):
    prompts = rig["prompts"]
    ref = engine.gpt_generate(prompts, MAX_NEW, **kw)
    cancel = {1: 10, 4: 1, 6: 33}
    got = _serve(engine, prompts, 4, cancel=cancel, **kw)
    for i in range(N_REQ):
        if i in cancel and len(got[i]) < len(ref[i]):
            np.testing.assert_array_equal(got[i], ref[i][:len(got[i])])      # the cancelled request's committed codes
        else:
            np.testing.assert_array_equal(got[i], ref[i], err_msg=f"request {i}")


def _window(rng, t, n):
    from indextts_b200.streaming import window_frames
    codes = rng.integers(0, 8192, n).astype(np.int32)
    F = window_frames(n)
    z = rng.standard_normal((80, t["ref_mel"].shape[-1] + F)).astype(np.float32)
    return dict(codes=codes, prompt_condition=t["prompt_condition"], ref_mel=t["ref_mel"], style=t["style"], z=z, F=F)


@pytest.mark.gpu
def test_tail_calls_between_next_calls_change_nothing(engine, rig):
    from indextts_b200.streaming import overlap_samples
    rng = np.random.default_rng(3)
    t, t2 = rig["tail"], rig["tail2"]
    w0, w1 = _window(rng, t, 30), _window(rng, t2, 30)

    def tail():
        engine.codes_to_wav(**w0, want_wav=True)
        engine.stream_vocode_batch([dict(w0, slot=0, first=True, overlap_samples=overlap_samples(5)),
                                    dict(w1, slot=1, first=True, last=True)])

    prompts = rig["prompts"]
    ref = engine.gpt_generate(prompts, MAX_NEW, **SAMPLE)
    busy = _serve(engine, prompts, 4, between=tail, **SAMPLE)
    for i in range(N_REQ):
        np.testing.assert_array_equal(busy[i], ref[i])


def _np(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _close(got, want, what):
    got = _np(got)
    assert got.dtype == np.int16 and len(got) == len(want), (what, len(got), len(want))
    assert int(np.abs(got.astype(np.int32) - want.astype(np.int32)).max(initial=0)) <= 1, what


@pytest.mark.gpu
def test_stream_server_end_to_end(engine, rig):
    from indextts_b200 import streaming
    prompts = [rig["prompts"][i] for i in (0, 4, 7, 9, 2, 11)]
    spk = [rig["tail"], rig["tail2"]] * 3
    chunk, ov = 40, 10
    ovlp = streaming.overlap_samples(ov)
    ref = engine.gpt_generate(prompts, MAX_NEW, **SAMPLE)
    arrive = {0: [0, 1], 2: [2], 3: [3, 4], 6: [5]}           # round -> requests submitted before it
    cancel_at, cancelled = 5, 3                                 # request 3 is cancelled before round 5
    calls, orig = [], engine.stream_vocode_batch
    srv = streaming.StreamServer(engine, slots=3, chunk_codes=chunk, overlap_codes=ov, max_new_tokens=MAX_NEW, **SAMPLE)

    def spy(windows, *a, **k):
        calls.append([dict(rid=srv._slot[w["slot"]], z=None if w.get("codes") is None else np.array(w["z"]), F=w.get("F"),
                           codes=None if w.get("codes") is None else np.array(w["codes"]), first=w.get("first"),
                           last=w.get("last")) for w in windows])
        return orig(windows, *a, **k)
    engine.stream_vocode_batch = spy
    got, n_done, submitted, r = {}, {}, 0, 0
    try:
        torch.manual_seed(1234)
        with srv:
            while submitted < len(prompts) or srv.busy:
                for i in arrive.get(r, []):
                    s = spk[i]
                    assert srv.submit(prompts[i], s["prompt_condition"], s["ref_mel"], s["style"]) == i
                    submitted += 1
                if r == cancel_at:
                    assert srv.cancel(cancelled)
                for rid, pcm, done in srv.round():
                    assert rid < submitted, "audio before the request was submitted"
                    assert n_done.get(rid, 0) == 0, "event after done"
                    assert not (rid == cancelled and r >= cancel_at), "event after the cancel"
                    if pcm is not None:
                        got.setdefault(rid, []).append(_np(pcm))
                    n_done[rid] = n_done.get(rid, 0) + done
                r += 1
                assert r < 1000
    finally:
        del engine.stream_vocode_batch
    assert sorted(k for k, v in n_done.items() if v) == [i for i in range(len(prompts)) if i != cancelled]
    assert all(v == 1 for k, v in n_done.items() if k != cancelled)
    # the noise: torch.randn(80, P + F) per window, in round order and slot order within a round
    torch.manual_seed(1234)
    for call in calls:
        for w in call:
            if w["z"] is not None:
                z = torch.randn(80, int(spk[w["rid"]]["ref_mel"].shape[-1]) + w["F"]).numpy()
                assert z.tobytes() == w["z"].tobytes()
    for i in range(len(prompts)):
        if i == cancelled:
            continue
        codes = ref[i]
        n = int(np.flatnonzero(codes == STOP)[0]) if (codes == STOP).any() else len(codes)
        sched = streaming.schedule(n, chunk, ov)
        mine = [w for call in calls for w in call if w["rid"] == i]
        hj, want = HostJoin(), []
        for k, w in enumerate(mine):
            if w["codes"] is None:
                assert k == len(sched) and (not sched or not sched[-1][2])
                want.append(hj.flush())
                continue
            a, b, last = sched[k]
            assert w["first"] == (k == 0) and w["last"] == last
            np.testing.assert_array_equal(w["codes"], codes[a:b])
            s = spk[i]
            wav = np.asarray(engine.codes_to_wav(w["codes"], s["prompt_condition"], s["ref_mel"], s["style"], w["z"],
                                                 w["F"])["wav"])
            want.append(hj.push(wav, ovlp, first=k == 0, last=last))
        want = np.concatenate(want) if want else np.zeros(0, np.int16)
        _close(np.concatenate(got[i]) if got.get(i) else np.zeros(0, np.int16), want, f"request {i}")
        print(f"request {i}: {n} codes, {len(mine)} windows, {len(want)} samples")


def _rc(fn, *a, **k):
    with pytest.raises(RuntimeError) as ex:
        fn(*a, **k)
    return int(str(ex.value).split("failed (")[1].split(")")[0])


@pytest.mark.gpu
def test_refusals_leave_the_group_usable(engine, rig):
    from indextts_b200.engine import GptRequest
    lib, h, prompts = engine.lib, engine.h, rig["prompts"]
    assert _rc(engine.gpt_serve, 4, 40, **dict(SAMPLE, num_beams=2)) == 2
    assert _rc(engine.gpt_serve, 4, 40, do_sample=True, top_k=0) == 2          # refused by the sampler checks
    assert _rc(engine.gpt_serve, 1, 40) == 2
    assert _rc(engine.gpt_serve, 9, 40) == 2
    assert lib.idx_gpt_serve_admit(h, 0, C.byref(GptRequest()), 0) == 3         # no open group
    try:
        os.environ["IDX_GPT_V8"] = "0"
        rig["init"]()
        assert _rc(engine.gpt_serve, 4, 40) == 2                                  # no gpt_decode8_kernel
        del os.environ["IDX_GPT_V8"]
        rig["init"](bf16=False)
        assert _rc(engine.gpt_serve, 4, 40) == 2                                  # the strict fp32 path
    finally:
        os.environ.pop("IDX_GPT_V8", None)
        rig["init"]()
    ref = engine.gpt_generate(prompts[:3], 40, **SAMPLE)
    sv = engine.gpt_serve(4, 40, **SAMPLE)
    try:
        sv.admit(2, prompts[0], 0)
        sv.next([0, 0, 5, 0])
        assert _rc(sv.admit, 4, prompts[1], 1) == 2                               # slot out of range
        assert _rc(sv.admit, -1, prompts[1], 1) == 2
        assert _rc(sv.admit, 2, prompts[1], 1) == 2                               # occupied
        assert _rc(sv.admit, 0, prompts[1], -1) == 2                              # seq_index < 0
        too_long = np.zeros((97, prompts[1].shape[1]), np.float32)                # max_prompt 96
        assert _rc(sv.admit, 0, too_long, 1) == 2
        # prompt_len + max_new_tokens + 1 > KV positions cannot be reached through the API: the KV cache has
        # max_prompt + max_mel_positions + 8 positions, begin refuses max_new_tokens + 2 > max_mel_positions and admit
        # refuses prompt_len > max_prompt, so prompt_len + max_new_tokens + 1 <= max_prompt + max_mel_positions - 1
        fc = np.zeros(40, np.int32)
        req = GptRequest()
        req.prompt_emb, req.prompt_len, req.forced_codes = prompts[1].ctypes.data, prompts[1].shape[0], fc.ctypes.data
        assert lib.idx_gpt_serve_admit(h, 0, C.byref(req), 1) == 2                # forced_codes
        assert _rc(sv.release, 1) == 2                                            # empty slot
        assert _rc(engine.gpt_serve, 4, 40) == 3                                  # a second group
        assert _rc(engine.gpt_generate, [prompts[0]], 40) == 3
        assert _rc(engine.gpt_stream, prompts[0], 40) == 3
        u = (C.c_int32 * 4)(5, 5, 5, 5)
        bufs = [np.zeros(40, np.int32) for _ in range(4)]
        outs = (C.c_void_p * 4)(*[b.ctypes.data for b in bufs])
        assert lib.idx_gpt_stream_next_batch(h, u, outs, None, None) == 3       # not a plain stream
        assert sv.occupied == [False, False, True, False] and sv.n_committed[2] == min(5, len(ref[0]))
        sv.admit(0, prompts[1], 1)
        sv.admit(3, prompts[2], 2)
        while not all(sv.finished[s] for s in (0, 2, 3)):
            sv.next([40] * 4)
        for s, i in ((0, 1), (2, 0), (3, 2)):
            np.testing.assert_array_equal(sv.codes[s], ref[i])
    finally:
        sv.close()
