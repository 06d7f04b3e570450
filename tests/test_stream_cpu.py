"""Chunked streaming on the host: the window schedule of indextts_b200.streaming against a restatement of the
reference's generate_chunks, and the host model of the window join against the reference's own StreamingDecoder output
(tests/golden/stream_join.npz, minted by oracle/make_goldens_stream.py)."""
import os

import numpy as np
import pytest

from tests.stream_refs import HostJoin

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "stream_join.npz")
STOP = 8193


def generate_chunks_windows(codes, chunk, overlap, max_new):
    """The windows (start, end, is_last) generate_chunks (backends/trt/runtime/gpt_trtllm_runtime.py:381-519) yields for one
    sequence, token by token: `codes` is the decoded sequence (stop token included when produced)."""
    stride = chunk - overlap
    if stride <= 0:
        raise ValueError("overlap must be less than chunk")
    out, next_at, done, length = [], chunk, False, 0
    for step in range(1, min(len(codes), max_new) + 1):
        if not done:
            if codes[step - 1] == STOP:
                done, length = True, step - 1
            else:
                length = step
        while length >= next_at:
            out.append((next_at - chunk, next_at, False))
            next_at += stride
        if done:
            break
    pos = next_at - chunk
    if pos < length:
        out.append((pos, length, True))
    return out


def streaming_windows(codes, chunk, overlap, increments):
    """The windows stream_segment runs when the committed codes arrive in the given increments."""
    from indextts_b200.streaming import WindowSchedule
    ws = WindowSchedule(chunk, overlap)
    stops = np.flatnonzero(np.asarray(codes) == STOP)
    stop_at = int(stops[0]) if stops.size else len(codes)
    out, have, n = [], 0, 0
    for inc in increments:
        have = min(len(codes), have + inc)
        n = min(have, stop_at)                          # the committed codes cut before the stop token
        out += [(a, b, False) for a, b in ws.ready(n)]
        if have > stop_at or have == len(codes):
            break
    fin = ws.final(n)
    if fin is not None:
        out.append((fin[0], fin[1], True))
    return out


PAIRS = [(100, 20), (100, 0), (30, 10), (7, 3), (50, 49), (1, 0)]


@pytest.mark.parametrize("chunk,overlap", PAIRS)
def test_schedule_matches_generate_chunks(chunk, overlap):
    rng = np.random.default_rng(chunk * 1000 + overlap)
    for n in range(1, 601):
        for stop in (True, False):                      # a stop token after n codes, or max_new_tokens = n reached
            codes = list(rng.integers(0, 8192, n)) + ([STOP] if stop else [])
            want = generate_chunks_windows(codes, chunk, overlap, len(codes))
            for inc in (1, 7, 64, 100):                   # commits arrive in steps (the beam path commits in bursts)
                assert streaming_windows(codes, chunk, overlap, [inc] * (len(codes) // inc + 2)) == want, (n, stop, inc)


def test_schedule_edges():
    from indextts_b200.streaming import schedule
    assert schedule(100) == [(0, 100, False), (80, 100, True)]       # ends on a window boundary: a last overlap window
    assert schedule(60) == [(0, 60, True)]                           # shorter than one chunk: one last window
    assert schedule(100, 100, 0) == [(0, 100, False)]                # overlap 0 on a boundary: no last window (flush)
    assert schedule(0) == []
    assert schedule(260) == [(0, 100, False), (80, 180, False), (160, 260, False), (240, 260, True)]
    with pytest.raises(ValueError):
        schedule(10, 20, 20)


def test_overlap_rule_is_the_codec_frame_rule():
    from indextts_b200.streaming import overlap_samples, window_frames
    assert overlap_samples(20) == int(2 * 20 * 1.72) * 256 == 68 * 256
    assert window_frames(100, 1.1) == int(2 * 100 * 1.72 * 1.1)


def test_host_join_reproduces_reference_decoder():
    g = np.load(GOLDEN)
    names = sorted({k[:-len("_ovlp")] for k in g.files if k.endswith("_ovlp")})
    assert len(names) == 7
    for name in names:
        ovlp = int(g[name + "_ovlp"])
        lens, lasts, audio = g[name + "_win_lens"], g[name + "_win_last"], g[name + "_audio"]
        want_lens, want = g[name + "_out_lens"], g[name + "_out"]
        hj, outs, o = HostJoin(), [], 0
        for i, (n, last) in enumerate(zip(lens, lasts)):
            outs.append(hj.push(audio[o:o + n], ovlp, first=(i == 0), last=bool(last)))
            o += n
        fl = hj.flush()
        if fl is not None:
            outs.append(fl)
        assert [len(x) for x in outs] == list(want_lens), name
        np.testing.assert_array_equal(np.concatenate(outs), want, err_msg=name)
