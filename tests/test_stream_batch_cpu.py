"""Batched chunked streaming on the host: a per-slot host model of the join with the None / done bookkeeping of
indextts_b200.streaming.stream_segments against the reference's own batch StreamingDecoder output
(tests/golden/stream_join_batch.npz, minted by oracle/make_goldens_stream_batch.py), and each sample's windows in the
batch loop of generate_chunks against the solo window schedule."""
import os

import numpy as np
import pytest

from tests.stream_refs import HostJoin

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "stream_join_batch.npz")
CASES = ["early", "on_end", "flush", "overlap0", "wide"]


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.mark.parametrize("case", CASES)
def test_host_join_reproduces_reference_batch_rounds(golden, case):
    g = {k[len(case) + 1:]: golden[k] for k in golden.files if k.startswith(case + "_")}
    ovlp, in_lens, bdone, is_last = int(g["ovlp"]), g["in_lens"], g["batch_done"], g["is_last"]
    R, B = in_lens.shape
    audio, ai = g["audio"], 0
    pcm, pi = g["out"], 0
    joins = [HostJoin() for _ in range(B)]
    started, ended = [False] * B, [False] * B
    n_done = np.zeros(B, int)
    for r in range(R):
        flush_round = bool((in_lens[r] < 0).all())
        got, done = [None] * B, [False] * B
        for b in range(B):
            if flush_round:
                if started[b] and not ended[b]:
                    got[b], done[b] = joins[b].flush(), True
            else:
                wav = audio[ai:ai + in_lens[r, b]]
                ai += in_lens[r, b]
                if ended[b]:
                    continue
                last = bool(bdone[r, b] or is_last[r])
                got[b] = joins[b].push(wav, ovlp, first=not started[b], last=last)
                started[b], done[b] = True, last
            ended[b] = ended[b] or done[b]
        for b in range(B):
            want_len = int(g["out_lens"][r, b])
            if want_len < 0:
                assert got[b] is None, (case, r, b)
                continue
            want = pcm[pi:pi + want_len]
            pi += want_len
            assert got[b] is not None and got[b].dtype == np.int16, (case, r, b)
            np.testing.assert_array_equal(got[b], want, err_msg=f"{case} round {r} sample {b}")
        assert done == [bool(x) for x in g["done"][r]], (case, r)
        n_done += done
    assert ai == len(audio) and pi == len(pcm)
    assert (n_done == 1).all(), "done arrives exactly once per sample"


def generate_chunks_batch(lens, chunk, overlap, max_new):
    """Each sample's windows (start, end, last) in the batch loop of generate_chunks (gpt_trtllm_runtime.py:381-519): a
    shared next_chunk_at over max(sample_len), batch_done flags and chunk_code_lens; sample b's stop token follows its
    lens[b] codes.  A sample whose last window is empty (chunk_code_lens 0) or that never gets one ends with the flush."""
    stride = chunk - overlap
    B = len(lens)
    done, slen, fin = [False] * B, [0] * B, [False] * B
    out = [[] for _ in range(B)]
    next_at, step = chunk, 0

    def emit(pos, end, flags, code_lens):
        for b in range(B):
            if fin[b]:
                continue
            if code_lens[b] > 0:
                out[b].append((pos, pos + code_lens[b], bool(flags[b])))
            fin[b] = bool(flags[b])

    while step < max_new:
        step += 1
        for b in range(B):
            if not done[b]:
                if step - 1 == lens[b]:
                    done[b], slen[b] = True, step - 1
                else:
                    slen[b] = step
        cur = max(slen)
        while cur >= next_at:
            pos = next_at - chunk
            emit(pos, next_at, [done[b] and slen[b] <= next_at for b in range(B)],
                 [max(0, min(slen[b] - pos, chunk)) for b in range(B)])
            next_at += stride
        if all(done):
            break
    pos = next_at - chunk
    if pos < max(slen):
        emit(pos, max(slen), [True] * B, [max(0, slen[b] - pos) for b in range(B)])
    return out


@pytest.mark.parametrize("chunk,overlap", [(100, 20), (100, 0), (30, 10), (7, 3), (5, 4)])
def test_batch_windows_equal_solo_schedule(chunk, overlap):
    from indextts_b200.streaming import schedule
    rng = np.random.default_rng(chunk * 100 + overlap)
    stride = chunk - overlap
    ends = [chunk + k * stride for k in range(6)]
    for trial in range(40):
        B = int(rng.integers(2, 9))
        lens = [int(rng.choice(ends)) if rng.random() < 0.4 else int(rng.integers(0, chunk + 6 * stride)) for _ in range(B)]
        got = generate_chunks_batch(lens, chunk, overlap, max_new=10_000)
        for b in range(B):
            want = schedule(lens[b], chunk, overlap)
            assert got[b] == want, (lens, b)
