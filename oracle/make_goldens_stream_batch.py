"""Mint tests/golden/stream_join_batch.npz from the reference's own StreamingDecoder in batch mode (needs the reference
checkout, found as in oracle/make_goldens_stream.py).  `backends/trt/pipeline/streaming.py:StreamingDecoder.generate` runs with a fake
gpt_engine whose generate_chunks restates the batch loop of gpt_trtllm_runtime.py:381-519 for chosen per-sample code
lengths (a shared next_chunk_at, batch_done flags, chunk_code_lens), and a fake codes_to_audio_fn that returns seeded
audio of chunk_code_lens[b] * 256 samples per sample.  Each round's inputs and the (audio_list, done_list) the decoder
yields are stored, so that the per-slot host model of the join and the None / done bookkeeping of
indextts_b200.streaming.stream_segments can be checked anywhere (tests/test_stream_batch_cpu.py).

Cases: a sample that finishes two rounds before the others, a sample whose length falls exactly on a window end, the
final flush of several kept tails (overlap 0, samples ending on a window end), overlap 0 with partial windows, and an
overlap of 768 samples (2 of 10 codes).

    python -m oracle.make_goldens_stream_batch
"""
import os

import numpy as np

from oracle.make_goldens_stream import load_streaming

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "stream_join_batch.npz")
K = 256           # samples per code of the fake vocoder
STOP = 8193

# name: (chunk codes, overlap codes, code lengths per sample)
CASES = {
    "early": (4, 1, [5, 13, 12]),
    "on_end": (4, 1, [7, 11, 9]),
    "flush": (3, 0, [9, 9, 6]),
    "overlap0": (3, 0, [7, 5, 8]),
    "wide": (10, 2, [23, 17, 12]),
}


class FakeGpt:
    """generate_chunks of the TensorRT runtime for samples whose stop token comes right after lens[b] codes."""

    def __init__(self, lens):
        self.lens = lens

    def generate_chunks(self, chunk_size, overlap_size, max_new_tokens=1500, **kw):
        stride = chunk_size - overlap_size
        B = len(self.lens)
        codes = np.full((B, max_new_tokens), STOP, np.int32)
        sample_done, sample_len = [False] * B, [0] * B
        next_chunk_at, step_count = chunk_size, 0
        while step_count < max_new_tokens:
            step_count += 1
            for b in range(B):
                if step_count - 1 < self.lens[b]:
                    codes[b, step_count - 1] = 1
            for b in range(B):
                if not sample_done[b]:
                    if codes[b, step_count - 1] == STOP:
                        sample_done[b], sample_len[b] = True, step_count - 1
                    else:
                        sample_len[b] = step_count
            current_len = max(sample_len)
            while current_len >= next_chunk_at:
                pos = next_chunk_at - chunk_size
                flags = [sample_done[b] and sample_len[b] <= next_chunk_at for b in range(B)]
                lens = np.array([max(0, min(sample_len[b] - pos, chunk_size)) for b in range(B)])
                yield codes[:, pos:next_chunk_at], None, False, flags, lens
                next_chunk_at += stride
            if all(sample_done):
                break
        current_len = max(sample_len)
        pos = next_chunk_at - chunk_size
        if pos < current_len:
            lens = np.array([max(0, sample_len[b] - pos) for b in range(B)])
            yield codes[:, pos:current_len], None, True, [True] * B, lens


def main():
    sd = load_streaming()
    rng = np.random.default_rng(2026)
    out = {}
    for name, (chunk, ov, lens) in CASES.items():
        B = len(lens)
        rounds = []          # per round: (audio per sample, batch_done, is_last)
        gen = FakeGpt(lens)

        class Recorder:
            def generate_chunks(self, **kw):
                for c, lat, last, flags, cl in gen.generate_chunks(**kw):
                    rounds.append([None, list(flags), bool(last), [int(x) for x in cl]])
                    yield c, lat, last, flags, cl

        def to_audio(codes, latent, code_lens, *a, **k):
            audio = []
            for n in code_lens:
                x = (rng.uniform(-1.0, 1.0, int(n) * K) * 0.95).astype(np.float32)
                if len(x):
                    x[rng.integers(0, len(x), 2)] = np.float32(1.0)
                audio.append(x)
            rounds[-1][0] = audio
            return audio

        dec = sd.StreamingDecoder(Recorder(), to_audio, chunk_size=chunk, overlap_size=ov)
        outs = list(dec.generate(np.zeros((B, 1, 1), np.float32), None, STOP, None, None, None, max_new_tokens=400))
        R = len(outs)
        in_lens = np.full((R, B), -1, np.int64)          # -1: the decoder's final flush round (no vocoder call)
        bdone, last = np.zeros((R, B), bool), np.zeros(R, bool)
        audio = []
        for r, (au, flags, is_last, _) in enumerate(rounds):
            in_lens[r] = [len(x) for x in au]
            bdone[r], last[r] = flags, is_last
            audio += au
        out_lens = np.full((R, B), -1, np.int64)          # -1: None
        done = np.zeros((R, B), bool)
        pcm = []
        for r, (_, al, dl) in enumerate(outs):
            for b in range(B):
                if al[b] is not None:
                    out_lens[r, b] = len(al[b])
                    pcm.append(al[b])
            done[r] = dl
        out[name + "_ovlp"] = np.int64(sd.overlap_samples(ov))
        out[name + "_in_lens"] = in_lens
        out[name + "_batch_done"] = bdone
        out[name + "_is_last"] = last
        out[name + "_audio"] = np.concatenate(audio) if audio else np.zeros(0, np.float32)
        out[name + "_out_lens"] = out_lens
        out[name + "_done"] = done
        out[name + "_out"] = np.concatenate(pcm).astype(np.int16)
        out[name + "_code_lens"] = np.asarray(lens, np.int64)
        out[name + "_chunk"] = np.int64(chunk)
        out[name + "_overlap"] = np.int64(ov)
        print(f"{name}: ovlp {int(out[name + '_ovlp'])}, {R} rounds, out lens {out_lens.tolist()}, done {done.astype(int).tolist()}")
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
