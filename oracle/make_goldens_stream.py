"""Mint tests/golden/stream_join.npz from the reference's own StreamingDecoder (run in the build container only: needs
/root/reference).  `backends/trt/pipeline/streaming.py:StreamingDecoder.generate` runs with a fake gpt_engine whose
generate_chunks yields the chosen windows and a fake codes_to_audio_fn that returns seeded window audio; the windows and
the int16 chunks the decoder yields are stored, so that the host model of the join in tests/stream_refs.py (and through
it the device join of idx_stream_vocode) can be checked anywhere (tests/test_stream_cpu.py).

Cases: several windows, a last window shorter than the overlap, overlap 0 (pure concatenation, then the flush), a single
window, a stream that ends without a last window (the flush of a kept tail), a last chunk of at most 512 samples, and the
default overlap of 20 codes.

    python -m oracle.make_goldens_stream
"""
import importlib.util
import os

import numpy as np

REF = os.environ.get("IDX_REFERENCE", "/root/reference")
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "stream_join.npz")

# name: (overlap_size in codes, window lengths in samples, is_last per window)
CASES = {
    "multi": (2, [2000, 2500, 1900, 1200], [False, False, False, True]),
    "short_last": (3, [3000, 2800, 700], [False, False, True]),
    "overlap0": (0, [1000, 1500, 800], [False, False, False]),
    "single": (2, [1700], [True]),
    "flush": (2, [2000, 2100], [False, False]),
    "tiny_last": (1, [600, 300], [False, True]),
    "default20": (20, [22408, 22408, 9000], [False, False, True]),
}


def load_streaming():
    spec = importlib.util.spec_from_file_location("ref_trt_streaming", os.path.join(REF, "backends", "trt", "pipeline",
                                                                                    "streaming.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class FakeGpt:
    def __init__(self, lens, lasts):
        self.lens, self.lasts = lens, lasts

    def generate_chunks(self, **kw):
        for n, last in zip(self.lens, self.lasts):
            codes = np.zeros((1, max(1, n // 256)), np.int32)
            yield codes, None, last, [False], np.array([codes.shape[1]])


def main():
    sd = load_streaming()
    rng = np.random.default_rng(2025)
    out = {}
    for name, (ov, lens, lasts) in CASES.items():
        audio = []
        for n in lens:
            a = (rng.uniform(-1.0, 1.0, n) * 0.95).astype(np.float32)
            a[rng.integers(0, n, 4)] = np.float32(1.0)
            a[rng.integers(0, n, 4)] = np.float32(-1.0)
            audio.append(a)
        it = iter(audio)
        dec = sd.StreamingDecoder(FakeGpt(lens, lasts), lambda *a, **k: [next(it)], chunk_size=ov + 1, overlap_size=ov)
        chunks = [o[1][0] for o in dec.generate(np.zeros((1, 1, 1), np.float32), None, 0, None, None, None)]
        out[name + "_ovlp"] = np.int64(sd.overlap_samples(ov))
        out[name + "_win_lens"] = np.asarray(lens, np.int64)
        out[name + "_win_last"] = np.asarray(lasts, bool)
        out[name + "_audio"] = np.concatenate(audio)
        out[name + "_out_lens"] = np.asarray([len(c) for c in chunks], np.int64)
        out[name + "_out"] = np.concatenate(chunks).astype(np.int16)
        print(f"{name}: ovlp {int(out[name + '_ovlp'])}, {len(lens)} windows -> chunks {[len(c) for c in chunks]}")
    np.savez(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
