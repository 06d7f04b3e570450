"""Latency of chunked streaming (indextts_b200.streaming.stream_segment) on a BASELINE config-2 segment: 10 s prompt
(P = 861 frames), 256 speech tokens with forbid_stop_before = 256, greedy, chunk 100 / overlap 20 codes (StreamingDecoder's
defaults), 25 Euler steps, CFG 0.7; synthetic weights at the real geometry (bench.build_engine).

    python -m tests.tools.stream_latency OUT_DIR [--repeats 5]

Per repetition, on synchronized host clocks (every engine call returns after its last copy): the time from the start of
the segment to the first emitted int16 chunk, the time of each window's tail call, and the total stream time; against it
the whole segment as gpt_generate + codes_to_wav.  One warm-up repetition of each runs first.  Prints the medians with the
card's name and power limit read in the same run, and writes OUT_DIR/stream_latency.json."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from tests.tools.tail_batch_bench import gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    from indextts_b200 import streaming
    e, cfg, wg, _ = bench.build_engine(0)
    inp = bench.make_inputs(0, cfg, wg)
    prompt = e.gpt_prepare_inputs(inp["style"].numpy(), inp["emo"].numpy(), inp["text"].numpy(), 1)
    pc, mel, style = inp["prompt_condition"].numpy(), inp["ref_mel"].numpy(), inp["style"].numpy()
    n_tok = bench.N_TOKENS
    gen = dict(max_new_tokens=n_tok, forbid_stop_before=n_tok, repetition_penalty=10.0)

    def one_stream():
        # the window tails are timed by wrapping stream_vocode: the generator runs them serially on the engine stream
        tails, orig = [], e.stream_vocode

        def timed(*a, **k):
            t = time.perf_counter()
            r = orig(*a, **k)
            tails.append(time.perf_counter() - t)
            return r
        e.stream_vocode = timed
        try:
            e.sync()
            t0 = time.perf_counter()
            first, samples, chunks = None, 0, 0
            for pcm in streaming.stream_segment(e, prompt, pc, mel, style, chunk_codes=100, overlap_codes=20, **gen):
                if first is None and len(pcm):
                    first = time.perf_counter() - t0
                samples += len(pcm)
                chunks += 1
            total = time.perf_counter() - t0
        finally:
            del e.stream_vocode
        return dict(first_ms=first * 1e3, total_ms=total * 1e3, tail_ms=[x * 1e3 for x in tails], samples=samples, chunks=chunks)

    def one_whole():
        e.sync()
        t0 = time.perf_counter()
        (codes,) = e.gpt_generate([prompt], n_tok, 10.0, forbid_stop_before=n_tok)
        t1 = time.perf_counter()
        F = int(2 * len(codes) * 1.72)
        z = torch.randn(80, inp["ref_mel"].shape[-1] + F).numpy()
        e.codes_to_wav(codes, pc, mel, style, z, F, bench.CFM_STEPS, bench.CFG_RATE, want_wav=False, want_pcm16=True)
        t2 = time.perf_counter()
        return dict(gpt_ms=(t1 - t0) * 1e3, tail_ms=(t2 - t1) * 1e3, total_ms=(t2 - t0) * 1e3, samples=F * 256)

    one_stream(), one_whole()                     # warm-up: arenas, stream buffers, every shape
    streams, wholes = [], []
    for _ in range(args.repeats):
        streams.append(one_stream())
        wholes.append(one_whole())
    med = lambda xs: float(np.median(xs))
    res = dict(
        gpu=gpu_info(), repeats=args.repeats, segment=dict(prompt_frames=bench.P_FRAMES, tokens=n_tok, chunk_codes=100,
                                                           overlap_codes=20, cfm_steps=bench.CFM_STEPS),
        stream=dict(first_sample_ms=med([s["first_ms"] for s in streams]), total_ms=med([s["total_ms"] for s in streams]),
                    window_tail_ms=[med(col) for col in zip(*[s["tail_ms"] for s in streams])],
                    samples=streams[-1]["samples"], chunks=streams[-1]["chunks"]),
        whole=dict(gpt_ms=med([w["gpt_ms"] for w in wholes]), tail_ms=med([w["tail_ms"] for w in wholes]),
                   total_ms=med([w["total_ms"] for w in wholes]), samples=wholes[-1]["samples"]),
        raw=dict(stream=streams, whole=wholes))
    g = res["gpu"]
    print(f"GPU: {g.get('name')}, power limit {g.get('power_limit')}")
    s, w = res["stream"], res["whole"]
    print(f"stream: first sample after {s['first_sample_ms']:.1f} ms; window tails "
          f"{', '.join(f'{x:.1f}' for x in s['window_tail_ms'])} ms; total {s['total_ms']:.1f} ms, {s['samples']} samples in "
          f"{s['chunks']} chunks (median of {args.repeats})")
    print(f"whole segment: gpt_generate {w['gpt_ms']:.1f} ms + codes_to_wav {w['tail_ms']:.1f} ms = {w['total_ms']:.1f} ms "
          f"before the first sample, {w['samples']} samples")
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "stream_latency.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
