"""Latency of batched chunked streaming (indextts_b200.streaming.stream_segments) against the same segments streamed one
after another (stream_segment), on BASELINE config-2 segments: 10 s prompt (P = 861 frames), 256 speech tokens fixed by
forbid_stop_before = 256, chunk 100 / overlap 20 codes, 25 Euler steps, CFG 0.7; synthetic weights at the real geometry
(bench.build_engine with max_batch = 8).  n in {1, 2, 4, 8} greedy, and n = 2 with the beam-sample default (3 beams,
top_k 30, top_p 0.8, temperature 0.8).

    python -m tests.tools.stream_batch_latency OUT_DIR [--repeats 5]

Per repetition, on synchronized host clocks (every engine call returns after its last copy): per request the time from
the start to its first emitted samples, and the time of the whole batch; the two ways alternate, after one warm-up of
each.  Prints the medians with the card's name, power limit and max SM clock read in the same run, and writes
OUT_DIR/stream_batch_latency.json."""
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

BEAM_SAMPLE = dict(do_sample=True, num_beams=3, top_k=30, top_p=0.8, temperature=0.8, length_penalty=0.0, seed=3)
CASES = [("greedy", n, {}) for n in (1, 2, 4, 8)] + [("beam-sample", 2, BEAM_SAMPLE)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    from indextts_b200 import streaming
    e, cfg, wg, _ = bench.build_engine(0, max_batch=8)
    inp = bench.make_inputs(0, cfg, wg)
    pc, mel, style = inp["prompt_condition"].numpy(), inp["ref_mel"].numpy(), inp["style"].numpy()
    n_tok = bench.N_TOKENS
    prompts = []
    for i in range(8):       # the config-2 text with a different emotion vector per request
        g = torch.Generator().manual_seed(100 + i)
        emo = (inp["emo"] + 0.1 * torch.randn(inp["emo"].shape, generator=g)).numpy()
        prompts.append(e.gpt_prepare_inputs(style, emo, inp["text"].numpy(), 1))
    base = dict(chunk_codes=100, overlap_codes=20, max_new_tokens=n_tok, forbid_stop_before=n_tok, repetition_penalty=10.0)

    def batch(n, kw):
        e.sync()
        t0 = time.perf_counter()
        first = [None] * n
        for audio, _ in streaming.stream_segments(e, prompts[:n], pc, mel, style, **base, **kw):
            now = time.perf_counter() - t0
            for i in range(n):
                if first[i] is None and audio[i] is not None and len(audio[i]):
                    first[i] = now
        return dict(first_ms=[x * 1e3 for x in first], total_ms=(time.perf_counter() - t0) * 1e3)

    def serial(n, kw):
        e.sync()
        t0 = time.perf_counter()
        first = [None] * n
        for i in range(n):
            for pcm in streaming.stream_segment(e, prompts[i], pc, mel, style, **base, **kw):
                if first[i] is None and len(pcm):
                    first[i] = time.perf_counter() - t0
        return dict(first_ms=[x * 1e3 for x in first], total_ms=(time.perf_counter() - t0) * 1e3)

    med = lambda xs: float(np.median(xs))
    res = dict(gpu=gpu_info(), repeats=args.repeats,
               segment=dict(prompt_frames=bench.P_FRAMES, tokens=n_tok, chunk_codes=100, overlap_codes=20,
                            cfm_steps=bench.CFM_STEPS), cases=[])
    g = res["gpu"]
    print(f"GPU: {g.get('name')}, power limit {g.get('power_limit')}, max SM clock {g.get('max_sm_clock')}")
    for name, n, kw in CASES:
        batch(n, kw), serial(n, kw)                 # warm-up: arenas, stream buffers, every shape
        bs, ss = [], []
        for _ in range(args.repeats):
            bs.append(batch(n, kw))
            ss.append(serial(n, kw))
        row = dict(mode=name, n=n,
                   batch=dict(first_sample_ms=[med(c) for c in zip(*[b["first_ms"] for b in bs])],
                              total_ms=med([b["total_ms"] for b in bs])),
                   serial=dict(first_sample_ms=[med(c) for c in zip(*[s["first_ms"] for s in ss])],
                               total_ms=med([s["total_ms"] for s in ss])),
                   raw=dict(batch=bs, serial=ss))
        res["cases"].append(row)
        b, s = row["batch"], row["serial"]
        print(f"{name} n={n}: stream_segments first sample {', '.join(f'{x:.1f}' for x in b['first_sample_ms'])} ms, "
              f"all {b['total_ms']:.1f} ms | serial stream_segment first sample "
              f"{', '.join(f'{x:.1f}' for x in s['first_sample_ms'])} ms, all {s['total_ms']:.1f} ms "
              f"(median of {args.repeats})")
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "stream_batch_latency.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
