"""Latency of serving arriving requests: a StreamServer (requests join the running decode group as slots free up)
against stream_segments groups formed from whoever is waiting when the previous group ends.  BASELINE config-2 segments
(10 s prompt, P = 861 frames; 256 speech tokens fixed by forbid_stop_before = 256; chunk 100 / overlap 20 codes, 25 Euler
steps, CFG 0.7, greedy), synthetic weights at the real geometry (bench.build_engine with max_batch = 8), 8 slots, 16
requests arriving every --gap ms on the host clock.

    python -m tests.tools.stream_serve_latency OUT_DIR [--repeats 5] [--gap 100]

Per repetition, on synchronized host clocks (every engine call returns after its last copy): per request the time from
its arrival to its first emitted samples and to its last, the makespan (first arrival to last sample) and the host time
of each admission prefill (StreamServer) or group begin (stream_segments: the prefill of the whole group) during which
no request decodes.  The two ways alternate, after one warm-up of each.  Prints the medians over the repetitions with
the card's name, power limit and max SM clock read in the same run, and writes OUT_DIR/stream_serve_latency.json."""
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

N_REQ, SLOTS = 16, 8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--gap", type=float, default=100.0, help="ms between arrivals")
    args = ap.parse_args()
    from indextts_b200 import streaming
    e, cfg, wg, _ = bench.build_engine(0, max_batch=SLOTS)
    inp = bench.make_inputs(0, cfg, wg)
    pc, mel, style = inp["prompt_condition"].numpy(), inp["ref_mel"].numpy(), inp["style"].numpy()
    n_tok = bench.N_TOKENS
    prompts = []
    for i in range(N_REQ):       # the config-2 text with a different emotion vector per request
        g = torch.Generator().manual_seed(100 + i)
        emo = (inp["emo"] + 0.1 * torch.randn(inp["emo"].shape, generator=g)).numpy()
        prompts.append(e.gpt_prepare_inputs(style, emo, inp["text"].numpy(), 1))
    gen = dict(max_new_tokens=n_tok, forbid_stop_before=n_tok, repetition_penalty=10.0, seed=0)
    arrive = [i * args.gap * 1e-3 for i in range(N_REQ)]

    def wait_until(t0, t):
        d = t0 + t - time.perf_counter()
        if d > 0:
            time.sleep(d)

    def timed(obj, name, stalls):
        fn = getattr(obj, name)

        def wrap(*a, **k):
            t = time.perf_counter()
            r = fn(*a, **k)
            stalls.append((time.perf_counter() - t) * 1e3)
            return r
        setattr(obj, name, wrap)

    def server():
        e.sync()
        stalls, first, last = [], [None] * N_REQ, [None] * N_REQ
        srv = streaming.StreamServer(e, slots=SLOTS, chunk_codes=100, overlap_codes=20, **gen)
        timed(srv._gen, "admit", stalls)
        t0, nsub = time.perf_counter(), 0
        with srv:
            while nsub < N_REQ or srv.busy:
                now = time.perf_counter() - t0
                while nsub < N_REQ and arrive[nsub] <= now:
                    assert srv.submit(prompts[nsub], pc, mel, style) == nsub
                    nsub += 1
                if not srv.busy:
                    wait_until(t0, arrive[nsub])
                    continue
                for rid, pcm, done in srv.round():
                    now = time.perf_counter() - t0
                    if first[rid] is None and pcm is not None and len(pcm):
                        first[rid] = now
                    if done:
                        last[rid] = now
        return first, last, stalls

    def groups():
        e.sync()
        stalls, first, last = [], [None] * N_REQ, [None] * N_REQ
        timed(e, "gpt_stream_batch", stalls)
        t0, nxt = time.perf_counter(), 0
        try:
            while nxt < N_REQ:
                wait_until(t0, arrive[nxt])
                now = time.perf_counter() - t0
                grp = [i for i in range(nxt, N_REQ) if arrive[i] <= now][:SLOTS]
                nxt += len(grp)
                for audio, done in streaming.stream_segments(e, [prompts[i] for i in grp], pc, mel, style,
                                                             chunk_codes=100, overlap_codes=20, **gen):
                    now = time.perf_counter() - t0
                    for j, i in enumerate(grp):
                        if first[i] is None and audio[j] is not None and len(audio[j]):
                            first[i] = now
                        if done[j]:
                            last[i] = now
        finally:
            del e.gpt_stream_batch
        return first, last, stalls

    def summary(first, last, stalls):
        ttfs = [(f - a) * 1e3 for f, a in zip(first, arrive)]
        done = [(d - a) * 1e3 for d, a in zip(last, arrive)]
        return dict(first_sample_ms=ttfs, completion_ms=done, makespan_ms=max(last) * 1e3, stall_ms=stalls)

    med = lambda xs: float(np.median(xs))
    res = dict(gpu=gpu_info(), repeats=args.repeats, requests=N_REQ, slots=SLOTS, arrival_gap_ms=args.gap,
               segment=dict(prompt_frames=bench.P_FRAMES, tokens=n_tok, chunk_codes=100, overlap_codes=20,
                            cfm_steps=bench.CFM_STEPS), raw=dict(server=[], groups=[]))
    gi = res["gpu"]
    print(f"GPU: {gi.get('name')}, power limit {gi.get('power_limit')}, max SM clock {gi.get('max_sm_clock')}")
    server(), groups()                                   # warm-up: arenas, stream buffers, every shape
    for _ in range(args.repeats):
        res["raw"]["server"].append(summary(*server()))
        res["raw"]["groups"].append(summary(*groups()))
    for way in ("server", "groups"):
        runs = res["raw"][way]
        row = dict(first_sample_median_ms=med([med(r["first_sample_ms"]) for r in runs]),
                   first_sample_worst_ms=med([max(r["first_sample_ms"]) for r in runs]),
                   completion_median_ms=med([med(r["completion_ms"]) for r in runs]),
                   completion_worst_ms=med([max(r["completion_ms"]) for r in runs]),
                   makespan_ms=med([r["makespan_ms"] for r in runs]),
                   stall_median_ms=med([med(r["stall_ms"]) for r in runs]),
                   stall_max_ms=med([max(r["stall_ms"]) for r in runs]),
                   stalls=len(runs[0]["stall_ms"]))
        res[way] = row
        print(f"{way}: first sample median {row['first_sample_median_ms']:.1f} / worst {row['first_sample_worst_ms']:.1f} ms, "
              f"completion median {row['completion_median_ms']:.1f} / worst {row['completion_worst_ms']:.1f} ms, "
              f"makespan {row['makespan_ms']:.1f} ms, {row['stalls']} prefill stalls of median {row['stall_median_ms']:.1f} "
              f"/ max {row['stall_max_ms']:.1f} ms (medians of {args.repeats})")
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "stream_serve_latency.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
