"""Per-utterance tail (idx_codes_to_wav) against the packed CFM solve (idx_codes_to_wav_batch) on the config-5 utterance list.

    python -m tests.tools.tail_batch_bench OUT_DIR [--every 4] [--repeats 3]

bench.make_job("config5") gives 256 utterances (speech tokens U[128, 768], 4 speakers with 10 s references, P = 861);
F = int(2 n 1.72), 25 Euler steps, CFG 0.7, codes drawn at random (the tail does not depend on which codes).  --every k
keeps every k-th utterance of the list (k = 1: all 256).  The utterances run sorted by length, once per utterance and in
packed groups of 2, 4 and 8 consecutive utterances; a pass runs every variant once, the variants alternating, and the
first pass is a warm-up (every shape and arena size of the timed passes).  Per variant: CFM ms per utterance (the sum of
idx_s2mel_last_ms cfm_ms), tail ms per utterance (host clock around the calls, which return after the last copy), and
launches per utterance; median and spread over the timed passes.  Writes OUT_DIR/tail_batch_bench.json."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

GROUPS = [1, 2, 4, 8]


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (x.strip() for x in out.split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as ex:   # the timing itself does not depend on it
        return {"name": torch.cuda.get_device_name(0), "error": str(ex)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--every", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    assert torch.cuda.is_available(), "tail_batch_bench measures on the GPU"
    dev = torch.device("cuda", 0)
    info = gpu_info()
    e, cfg, wg, _ = bench.build_engine(0)
    job = bench.make_job("config5")[::args.every]
    lats = []
    for sp in range(4):
        inp = bench.make_inputs(100 + sp, cfg, wg)
        lats.append({k: inp[k].to(dev).contiguous() for k in ("prompt_condition", "ref_mel", "style")})
    gz = torch.Generator(device=dev).manual_seed(77)
    utts = []
    for u in sorted(job, key=lambda u: -u["n"]):
        F = int(2 * u["n"] * 1.72)
        codes = torch.randint(0, 8192, (u["n"],), generator=torch.Generator().manual_seed(9000 + u["idx"])).numpy().astype(np.int32)
        lat = lats[u["spk"]]
        utts.append(dict(codes=codes, prompt_condition=lat["prompt_condition"], ref_mel=lat["ref_mel"], style=lat["style"],
                         z=torch.randn(80, bench.P_FRAMES + F, device=dev, generator=gz), F=F))

    def run(g):
        cfm = 0.0
        l0 = e.launches
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(0, len(utts), g):
            grp = utts[i:i + g]
            if g == 1:
                u = grp[0]
                e.codes_to_wav(u["codes"], u["prompt_condition"], u["ref_mel"], u["style"], u["z"], u["F"], bench.CFM_STEPS,
                               bench.CFG_RATE, want_wav=False, want_pcm16=True)
            else:
                e.codes_to_wav_batch(grp, bench.CFM_STEPS, bench.CFG_RATE, want_wav=False, want_pcm16=True)
            cfm += e.s2mel_last_ms()["cfm_ms"]
        torch.cuda.synchronize()
        n = len(utts)
        return {"cfm_ms_per_utt": cfm / n, "tail_ms_per_utt": (time.perf_counter() - t0) * 1000 / n,
                "launches_per_utt": (e.launches - l0) / n}

    samples = {g: [] for g in GROUPS}
    for p in range(args.repeats + 1):
        for g in GROUPS:
            r = run(g)
            if p > 0:
                samples[g].append(r)
            print(f"pass {p}{' (warm-up)' if p == 0 else ''} group {g}: {r}", flush=True)
    res = {}
    for g in GROUPS:
        res[g] = {k: {"median": float(np.median([s[k] for s in samples[g]])), "min": min(s[k] for s in samples[g]),
                      "max": max(s[k] for s in samples[g])} for k in samples[g][0]}
    line = {"gpu": info, "utterances": len(utts), "speech_tokens": int(sum(u["n"] for u in job)),
            "frames_T_mean": float(np.mean([bench.P_FRAMES + u["F"] for u in utts])), "repeats": args.repeats,
            "cfm_steps": bench.CFM_STEPS, "cfg_rate": bench.CFG_RATE, "groups": res}
    for g in GROUPS:
        r = res[g]
        print(f"group {g}: CFM {r['cfm_ms_per_utt']['median']:.1f} ms/utt (range {r['cfm_ms_per_utt']['min']:.1f}-"
              f"{r['cfm_ms_per_utt']['max']:.1f}), tail {r['tail_ms_per_utt']['median']:.1f} ms/utt, "
              f"{r['launches_per_utt']['median']:.0f} launches/utt")
    print(json.dumps(info))
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "tail_batch_bench.json"), "w") as f:
        json.dump(line, f, indent=1)


if __name__ == "__main__":
    main()
