"""GPU-box diagnostic: full-size GPT decode timing + per-phase profile of the fused kernel.
    python -m tests.tools.gpt_perf [steps] [batch]"""
import sys

import numpy as np
import torch

from indextts_b200.engine import Engine
from tests.gpt_common import gpt_config, load_gpt, make_gpt_weights, prepare_gpt_inputs, r16


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 64
    batch = int(sys.argv[2]) if len(sys.argv) > 2 else 1
    cfg = gpt_config()
    w = make_gpt_weights(cfg, seed=2025, bf16=True)
    e = Engine(0)
    load_gpt(e, cfg, w, max_batch=max(1, batch), max_prompt=64)
    g = torch.Generator().manual_seed(11)
    prompts = []
    for b in range(batch):
        style = torch.randn(192, generator=g)
        emo = r16(torch.randn(cfg["model_dim"], generator=g) * 0.5)
        text = torch.randint(2, 12000, (32,), generator=g)
        prompts.append(prepare_gpt_inputs(w, style, emo, text, lang=1, bf16=True).numpy())
    e.gpt_generate(prompts, 8, 10.0, forbid_stop_before=8)  # warm-up
    e.gpt_profile(True)
    for rep in range(3):
        e.gpt_generate(prompts, steps, 10.0, forbid_stop_before=steps)
        t = e.gpt_last_timing()
        print(f"batch {batch}: prefill {t['prefill_ms']:.2f} ms, decode {t['decode_ms']:.2f} ms for {t['steps']} steps "
              f"= {t['decode_ms'] / t['steps'] * 1000:.1f} us/step, launches {t['launches']}")
    st_all = e.gpt_profile(True, read=True)
    import os
    if batch == 1 and os.environ.get("IDX_GPT_V2") != "0":      # gpt_decode1_kernel keeps its own per-CTA timeline: tests/tools/gpt_fine.py
        e.close()
        return
    fine = st_all[256:]
    print('fine QKV (ns deltas):', np.diff(fine[:12][fine[:12] > 0]).tolist())
    print('fine FC  (ns deltas):', np.diff(fine[16:28][fine[16:28] > 0]).tolist())
    fs = fine[32:35]
    if (fs > 0).all():
        print('sampling phase (us): seen copy+sync -> pick', (fs[1] - fs[0]) / 1000, '-> bookkeeping', (fs[2] - fs[1]) / 1000)
    st = st_all[:256]
    st = st[st > 0]
    d = np.diff(st)
    L = cfg["layers"]
    # stamps: step start, [before,after] prologue barrier, per layer 5x[before,after], head [b,a], sample [b,a]
    print(f"stamps {len(st)}; last step total {(st[-1] - st[0]) / 1000:.1f} us")
    names = ["QKV", "ATTN", "OPROJ", "FC", "PROJ"]
    comp = {n: [] for n in names}
    wait = {n: [] for n in names}
    i = 3  # index of the stamp after the prologue barrier
    for l in range(L):
        for n in names:
            comp[n].append(st[i] - st[i - 1])
            wait[n].append(st[i + 1] - st[i])
            i += 2
    print(f"prologue: compute {(st[1] - st[0]) / 1000:.2f} us, barrier {(st[2] - st[1]) / 1000:.2f} us")
    for n in names:
        print(f"{n:6s}: compute mean {np.mean(comp[n]) / 1000:.2f} us (max {np.max(comp[n]) / 1000:.2f}), "
              f"barrier mean {np.mean(wait[n]) / 1000:.2f} us (max {np.max(wait[n]) / 1000:.2f})")
    rest = st[i - 1:]
    print("head/sample stamps (us):", [round(float(x) / 1000, 2) for x in np.diff(rest)])
    e.close()


if __name__ == "__main__":
    main()
