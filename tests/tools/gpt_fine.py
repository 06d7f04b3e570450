"""GPU-box diagnostic: sub-phase timeline of the batch-1 decode kernel (gpt_decode1_kernel) for ALL CTAs
(middle layer, last step): %globaltimer for the cross-CTA picture, clock64 deltas for the per-CTA costs.
    python -m tests.tools.gpt_fine [steps]
Environment switches of the library that make sense here: IDX_GPT_DBG (1 skip the MMA loops, 2 skip the attention key
loop, 4 do not wait in polls), IDX_GPT_RING (ring rows)."""
import os
import sys

import numpy as np
import torch

from indextts_b200.engine import Engine
from tests.gpt_common import gpt_config, load_gpt, make_gpt_weights, prepare_gpt_inputs, r16

NAMES = {0: "layer start", 1: "QKV x polled", 2: "QKV LN done", 3: "QKV weights ready", 4: "QKV mma loop done", 5: "QKV partials synced",
         6: "QKV epilogue done", 7: "ATT q polled", 8: "ATT keys done", 9: "ATT smem published", 10: "ATT end", 11: "OPJ o polled",
         12: "OPJ weights ready", 13: "OPJ mma loop done", 14: "OPJ partials synced", 15: "OPJ epilogue done", 16: "FC x polled",
         17: "FC LN done", 18: "FC weights ready", 19: "FC mma loop done", 20: "FC partials synced", 21: "FC epilogue done",
         22: "PRJ f polled", 23: "PRJ weights ready", 24: "PRJ mma loop done", 25: "PRJ partials synced", 26: "PRJ epilogue done"}


NAMES8 = {0: "P1 start", 1: "QKV LN done", 2: "QKV weights ready", 3: "QKV mma done", 4: "QKV epilogue done", 5: "P2 start (barrier)",
          6: "ATT done", 7: "P3 start (barrier)", 8: "OPJ weights + B ready", 9: "OPJ mma done", 10: "OPJ epilogue done",
          11: "P4 start (barrier)", 12: "FC LN done", 13: "FC weights ready", 14: "FC mma done", 15: "FC epilogue done",
          16: "P5 start (barrier)", 17: "PRJ weights ready", 18: "PRJ mma done", 19: "PRJ epilogue done", 20: "next layer (barrier)"}


def main8(steps, batch):
    """8-row kernel (gpt_decode8_kernel): globaltimer stamps of every CTA, middle layer of the last step."""
    cfg = gpt_config()
    w = make_gpt_weights(cfg, seed=2025, bf16=True)
    e = Engine(0)
    load_gpt(e, cfg, w, max_batch=batch, max_prompt=64)
    g = torch.Generator().manual_seed(11)
    prompts = []
    for b in range(batch):
        style = torch.randn(192, generator=g)
        emo = r16(torch.randn(cfg["model_dim"], generator=g) * 0.5)
        text = torch.randint(2, 12000, (32,), generator=g)
        prompts.append(prepare_gpt_inputs(w, style, emo, text, lang=1, bf16=True).numpy())
    e.gpt_generate(prompts, 8, 10.0, forbid_stop_before=8)
    for rep in range(2):
        e.gpt_generate(prompts, steps, 10.0, forbid_stop_before=steps)
        t = e.gpt_last_timing()
        print(f"batch {batch}: decode {t['decode_ms'] / max(1, t['steps']) * 1000:.1f} us/step ({t['steps']} steps)")
    e.gpt_profile(True)
    e.gpt_generate(prompts, steps, 10.0, forbid_stop_before=steps)
    f = e.gpt_profile_fine().astype(np.float64)
    t0 = f[:, 0].min()
    print(f"{'slot':>4} {'name':24s} {'min':>7} {'med':>7} {'p90':>7} {'max':>7} us after the earliest P1 start | CTA 0 | argmax CTA")
    for i in range(21):
        r = (f[:, i] - t0) / 1000.0
        if i == 6:
            r = r[:batch * cfg["heads"] // 2]          # the CTAs that own a (sequence, head pair)
        print(f"{i:4d} {NAMES8[i]:24s} {r.min():7.2f} {np.median(r):7.2f} {np.percentile(r, 90):7.2f} {r.max():7.2f} | {r[0]:7.2f} | {int(np.argmax(r))}")
    os.makedirs("gpurun_out", exist_ok=True)
    np.save("gpurun_out/gpt_fine8.npy", f)
    e.close()


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 64
    if len(sys.argv) > 2 and sys.argv[2].isdigit() and int(sys.argv[2]) > 1:
        return main8(steps, int(sys.argv[2]))
    cfg = gpt_config()
    w = make_gpt_weights(cfg, seed=2025, bf16=True)
    e = Engine(0)
    load_gpt(e, cfg, w, max_batch=1, max_prompt=64)
    g = torch.Generator().manual_seed(11)
    style = torch.randn(192, generator=g)
    emo = r16(torch.randn(cfg["model_dim"], generator=g) * 0.5)
    text = torch.randint(2, 12000, (32,), generator=g)
    prompts = [prepare_gpt_inputs(w, style, emo, text, lang=1, bf16=True).numpy()]
    e.gpt_generate(prompts, 8, 10.0, forbid_stop_before=8)
    tag = " ".join(f"{k}={os.environ[k]}" for k in ("IDX_GPT_DBG", "IDX_GPT_RING") if k in os.environ) or "default"
    for rep in range(3):
        e.gpt_generate(prompts, steps, 10.0, forbid_stop_before=steps)
        t = e.gpt_last_timing()
        print(f"[{tag}] decode {t['decode_ms'] / max(1, t['steps']) * 1000:.1f} us/step ({t['steps']} steps)")
    if "-q" in sys.argv:
        e.close()
        return
    e.gpt_profile(True)
    e.gpt_generate(prompts, steps, 10.0, forbid_stop_before=steps)
    f = e.gpt_profile_fine().astype(np.float64)
    t0 = f[:, 0].min()
    print(f"{'slot':>4} {'name':22s} {'min':>7} {'med':>7} {'max':>7} us after the earliest layer start | per-CTA clock64 delta to the previous "
          f"slot: med / p90 / max cycles")
    prev = None
    for i in range(27):
        r = (f[:, i] - t0) / 1000.0
        line = f"{i:4d} {NAMES[i]:22s} {r.min():7.2f} {np.median(r):7.2f} {r.max():7.2f}"
        if prev is not None:
            d = f[:, 32 + i] - f[:, 32 + prev]
            if i in (7, 8, 9):               # attention stamps exist only on the CTAs that own a head
                m = (f[:, i] >= t0) & (f[:, i] < t0 + 1e6)
                d = d[m] if m.any() else d
                line = f"{i:4d} {NAMES[i]:22s} {r[m].min():7.2f} {np.median(r[m]):7.2f} {r[m].max():7.2f}" if m.any() else line
            line += f" | {np.median(d):8.0f} {np.percentile(d, 90):8.0f} {d.max():8.0f}"
        print(line)
        prev = i
    os.makedirs("gpurun_out", exist_ok=True)
    np.save("gpurun_out/gpt_fine.npy", f)
    e.close()


if __name__ == "__main__":
    main()
