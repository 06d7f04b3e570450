"""GPU-box diagnostic: sweep the weight-ring pacing knobs of the batch-1 decode kernel (gpt_decode1_kernel) in ONE process
(the model is built once), settings alternated round by round so that drift of the shared machine hits all of them alike.
    python -m tests.tools.gpt_ring_sweep [steps] [rounds] [setting ...]
A setting is an IDX_GPT_DBG value (decimal or 0x...; "0" = the defaults).  Bits the kernel reads: 8-15 rows per issue
call (cap), 16 (bit 4) no issues from inside the hand-over polls, 32-39 rows in flight (target), 40-47 poll rounds
between two issue attempts.  Prints the median / min / max decode us per step of every setting and checks that every
setting produced the same codes as the first (the knobs move only the time at which weights are copied)."""
import os
import sys

import numpy as np
import torch

from indextts_b200.engine import Engine
from tests.gpt_common import gpt_config, load_gpt, make_gpt_weights, prepare_gpt_inputs, r16


def knob(target=0, every=0, cap=0, no_spin=False):
    return (target << 32) | (every << 40) | (cap << 8) | (16 if no_spin else 0)


def describe(v):
    if v == 0:
        return "defaults"
    parts = []
    if v & 16:
        parts.append("no spin issues")
    if (v >> 8) & 0xff:
        parts.append(f"cap {(v >> 8) & 0xff}")
    if (v >> 32) & 0xff:
        parts.append(f"in flight {(v >> 32) & 0xff}")
    if (v >> 40) & 0xff:
        parts.append(f"every {(v >> 40) & 0xff} rounds")
    return ", ".join(parts)


# the previous schedule (issues only after a poll, cap rows per call), then the neighbourhood of the defaults (54 rows, 8 rounds)
DEFAULT_SETTINGS = [knob(no_spin=True, target=255)] + [knob(target=t, every=n) for t in (36, 54, 72) for n in (4, 8, 16)]


def main():
    args = [a for a in sys.argv[1:]]
    steps = int(args[0]) if args else 256
    rounds = int(args[1]) if len(args) > 1 else 3
    settings = [int(a, 0) for a in args[2:]] or DEFAULT_SETTINGS
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
    us = {s: [] for s in settings}
    ref = None
    for _ in range(rounds):
        for s in settings:
            os.environ["IDX_GPT_DBG"] = str(s)
            codes = e.gpt_generate(prompts, steps, 10.0, forbid_stop_before=steps)[0]
            t = e.gpt_last_timing()
            us[s].append(t["decode_ms"] / max(1, t["steps"]) * 1000)
            if ref is None:
                ref = np.asarray(codes).copy()
            assert np.array_equal(np.asarray(codes), ref), f"setting {s:#x} changed the codes"
    os.environ.pop("IDX_GPT_DBG", None)
    print(f"{'IDX_GPT_DBG':>14} {'med':>7} {'min':>7} {'max':>7}  us/step over {rounds} rounds of {steps} steps")
    for s in settings:
        v = np.array(us[s])
        print(f"{s:#14x} {np.median(v):7.1f} {v.min():7.1f} {v.max():7.1f}  {describe(s)}")
    print("codes identical across settings:", True)
    e.close()


if __name__ == "__main__":
    main()
