"""GPU-box measurement: ms per decode step of the strict fp32 GPT path at the IndexTTS-1.5 geometry (24 x 1280, V = 8194),
one sequence (m = 1) and three beams (m = 3, the `.infer()` default).
    python -m tests.tools.strict_beam_perf [steps] [reps]

A step's time is the difference of two decodes timed by the engine's CUDA events (prefill + decode), one `steps` longer
than the other, over the difference in steps; forbid_stop_before keeps every run at its full length.  The fp32 weight
bytes one step has to stream are computed from the shapes: with m = 3 the R-row kernels read each weight once per step
for all rows, so the aim is that m = 3 costs about one weight pass, not three.  m = 1 runs through the one-sequence
driver, which synchronises with the host after every step; the beam driver polls every 8 steps, so the ratio of the
two also compares the drivers."""
import subprocess
import sys

import numpy as np
import torch

from indextts_b200 import synth
from indextts_b200.engine import Engine
from oracle import v1
from tests.gpt_common import load_gpt

SHORT = 16


def weight_bytes(cfg):
    D, L, V = cfg["model_dim"], cfg["layers"], cfg["number_mel_codes"]
    per_layer = D * 3 * D + D * D + D * 4 * D + 4 * D * D            # c_attn, attn.c_proj, c_fc, mlp.c_proj
    return 4 * (L * per_layer + V * D)                               # + mel_head


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 128
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    assert torch.cuda.is_available(), "this measurement needs the GPU"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"card: {q}")
    cfg = synth.gpt_config(max_mel_tokens=605, max_text_tokens=402)
    w = synth.make_gpt_v1_weights(cfg, synth.V1_COND_CFG, seed=1500)
    w = {k: v for k, v in w.items() if not k.startswith(("conditioning_encoder.", "perceiver_encoder."))}
    e = Engine(0)
    load_gpt(e, cfg, w, max_batch=4, max_prompt=425, bf16=False)
    conds = torch.randn(32, cfg["model_dim"], generator=torch.Generator().manual_seed(15)) * 0.5
    prompt = v1.prepare_inputs_v1(w, conds, torch.randint(2, 100, (30,), generator=torch.Generator().manual_seed(30))).numpy()
    wb = weight_bytes(cfg)
    print(f"prompt rows {prompt.shape[0]}; fp32 weight bytes per step (from the shapes) {wb / 1e9:.3f} GB")

    def timed(m, n):
        kw = dict(num_beams=m, do_sample=True, top_k=30, top_p=0.8, temperature=1.0, seed=1, mel_pos_mode=1)
        e.gpt_generate([prompt], n, 10.0, forbid_stop_before=n, **kw)
        t = e.gpt_last_timing()
        assert t["steps"] == n, t
        return t["prefill_ms"] + t["decode_ms"], t["launches"]

    for m in (1, 3):
        timed(m, SHORT)                                               # warm-up
        per = []
        for _ in range(reps):
            t_long, l_long = timed(m, SHORT + steps)
            t_short, l_short = timed(m, SHORT)
            per.append((t_long - t_short) / steps)
        launches = (l_long - l_short) / steps
        ms = float(np.median(per))
        print(f"m = {m}: {ms:.3f} ms per step (median of {reps}; {', '.join(f'{x:.3f}' for x in per)}), "
              f"{launches:.0f} launches per step, weight stream {wb / 1e9 / (ms * 1e-3):.0f} GB/s")
    e.close()


if __name__ == "__main__":
    main()
