"""GPU-box check that a change leaves the one-sequence strict fp32 GPT path bitwise unchanged.
    python -m tests.tools.strict_record record OUT.npz       (run on each build)
    python -m tests.tools.strict_record compare A.npz B.npz  (needs no GPU)

`record` decodes seeded prompts on the strict path (num_beams = 1): the small test geometry (two requests of different
prompt lengths, 40 steps) and the v1.5 geometry (24 x 1280, V = 8194, a 64-row v1 prompt, 48 steps), each greedy and
sampled (top_k 30, top_p 0.8, temperature 0.8) under both mel_pos_mode values, and stores every request's codes and
raw fp32 logits.  `compare` reports every array whose shape or bits differ and exits non-zero if any does."""
import sys

import numpy as np
import torch

SAMPLED = dict(do_sample=True, top_k=30, top_p=0.8, temperature=0.8, seed=123)


def record(path):
    from indextts_b200 import synth
    from indextts_b200.engine import Engine
    from oracle import v1
    from oracle.validate_gpt_vs_hf import small_case
    from tests.gpt_common import load_gpt, make_gpt_weights, prepare_gpt_inputs

    out = {}
    e = Engine(0)

    def run(name, prompts, n):
        for mode in (0, 1):
            for sampled in (False, True):
                kw = dict(forbid_stop_before=n // 2, return_logits=True, mel_pos_mode=mode, **(SAMPLED if sampled else {}))
                codes, logits = e.gpt_generate(prompts, n, 10.0, **kw)
                for i, (c, lg) in enumerate(zip(codes, logits)):
                    key = f"{name}_m{mode}_{'s' if sampled else 'g'}_{i}"
                    out[key + "_codes"], out[key + "_logits"] = c, lg

    cfg, style, emo, text = small_case()
    w = make_gpt_weights(cfg, seed=1234, bf16=False)
    load_gpt(e, cfg, w, max_batch=2, bf16=False)
    p0 = prepare_gpt_inputs(w, style, emo, text, lang=1, bf16=False).numpy()
    run("small", [p0, p0[:-3]], 40)

    cfg = synth.gpt_config(max_mel_tokens=605, max_text_tokens=402)
    w = synth.make_gpt_v1_weights(cfg, synth.V1_COND_CFG, seed=1500)
    w = {k: v for k, v in w.items() if not k.startswith(("conditioning_encoder.", "perceiver_encoder."))}
    load_gpt(e, cfg, w, max_prompt=425, bf16=False)
    conds = torch.randn(32, 1280, generator=torch.Generator().manual_seed(15)) * 0.5
    text = torch.randint(2, 100, (30,), generator=torch.Generator().manual_seed(30))
    run("v15", [v1.prepare_inputs_v1(w, conds, text).numpy()], 48)
    e.close()
    np.savez(path, **out)
    print(f"recorded {len(out)} arrays to {path}")


def compare(pa, pb):
    a, b = np.load(pa), np.load(pb)
    bits = lambda x: x.view(np.uint32) if x.dtype == np.float32 else x       # noqa: E731
    keys = sorted(set(a.files) | set(b.files))
    bad = [k for k in keys if k not in a.files or k not in b.files or a[k].shape != b[k].shape
           or not np.array_equal(bits(a[k]), bits(b[k]))]
    print(f"{len(keys)} arrays, {len(bad)} differ" + (": " + ", ".join(bad) if bad else " (bitwise identical)"))
    return 1 if bad else 0


if __name__ == "__main__":
    if sys.argv[1:2] == ["record"] and len(sys.argv) == 3:
        record(sys.argv[2])
    elif sys.argv[1:2] == ["compare"] and len(sys.argv) == 4:
        sys.exit(compare(sys.argv[2], sys.argv[3]))
    else:
        sys.exit(__doc__)
