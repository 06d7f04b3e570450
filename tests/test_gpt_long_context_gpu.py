"""GPU: the GPT decode kernels at long contexts.

The attention of every decode step is checked on its own, against a float64 reference computed on the kernel's exact
operands: the attention probe (idx_gpt_probe_attention) records q as the kernel read it and the normalised attention
output before its bf16 rounding, and idx_gpt_debug_kv returns the K / V cache the kernel read.  The bound per element is
C_ATT * Σp|v|/Σp; on an NVIDIA H100 80GB HBM3 (400 W power limit) the largest error of both decode kernels over all of
these tests was 0.017 * 2e-5 = 3.4e-7 of that scale, 17 % of C_ATT = 2e-6.  A logit comparison alone hardly sees a
single missing or doubled key (on the 2-layer geometry that moves the logits by rms ~0.02, inside the bf16 noise of the
path); here one key dropped or counted twice at each split boundary moved rows by up to 2.6 % of Σp|v|/Σp, four orders
of magnitude above the bound.

Contexts run from the prompt (605 rows) to 605 + 1816 = 2421 keys, the model's limit (max_mel_positions = 1818): the
batch-1 kernel goes through one CTA per head (<= 640 keys) and every key-split count its grid allows (at most
min(7, SMs / heads) splits), across the 64-step launch boundaries; the 8-sequence kernel through very ragged contexts
inside one group.  Logits are also checked end to end against the bf16 oracle at the same lengths, and at full depth
against the round-1 fused kernel."""
import os

import numpy as np
import pytest
import torch

from tests import kernel_refs as kr
from tests.gpt_common import GptOracle, check_teacher_forced, gpt_config, load_gpt, make_gpt_weights, prepare_gpt_inputs, r16

pytestmark = pytest.mark.gpu
TOL = dict(max_abs=0.16, max_rms=0.035, tie_tol=0.13)       # tests/test_gpt_gpu.py
C_ATT = 2e-6            # |kernel - fp64| <= C_ATT * Σp|v|/Σp per element: fp32 online softmax with __expf (see above)
MAX_PROMPT = 640


def _prompt(cfg, w, n_text, seed):
    g = torch.Generator().manual_seed(seed)
    style = torch.randn(192, generator=g)
    emo = r16(torch.randn(cfg["model_dim"], generator=g) * 0.5)
    text = torch.randint(2, cfg["number_text_tokens"], (n_text,), generator=g)
    return prepare_gpt_inputs(w, style, emo, text, lang=1, bf16=True).numpy()


def _codes(cfg, n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, cfg["start_mel_token"], (n,), generator=g).numpy().astype(np.int32)


def _nsplit_expected(ctx, heads, split_at=640, split_len=320):
    """Key splits per head of gpt_decode1_kernel at `ctx` keys on this device (DESIGN.md section 4a)."""
    max_split = min(7, torch.cuda.get_device_properties(0).multi_processor_count // heads)
    if ctx <= split_at or max_split < 2:
        return 1
    return min(max_split, -(-ctx // split_len))


def _check_probe(engine, qo, plens, n, layers, what):
    """Every probed (step, layer, sequence) row against ref_decode_attention on the sequence's own cache slot.
    Returns the largest error as a fraction of its bound."""
    worst = 0.0
    for li, l in enumerate(layers):
        for b, plen in enumerate(plens):
            K, V = engine.gpt_kv(l, b, 0, plen + n)
            q, got = qo[:n, li, b, 0], qo[:n, li, b, 1]
            assert np.all(np.abs(q).max(-1) > 0) and np.all(np.abs(got).max(-1) > 0), f"{what}: probe rows missing (layer {l}, seq {b})"
            assert np.isfinite(got).all()
            ctx = plen + 1 + np.arange(n)
            ref, vmag = kr.ref_decode_attention(q, K, V, ctx)
            r = np.abs(got - ref) / (C_ATT * vmag)
            k, c = np.unravel_index(int(np.argmax(r)), r.shape)
            assert r[k, c] <= 1.0, (f"{what}: layer {l} seq {b} step {k} (ctx {ctx[k]}) head {c // 64}: |err| {abs(got[k, c] - ref[k, c]):.3e} "
                                    f"> {C_ATT} * {vmag[k, c]:.3e}")
            worst = max(worst, float(r[k, c]))
    return worst


def test_decode1_attention_long_context_default_splits(engine):
    """4a. Batch-1 kernel, v2.5 geometry (D = 1280, H = 20, V = 8194) at 2 layers, 605-row prompt, 1816 teacher-forced
    steps: ctx 606 .. 2421 with the default knobs."""
    cfg = gpt_config(layers=2)
    w = make_gpt_weights(cfg, seed=31, bf16=True)
    load_gpt(engine, cfg, w, max_prompt=MAX_PROMPT)
    prompt = _prompt(cfg, w, 600, seed=3)
    assert prompt.shape[0] == 605
    n = cfg["max_mel_positions"] - 2
    qo, ns = engine.gpt_probe_attention(-1, n)
    (codes,) = engine.gpt_generate([prompt], n, 10.0, forbid_stop_before=n, forced_codes=[_codes(cfg, n, 4)])
    assert len(codes) == n
    ctx = 605 + 1 + np.arange(n)
    want = np.array([_nsplit_expected(int(c), cfg["heads"]) for c in ctx])
    assert np.array_equal(ns[:, 0], want) and np.array_equal(ns[:, 1], want), sorted(set(ns[:, 0].tolist()))
    worst = _check_probe(engine, qo, [605], n, [0, 1], "decode1")
    print(f"decode1, default splits {sorted(set(want.tolist()))} over ctx {ctx[0]}..{ctx[-1]}: "
          f"largest attention error {worst:.3f} of the bound")


def test_decode1_attention_forced_splits(engine):
    """4b. Batch-1 kernel at D = 256 (gpt_decode1_kernel<8>, H = 4) with split_at = split_len = 32 keys (IDX_GPT_DBG bits
    16-23 / 24-30): ctx 14 .. 333 covers one CTA per head and every split count up to 7."""
    cfg = gpt_config(layers=2, model_dim=256, heads=4, number_mel_codes=322, start_mel_token=320, stop_mel_token=321,
                     max_mel_tokens=330, max_text_tokens=30, number_text_tokens=100, n_langs=3)
    w = make_gpt_weights(cfg, seed=32, bf16=True)
    load_gpt(engine, cfg, w, max_prompt=64)
    prompt = _prompt(cfg, w, 8, seed=5)
    plen, n = prompt.shape[0], 320
    qo, ns = engine.gpt_probe_attention(-1, n)
    os.environ["IDX_GPT_DBG"] = str((1 << 16) | (1 << 24))
    try:
        (codes,) = engine.gpt_generate([prompt], n, 10.0, forbid_stop_before=n, forced_codes=[_codes(cfg, n, 6)])
    finally:
        del os.environ["IDX_GPT_DBG"]
    assert len(codes) == n
    ctx = plen + 1 + np.arange(n)
    want = np.array([_nsplit_expected(int(c), cfg["heads"], 32, 32) for c in ctx])
    assert np.array_equal(ns[:, 0], want) and np.array_equal(ns[:, 1], want), sorted(set(ns[:, 0].tolist()))
    assert {1, 2, 7} <= set(want.tolist())
    worst = _check_probe(engine, qo, [plen], n, [0, 1], "decode1 forced splits")
    print(f"decode1, forced splits {sorted(set(want.tolist()))} over ctx {ctx[0]}..{ctx[-1]}: "
          f"largest attention error {worst:.3f} of the bound")


def test_decode8_attention_ragged_contexts(engine):
    """4c. 8-sequence kernel, one group of very ragged prompts (1 .. 605 rows), 400 teacher-forced steps."""
    cfg = gpt_config(layers=2)
    w = make_gpt_weights(cfg, seed=33, bf16=True)
    load_gpt(engine, cfg, w, max_batch=8, max_prompt=MAX_PROMPT)
    plens = [1, 2, 5, 37, 150, 300, 605, 605]
    prompts = [_prompt(cfg, w, 600, seed=40 + i)[:m] for i, m in enumerate(plens)]
    n = 400
    qo, ns = engine.gpt_probe_attention(-1, n, max_seqs=8)
    out = engine.gpt_generate(prompts, n, 10.0, forbid_stop_before=n, forced_codes=[_codes(cfg, n, 50 + i) for i in range(8)])
    assert [len(c) for c in out] == [n] * 8
    assert not ns.any()
    worst = _check_probe(engine, qo, plens, n, [0, 1], "decode8")
    print(f"decode8, prompts {plens}, {n} steps: largest attention error {worst:.3f} of the bound")


def test_long_context_logits_vs_oracle(engine):
    """4d. End to end against the bf16 oracle at long contexts (2 layers, v2.5 widths, 1816 teacher-forced steps):
    the batch-1 kernel on a 605-row prompt, and the 8-sequence kernel on a group of three ragged prompts."""
    cfg = gpt_config(layers=2)
    w = make_gpt_weights(cfg, seed=34, bf16=True)
    n = cfg["max_mel_positions"] - 2
    oracle = GptOracle(cfg, w, bf16=True)
    prompts = [_prompt(cfg, w, 600, seed=60)]
    prompts += [_prompt(cfg, w, 600, seed=61)[:300], _prompt(cfg, w, 600, seed=62)[:37]]
    ref = [oracle.generate(p, n, 10.0, n) for p in prompts]
    load_gpt(engine, cfg, w, max_prompt=MAX_PROMPT)
    (e_codes,), (e_logits,) = engine.gpt_generate([prompts[0]], n, 10.0, forbid_stop_before=n, forced_codes=[ref[0][0]],
                                                  return_logits=True)
    ties = check_teacher_forced(cfg, ref[0][0], ref[0][1], e_codes, e_logits, 10.0, n, **TOL)
    d = e_logits - ref[0][1]
    print(f"decode1 vs oracle, {n} steps: near-ties {ties}, max |dlogit| {np.abs(d).max():.3f}, rms {np.sqrt((d.astype(np.float64) ** 2).mean()):.4f}")
    load_gpt(engine, cfg, w, max_batch=8, max_prompt=MAX_PROMPT)
    e_codes, e_logits = engine.gpt_generate(prompts, n, 10.0, forbid_stop_before=n, forced_codes=[r[0] for r in ref],
                                            return_logits=True)
    for i, (o_codes, o_logits) in enumerate(ref):
        ties = check_teacher_forced(cfg, o_codes, o_logits, e_codes[i], e_logits[i], 10.0, n, **TOL)
        d = e_logits[i] - o_logits
        print(f"decode8 seq {i} (prompt {prompts[i].shape[0]}) vs oracle: near-ties {ties}, max |dlogit| {np.abs(d).max():.3f}, "
              f"rms {np.sqrt((d.astype(np.float64) ** 2).mean()):.4f}")


def test_full_depth_decode1_above_1920_keys(engine):
    """4e. 24 layers, 605-row prompt, 1816 teacher-forced steps (ctx up to 2421, where an unbounded split count would
    need more CTAs than the grid has): the batch-1 kernel's logits against gpt_fused_kernel<1, .> (IDX_GPT_V2=0 at init,
    splits bounded by the grid), and its attention of the first and the last layer against the fp64 reference."""
    cfg = gpt_config()
    w = make_gpt_weights(cfg, seed=2025, bf16=True)
    load_gpt(engine, cfg, w, max_prompt=MAX_PROMPT)
    prompt = _prompt(cfg, w, 600, seed=11)
    n = cfg["max_mel_positions"] - 2
    forced = _codes(cfg, n, 12)
    runs = []
    for layer in (0, cfg["layers"] - 1):
        qo, ns = engine.gpt_probe_attention(layer, n)
        (_,), (lg,) = engine.gpt_generate([prompt], n, 10.0, forbid_stop_before=n, forced_codes=[forced], return_logits=True)
        t = engine.gpt_last_timing()
        worst = _check_probe(engine, qo, [605], n, [layer], f"full depth layer {layer}")
        print(f"full depth, layer {layer}: largest attention error {worst:.3f} of the bound; splits {sorted(set(ns[:, 0].tolist()))}; "
              f"decode {t['decode_ms'] / t['steps'] * 1000:.1f} us/step")
        runs.append(lg)
    assert np.array_equal(runs[0], runs[1])          # the probe does not change what the kernel computes
    os.environ["IDX_GPT_V2"] = "0"
    try:
        load_gpt(engine, cfg, w, max_prompt=MAX_PROMPT)
    finally:
        del os.environ["IDX_GPT_V2"]
    (_,), (lf,) = engine.gpt_generate([prompt], n, 10.0, forbid_stop_before=n, forced_codes=[forced], return_logits=True)
    d = runs[0].astype(np.float64) - lf
    per_step_max = np.abs(d).max(axis=1)
    per_step_rms = np.sqrt((d ** 2).mean(axis=1))
    k = int(np.argmax(per_step_max))
    print(f"full depth decode1 vs fused kernel over {n} steps: max |dlogit| {per_step_max.max():.3f} (step {k}), "
          f"max per-step rms {per_step_rms.max():.4f}")
    assert per_step_max.max() <= TOL["max_abs"] and per_step_rms.max() <= TOL["max_rms"]
