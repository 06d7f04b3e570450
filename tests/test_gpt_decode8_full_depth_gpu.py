"""GPU: gpt_decode8_kernel, the decode of every group of 2..8 requests, at the real geometry (24 layers x 1280, 20 heads,
V = 8194; synthetic bf16 weights).

At full depth the kernel works in a regime the 2-layer tests never reach: on a 132-SM H100 its weight ring is exactly
the 63-row mel-head phase (no spare row), and its shared-memory bias table holds 24 layers.  The tests here check it
there against references that do not run it:

  * which kernel decodes a group (the attention probe's split count: 0 for the 8-sequence kernel, the grid's split
    count for gpt_fused_kernel), so that a fall-back cannot turn every other "decode8" test into a test of the fused
    kernel;
  * its logits, teacher-forced, against the bf16 oracle for groups of 3 and 8 ragged prompts;
  * the attention of its first and last layer against the fp64 reference on the cache it read, over very ragged
    contexts (tests/test_gpt_long_context_gpu.py: _check_probe, C_ATT);
  * its logits against gpt_fused_kernel over the whole context range (ctx up to 2421);
  * a serving group (requests admitted into free rows at staggered steps, a slot reused after a longer request): every
    served code against the oracle's pick on the served codes.

On an NVIDIA H100 80GB HBM3 (132 SMs, 700 W power limit): attention errors at most 0.171 of the C_ATT bound (layer 23);
logits within 0.141 (max) / 0.0293 (rms) of the oracle, and within 0.156 / 0.0308 of gpt_fused_kernel over 1816 steps
(bounds 0.16 / 0.035); every served code the oracle's argmax or a near-tie within 0.062 (tie_tol 0.13).  The CPU
oracle took 37 s for its 384 steps there."""
import os
import time

import numpy as np
import pytest
import torch

from tests.gpt_common import GptOracle, check_teacher_forced, gpt_config, load_gpt, make_gpt_weights, processed
from tests.test_gpt_long_context_gpu import C_ATT, MAX_PROMPT, TOL, _check_probe, _codes, _prompt

pytestmark = pytest.mark.gpu
TEXT = (9, 32, 71, 3, 17, 48, 100, 140)     # text tokens of the short prompts (prompt rows = text + 5)
N_REF = (48, 48, 48, 48, 24, 24, 24, 24)    # oracle steps of each short prompt: groups of 3 (48 steps) and 8 (24), serve
PLENS = (1, 2, 5, 37, 150, 300, 605, 605)   # the long ragged prompts


@pytest.fixture(scope="module")
def rig(engine):
    cfg = gpt_config()
    w = make_gpt_weights(cfg, seed=2026, bf16=True)
    load_gpt(engine, cfg, w, max_batch=8, max_prompt=MAX_PROMPT)
    short = [_prompt(cfg, w, n, seed=80 + i) for i, n in enumerate(TEXT)]
    long_ = [_prompt(cfg, w, 600, seed=40 + i)[:m] for i, m in enumerate(PLENS)]
    oracle, refs, spent = GptOracle(cfg, w, bf16=True), {}, [0.0, 0]

    def ref(i, n):
        """(codes, logits) of the oracle's greedy decode of short prompt i, first n steps.  One run of N_REF[i] steps
        serves every n <= N_REF[i]: the stop code is forbidden throughout, so a shorter run is its prefix."""
        assert n <= N_REF[i]
        if i not in refs:
            t = time.perf_counter()
            refs[i] = oracle.generate(short[i], N_REF[i], 10.0, N_REF[i])
            spent[0] += time.perf_counter() - t
            spent[1] += N_REF[i]
        return refs[i][0][:n], refs[i][1][:n]

    def init(v8=True):
        """idx_gpt_init of the loaded weights; v8=False: under IDX_GPT_V8=0 (gpt_fused_kernel decodes the groups)."""
        old = os.environ.get("IDX_GPT_V8")
        if not v8:
            os.environ["IDX_GPT_V8"] = "0"
        try:
            engine.gpt_init(cfg["layers"], cfg["model_dim"], cfg["heads"], cfg["number_mel_codes"], cfg["start_mel_token"],
                            cfg["stop_mel_token"], cfg["max_mel_positions"], max_prompt=MAX_PROMPT, max_batch=8)
        finally:
            if old is None:
                os.environ.pop("IDX_GPT_V8", None)
            else:
                os.environ["IDX_GPT_V8"] = old

    return dict(cfg=cfg, w=w, short=short, long=long_, ref=ref, init=init, oracle=oracle, spent=spent)


def _oracle_time(rig):
    return f"CPU oracle so far: {rig['spent'][0]:.1f} s for {rig['spent'][1]} steps"


def test_groups_decode_on_the_8_sequence_kernel(engine, rig):
    """1. Groups of 2, 3 and 8 requests run on gpt_decode8_kernel (probe split count 0 at every step and layer), and on
    gpt_fused_kernel only under IDX_GPT_V8=0; every layer's attention of both against fp64 on the way."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if sms != 132:
        pytest.skip(f"gpt_decode8_kernel at 24 x 1280 is sized for the 132-SM H100 SXM; this device has {sms} SMs")
    cfg, short = rig["cfg"], rig["short"]
    L, H, n = cfg["layers"], cfg["heads"], 8
    plens = [p.shape[0] for p in short]
    for k in (2, 3, 8):
        qo, ns = engine.gpt_probe_attention(-1, n, max_seqs=8)
        out = engine.gpt_generate(short[:k], n, 10.0, forbid_stop_before=n)
        assert [len(c) for c in out] == [n] * k
        assert not ns.any(), f"group of {k}: key splits {sorted(set(ns.ravel().tolist()))}: gpt_fused_kernel decoded it"
        worst = _check_probe(engine, qo, plens[:k], n, range(L), f"decode8, group of {k}")
        print(f"group of {k}: nsplit all 0 (gpt_decode8_kernel); largest attention error over {L} layers "
              f"{worst:.3f} of the bound")
    rig["init"](v8=False)
    try:
        qo, ns = engine.gpt_probe_attention(-1, n, max_seqs=8)
        engine.gpt_generate(short[:3], n, 10.0, forbid_stop_before=n)
        want = min(8, max(1, sms // (3 * H)))
        assert (ns == want).all(), f"IDX_GPT_V8=0: key splits {sorted(set(ns.ravel().tolist()))}, gpt_fused_kernel has {want}"
        worst = _check_probe(engine, qo, plens[:3], n, range(L), "gpt_fused_kernel, group of 3")
        print(f"IDX_GPT_V8=0, group of 3: nsplit {want} (gpt_fused_kernel); largest attention error {worst:.3f} of the bound")
    finally:
        rig["init"]()


@pytest.mark.parametrize("rows,n", [(3, 48), (8, 24)])
def test_logits_vs_oracle(engine, rig, rows, n):
    """2. Teacher-forced on the oracle's greedy codes, every row's logits within the bf16 tolerance of the oracle's
    (prompts of 8 .. 145 rows); free-running, a row without a near-tie picks the oracle's codes."""
    cfg, short = rig["cfg"], rig["short"][:rows]
    ref = [rig["ref"](i, n) for i in range(rows)]
    e_codes, e_logits = engine.gpt_generate(short, n, 10.0, forbid_stop_before=n, forced_codes=[r[0] for r in ref],
                                            return_logits=True)
    free = engine.gpt_generate(short, n, 10.0, forbid_stop_before=n)
    for i, (o_codes, o_logits) in enumerate(ref):
        ties = check_teacher_forced(cfg, o_codes, o_logits, e_codes[i], e_logits[i], 10.0, n, **TOL)
        d = e_logits[i].astype(np.float64) - o_logits
        print(f"group of {rows}, row {i} (prompt {short[i].shape[0]}), {n} steps: near-ties {ties}, "
              f"max |dlogit| {np.abs(d).max():.3f}, rms {np.sqrt((d ** 2).mean()):.4f}; free run "
              f"{int((free[i] == o_codes).sum())}/{n} codes equal the oracle's")
        if ties == 0:
            np.testing.assert_array_equal(free[i], o_codes, err_msg=f"group of {rows}, row {i}")
    print(_oracle_time(rig))


def test_first_and_last_layer_attention_vs_fp64(engine, rig):
    """3. Eight very ragged prompts (1 .. 605 rows), 400 teacher-forced steps: the attention of layer 0 and of layer 23
    against the fp64 reference on each row's own cache slot.  The probe does not change what the kernel computes."""
    cfg, prompts = rig["cfg"], rig["long"]
    n = 400
    forced = [_codes(cfg, n, 50 + i) for i in range(8)]
    runs = []
    for layer in (0, cfg["layers"] - 1):
        qo, ns = engine.gpt_probe_attention(layer, n, max_seqs=8)
        out, lg = engine.gpt_generate(prompts, n, 10.0, forbid_stop_before=n, forced_codes=forced, return_logits=True)
        assert [len(c) for c in out] == [n] * 8
        worst = _check_probe(engine, qo, PLENS, n, [layer], f"decode8 full depth, layer {layer}")
        print(f"layer {layer}, prompts {list(PLENS)}, {n} steps: largest attention error {worst:.3f} of the bound "
              f"({worst * C_ATT:.2e} x sum p|v| / sum p); splits {sorted(set(ns.ravel().tolist()))}")
        runs.append(lg)
    for i in range(8):
        assert np.array_equal(runs[0][i], runs[1][i]), f"row {i}: the probe of another layer changed the logits"


def test_decode8_vs_fused_kernel_whole_context(engine, rig):
    """4. Eight ragged prompts, max_mel_positions - 2 = 1816 forced random codes (ctx up to 2421): the 8-sequence kernel's
    logits against gpt_fused_kernel's (IDX_GPT_V8=0 at init), step by step."""
    cfg, prompts = rig["cfg"], rig["long"]
    n = cfg["max_mel_positions"] - 2
    forced = [_codes(cfg, n, 50 + i) for i in range(8)]
    _, l8 = engine.gpt_generate(prompts, n, 10.0, forbid_stop_before=n, forced_codes=forced, return_logits=True)
    rig["init"](v8=False)
    try:
        _, lf = engine.gpt_generate(prompts, n, 10.0, forbid_stop_before=n, forced_codes=forced, return_logits=True)
    finally:
        rig["init"]()
    for i in range(8):
        assert l8[i].shape == lf[i].shape == (n, cfg["number_mel_codes"])
        d = l8[i].astype(np.float64) - lf[i]
        per_step_max = np.abs(d).max(axis=1)
        per_step_rms = np.sqrt((d ** 2).mean(axis=1))
        k, kr = int(np.argmax(per_step_max)), int(np.argmax(per_step_rms))
        print(f"row {i} (prompt {PLENS[i]}, ctx {PLENS[i] + 1}..{PLENS[i] + n}): decode8 vs fused over {n} steps: "
              f"max |dlogit| {per_step_max[k]:.3f} (step {k}), max per-step rms {per_step_rms[kr]:.4f} (step {kr})")
        assert per_step_max[k] <= TOL["max_abs"], (i, k, float(per_step_max[k]))
        assert per_step_rms[kr] <= TOL["max_rms"], (i, kr, float(per_step_rms[kr]))


def test_serving_group_picks_vs_oracle(engine, rig):
    """5. Greedy serving group of 3 slots: four requests admitted at staggered steps (rows at different steps of one
    launch), the last into the slot of the longest, finished request.  Every served code is the oracle's pick on the
    served codes (teacher-forced), or within tie_tol of it."""
    cfg, short = rig["cfg"], rig["short"]
    n = N_REF[0]
    served, where = {}, {}                        # request -> its codes; request -> (slot, group step at its admission)

    def admit(sv, slot, i, step):
        sv.admit(slot, short[i], i)
        where[i] = (slot, step)

    def collect(sv, reqs):
        for s, i in enumerate(reqs):
            if sv.finished[s] and i not in served:
                served[i] = sv.codes[s].copy()

    # request 2 (the longest prompt) runs in slot 0 from group step 0: its code count is the group's step count
    with engine.gpt_serve(3, n, 10.0, forbid_stop_before=n) as sv:
        admit(sv, 0, 2, 0)
        sv.next([7, 1, 1])
        admit(sv, 1, 1, sv.n_committed[0])
        sv.next([sv.n_committed[0] + 20, 5, 1])   # ends when request 1 has 5 codes
        admit(sv, 2, 3, sv.n_committed[0])
        while not sv.finished[0]:
            sv.next([n, sv.n_committed[1] + 9, sv.n_committed[2] + 13])
        collect(sv, [2, 1, 3])
        sv.release(0)                             # its prompt and codes stay in the slot's cache rows
        admit(sv, 0, 0, n)
        while not all(sv.finished):
            sv.next([n, n, n])
        collect(sv, [0, 1, 3])
    steps = [where[i][1] for i in (2, 1, 3)]
    assert steps[0] == 0 and 7 <= steps[1] < steps[2] < n, steps
    stop = cfg["stop_mel_token"]
    for i in (2, 1, 3, 0):
        got = served[i]
        assert len(got) == n, (i, len(got))
        o_codes, o_logits = rig["ref"](i, n)
        if not np.array_equal(got, o_codes):       # the oracle's logits along the served codes
            t = time.perf_counter()
            o_codes, o_logits = rig["oracle"].generate(short[i], n, 10.0, n, forced=got)
            rig["spent"][0] += time.perf_counter() - t
            rig["spent"][1] += n
        seen, ties, worst = {1, cfg["start_mel_token"]}, 0, 0.0
        for k in range(n):
            s = processed(o_logits[k], seen, 10.0, stop, k < n)
            best = int(np.argmax(s))
            gap = float(s[best]) - float(s[got[k]])
            assert got[k] == best or gap <= TOL["tie_tol"], f"request {i} step {k}: served {got[k]}, oracle {best}, gap {gap}"
            ties += int(got[k] != best)
            worst = max(worst, gap)
            seen.add(int(got[k]))
        print(f"serve request {i} (prompt {short[i].shape[0]} rows, slot {where[i][0]}, admitted at group step {where[i][1]}): "
              f"{n} codes, {n - ties} the oracle's argmax, {ties} near-ties (largest gap {worst:.3f})")
    print(_oracle_time(rig))
