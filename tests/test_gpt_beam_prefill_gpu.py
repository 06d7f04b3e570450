"""GPU: the attention of gpt_fused_kernel, the kernel of every prompt's prefill and of every beam-search decode step,
checked on its own against a float64 reference on the kernel's exact operands.

* Prefill: the prompts of one call run as tiles of 8 positions through one launch (mode 0); causality comes only from
  the key bound ctx = position + 1.  idx_gpt_probe_prefill records q and the normalised attention output of every
  prompt row, and every row is checked with its own ctx.
* Beam search: beam row r of an utterance reads its prompt keys from the utterance's first cache slot and generated
  position plen + i from the slot of its ancestor at step i, through the lineage map that beam_step_kernel rewrites
  after every step.  The reference takes each key from where the beams' traced ancestry says it must be
  (kernel_refs.beam_key_slots, which never reads that map), so a beam that attends to a sibling's key fails here even
  though siblings share most of their history and the logits hardly move.

Bound per element: C_ATT * Σp|v|/Σp with C_ATT = 2e-6, as for the decode kernels (tests/test_gpt_long_context_gpu.py):
the fused kernel runs the same fp32 online softmax with __expf, merged over warps and key splits."""
import numpy as np
import pytest
import torch

from tests import kernel_refs as kr
from tests.gpt_common import gpt_config, load_gpt, make_gpt_weights, prepare_gpt_inputs, r16
from tests.test_gpt_gpu import _beam_params, _check_beam_run

pytestmark = pytest.mark.gpu
C_ATT = 2e-6
MAX_PROMPT = 640


def _prompt(cfg, w, n_text, seed):
    g = torch.Generator().manual_seed(seed)
    style = torch.randn(192, generator=g)
    emo = r16(torch.randn(cfg["model_dim"], generator=g) * 0.5)
    text = torch.randint(2, cfg["number_text_tokens"], (n_text,), generator=g)
    return prepare_gpt_inputs(w, style, emo, text, lang=1, bf16=True).numpy()


def _small_cfg():
    """D = 256, H = 4: the fused kernel splits the keys of every (row, head) of a full tile over several CTAs."""
    return gpt_config(layers=2, model_dim=256, heads=4, number_mel_codes=322, start_mel_token=320, stop_mel_token=321,
                      max_mel_tokens=330, max_text_tokens=30, number_text_tokens=100, n_langs=3)


def _fused_nsplit(rows, heads):
    """Key splits per (row, head) of gpt_fused_kernel with `rows` rows on this device: min(8, max(1, SMs / (rows * heads)))."""
    return min(8, max(1, torch.cuda.get_device_properties(0).multi_processor_count // (rows * heads)))


def _bound_ratio(got, ref, vmag, what):
    assert np.isfinite(got).all(), what
    r = np.abs(got - ref) / (C_ATT * vmag)
    i, c = np.unravel_index(int(np.argmax(r)), r.shape)
    assert r[i, c] <= 1.0, (f"{what}: row {i} head {c // 64}: |err| {abs(got[i, c] - ref[i, c]):.3e} > {C_ATT} * {vmag[i, c]:.3e}")
    return float(r[i, c])


def _check_prefill(engine, qo, plens, layers, slot_of, what):
    """Every prompt row of every request at every probed layer, with ctx = position + 1 on the request's cache slot."""
    worst = 0.0
    for u, plen in enumerate(plens):
        assert not qo[u, plen:].any(), f"{what}: rows past the prompt of request {u} were written"
        for li, l in enumerate(layers):
            K, V = engine.gpt_kv(l, slot_of(u), 0, plen)
            q, got = qo[u, :plen, li, 0], qo[u, :plen, li, 1]
            assert np.all(np.abs(q).max(-1) > 0) and np.all(np.abs(got).max(-1) > 0), f"{what}: rows missing (req {u}, layer {l})"
            ref, vmag = kr.ref_decode_attention(q, K, V, np.arange(plen) + 1)
            worst = max(worst, _bound_ratio(got, ref, vmag, f"{what}: request {u} (prompt {plen}) layer {l}"))
    return worst


def _check_beams(engine, qo, steps, li, layer, plens, m, what):
    """Every beam row of every utterance at every step the call ran (pad steps after an utterance is done included),
    against the keys its traced ancestry names.  The keys of an utterance are gathered once into a union cache: its
    prompt (first slot), then positions plen .. plen + steps - 1 of each of its m slots; each row attends to the subset
    kernel_refs.beam_key_slots gives."""
    D = qo.shape[-1]
    worst = 0.0
    for u, plen in enumerate(plens):
        par, tok, _, _ = engine.gpt_beam_trace(u, num_beams=m)
        assert len(par) == steps, (len(par), steps)
        row0 = u * m
        slots = kr.beam_key_slots(par, plen, m, row0)                               # [steps][m][plen + steps]
        j = np.arange(plen + steps)
        col = np.where(j < plen, j, plen + (slots - row0) * steps + (j - plen))
        keys = np.zeros((steps * m, plen + m * steps), bool)
        on = slots >= 0
        rows = np.broadcast_to(np.arange(steps * m).reshape(steps, m, 1), slots.shape)
        keys[rows[on], col[on]] = True
        Kp, Vp = engine.gpt_kv(layer, row0, 0, plen)
        gen = [engine.gpt_kv(layer, row0 + r, plen, steps) for r in range(m)]
        K = np.concatenate([Kp] + [g[0] for g in gen])
        V = np.concatenate([Vp] + [g[1] for g in gen])
        q = qo[:steps, li, row0:row0 + m, 0].reshape(steps * m, D)
        got = qo[:steps, li, row0:row0 + m, 1].reshape(steps * m, D)
        assert np.all(np.abs(q).max(-1) > 0) and np.all(np.abs(got).max(-1) > 0), f"{what}: rows missing (utterance {u})"
        ref, vmag = kr.ref_decode_attention(q, K, V, keys=keys)
        worst = max(worst, _bound_ratio(got, ref, vmag, f"{what}: utterance {u} layer {layer} (row = step * {m} + beam)"))
    return worst


def test_prefill_v25_widths(engine):
    """D = 1280, H = 20, 2 layers: prompts of 1, 7, 8, 9, 17, 64 and 605 rows in one tile list (num_beams = 1), then a
    2-utterance beam call with ragged prompts of 605 and 37 rows (prompt KV in slots 0 and 3)."""
    cfg = gpt_config(layers=2)
    w = make_gpt_weights(cfg, seed=71, bf16=True)
    load_gpt(engine, cfg, w, max_batch=8, max_prompt=MAX_PROMPT)
    full = _prompt(cfg, w, 600, seed=72)
    assert full.shape[0] == 605
    plens = [1, 7, 8, 9, 17, 64, 605]
    prompts = [_prompt(cfg, w, 600, seed=80 + i)[:n] for i, n in enumerate(plens[:-1])] + [full]
    qo = engine.gpt_probe_prefill(-1, 605, max_seqs=len(plens))
    engine.gpt_generate(prompts, 2, 10.0, forbid_stop_before=2)
    worst = _check_prefill(engine, qo, plens, [0, 1], lambda u: u, "prefill, num_beams = 1")
    print(f"prefill v2.5 widths, prompts {plens}: largest attention error {worst:.3f} of the bound "
          f"({_fused_nsplit(8, cfg['heads'])} key split(s) per (row, head))")
    plens2 = [605, 37]
    qo = engine.gpt_probe_prefill(-1, 605, max_seqs=2)
    engine.gpt_generate([full, _prompt(cfg, w, 600, seed=81)[:37]], 2, 10.0, num_beams=3,
                        do_sample=True, top_k=30, top_p=0.8, temperature=0.8, seed=3, forbid_stop_before=2)
    worst2 = _check_prefill(engine, qo, plens2, [0, 1], lambda u: 3 * u, "prefill, 2 x 3 beams")
    print(f"prefill v2.5 widths, beam call prompts {plens2}: largest attention error {worst2:.3f} of the bound")


def test_prefill_and_beams_small_geometry(engine):
    """D = 256, H = 4: a full tile has 8 * 4 (row, head) items, so the keys are split over several CTAs
    (min(8, SMs / 32), 4 on a 132-SM H100), with empty splits for rows whose ctx is below the split count.  Prefill
    of prompts 1 .. 35 rows, then beam decode with 2 rows (8 splits) and 2 x 4 rows, checked against the ancestry."""
    cfg = _small_cfg()
    w = make_gpt_weights(cfg, seed=73, bf16=True)
    load_gpt(engine, cfg, w, max_batch=8, max_prompt=64)
    nsplit = _fused_nsplit(8, cfg["heads"])
    assert nsplit > 1, "the device has too few SMs for this test's split count"
    plens = [1, 7, 8, 9, 17, 35]
    prompts = [_prompt(cfg, w, 30, seed=90 + i)[:n] for i, n in enumerate(plens)]
    qo = engine.gpt_probe_prefill(-1, 35, max_seqs=len(plens))
    engine.gpt_generate(prompts, 2, 10.0, forbid_stop_before=2)
    worst = _check_prefill(engine, qo, plens, [0, 1], lambda u: u, "small prefill")
    print(f"prefill D = 256, {nsplit} key splits, prompts {plens}: largest attention error {worst:.3f} of the bound")
    n = 300
    for m, ps in ((2, [prompts[5]]), (4, [prompts[5], prompts[2]])):
        rows = m * len(ps)
        qo, ns = engine.gpt_probe_attention(-1, n, max_seqs=rows)
        pq = engine.gpt_probe_prefill(-1, 35, max_seqs=len(ps))
        engine.gpt_generate(ps, n, 10.0, num_beams=m, do_sample=True, top_k=30, top_p=0.8, temperature=0.8, seed=5,
                            forbid_stop_before=n)
        steps = engine.gpt_last_timing()["steps"]
        assert steps == n
        assert (ns[:steps] == _fused_nsplit(rows, cfg["heads"])).all(), sorted(set(ns[:steps].ravel().tolist()))
        worst_p = _check_prefill(engine, pq, [len(p) for p in ps], [0, 1], lambda u: u * m, f"small {len(ps)} x {m} prefill")
        worst_b = max(_check_beams(engine, qo, steps, li, li, [len(p) for p in ps], m, f"small {len(ps)} x {m} beams")
                      for li in (0, 1))
        print(f"beams D = 256, {len(ps)} x {m} rows, {_fused_nsplit(rows, cfg['heads'])} splits, {steps} steps: "
              f"largest attention error {worst_b:.3f} (prefill {worst_p:.3f}) of the bound")


BEAM_CASES = [(2, 1, True), (2, 1, False), (3, 1, True), (3, 1, False), (4, 1, True), (4, 1, False), (3, 2, False), (4, 2, True)]


@pytest.mark.parametrize("m,nutt,do_sample", BEAM_CASES, ids=[f"{u}x{m}-{'sample' if s else 'beam'}" for m, u, s in BEAM_CASES])
def test_beam_decode_v25_widths(engine, m, nutt, do_sample):
    """D = 1280, H = 20, 2 layers, 605-row prompt (with a ragged 37-row second utterance), 1190 steps with the stop token
    forbidden: contexts up to 1795 keys.  Every row at every step against its ancestry; the split count
    min(8, SMs / (rows * 20)) is 3, 2 and 1 for 2, 3 and 4 rows on a 132-SM H100."""
    cfg = gpt_config(layers=2)
    w = make_gpt_weights(cfg, seed=74, bf16=True)
    load_gpt(engine, cfg, w, max_batch=8, max_prompt=MAX_PROMPT)
    prompts = [_prompt(cfg, w, 600, seed=75), _prompt(cfg, w, 600, seed=76)[:37]][:nutt]
    plens = [p.shape[0] for p in prompts]
    n = 1190
    rows = m * nutt
    qo, ns = engine.gpt_probe_attention(-1, n, max_seqs=rows)
    kw = dict(do_sample=True, top_k=30, top_p=0.8, temperature=0.8) if do_sample else {}
    engine.gpt_generate(prompts, n, 10.0, num_beams=m, seed=11 + m, forbid_stop_before=n, **kw)
    steps = engine.gpt_last_timing()["steps"]
    assert steps == n
    want = _fused_nsplit(rows, cfg["heads"])
    assert (ns[:steps] == want).all(), sorted(set(ns[:steps].ravel().tolist()))
    worst = max(_check_beams(engine, qo, steps, li, li, plens, m, f"{nutt} x {m} beams") for li in (0, 1))
    print(f"beams v2.5 widths, {nutt} x {m} rows ({'sample' if do_sample else 'beam search'}), {want} split(s), prompts {plens}, "
          f"ctx up to {max(plens) + steps}: largest attention error {worst:.3f} of the bound")


def test_beam_pad_steps_after_done(engine):
    """A stop token that wins as soon as it is allowed ends both utterances early; the host looks at the done flags
    every 8 steps, so the kernel runs pad steps with the identity reorder.  Those rows are checked too."""
    cfg = gpt_config(layers=2)
    w = make_gpt_weights(cfg, seed=77, bf16=True)
    w["mel_head.bias"] = w["mel_head.bias"].clone()
    w["mel_head.bias"][cfg["stop_mel_token"]] += 100.0
    load_gpt(engine, cfg, w, max_batch=8, max_prompt=MAX_PROMPT)
    prompts = [_prompt(cfg, w, 600, seed=78), _prompt(cfg, w, 600, seed=79)[:37]]
    n, m = 400, 3
    qo, ns = engine.gpt_probe_attention(-1, n, max_seqs=2 * m)
    engine.gpt_generate(prompts, n, 10.0, num_beams=m, do_sample=True, top_k=30, top_p=0.8, temperature=0.8, seed=9,
                        forbid_stop_before=250)
    steps = engine.gpt_last_timing()["steps"]
    assert 250 <= steps < n and steps % 8 == 0, steps
    pads = []
    for u in range(2):
        par, tok, _, _ = engine.gpt_beam_trace(u, num_beams=m)
        pad = np.flatnonzero((tok == cfg["stop_mel_token"]).all(axis=1))       # a live beam never carries the stop token
        assert np.array_equal(pad, np.arange(steps - len(pad), steps)) and (par[pad] == np.arange(m)).all()
        pads.append(len(pad))
    assert max(pads) > 0, "no pad steps ran"
    assert (ns[:steps] == _fused_nsplit(2 * m, cfg["heads"])).all()
    worst = max(_check_beams(engine, qo, steps, li, li, [p.shape[0] for p in prompts], m, "pad steps") for li in (0, 1))
    print(f"beams with early stop: {steps} steps, pad steps per utterance {pads}: largest attention error {worst:.3f} of the bound")


def test_full_depth_beam_sample_defaults(engine):
    """24 layers, the `.infer()` defaults (num_beams = 3, do_sample, top_k = 30, top_p = 0.8, temperature = 0.8,
    repetition penalty 10), 605-row prompt, 300 steps: layers 0 and 23 of the prefill and of every beam step against
    fp64, and the whole run replayed through the oracle's beam logic (_check_beam_run)."""
    cfg = gpt_config()
    w = make_gpt_weights(cfg, seed=2025, bf16=True)
    load_gpt(engine, cfg, w, max_batch=3, max_prompt=MAX_PROMPT)
    prompt = _prompt(cfg, w, 600, seed=12)
    n, m = 300, 3
    p = _beam_params(cfg, seed=13)
    kw = dict(do_sample=True, num_beams=m, top_k=30, top_p=0.8, temperature=0.8, seed=13, length_penalty=0.0)
    runs = []
    for layer in (0, cfg["layers"] - 1):
        qo, ns = engine.gpt_probe_attention(layer, n, max_seqs=m)
        pq = engine.gpt_probe_prefill(layer, 605, max_seqs=1)
        (codes,), (lg,) = engine.gpt_generate([prompt], n, 10.0, return_logits=True, **kw)
        steps = engine.gpt_last_timing()["steps"]
        _check_beam_run(engine, cfg, prompt, n, p, 0, codes, lg)
        assert (ns[:steps] == _fused_nsplit(m, cfg["heads"])).all()
        worst_p = _check_prefill(engine, pq, [605], [layer], lambda u: 0, f"full depth prefill layer {layer}")
        worst_b = _check_beams(engine, qo, steps, 0, layer, [605], m, f"full depth beams layer {layer}")
        print(f"full depth beam-sample, layer {layer}: {steps} steps, {len(codes)} codes; largest attention error "
              f"{worst_b:.3f} (prefill {worst_p:.3f}) of the bound")
        runs.append((codes, lg))
    assert np.array_equal(runs[0][0], runs[1][0]) and np.array_equal(runs[0][1], runs[1][1])   # the probes change nothing
