"""The fp64 pick reference (tests/pick_refs.py) against transformers' own logits processors, and against the oracle's
fp32 restatement of the device sampler (`oracle.gpt.sample_token`)."""
import numpy as np
import pytest
import torch

from oracle.gpt import sample_token
from tests import pick_refs as pr

V = 300
STOP = V - 1


def _cases(n, seed=0):
    """Random fp32 logits, some with a block of exactly tied scores at or near the top."""
    rng = np.random.default_rng(seed)
    for i in range(n):
        lg = (rng.standard_normal(V) * rng.choice([0.5, 2.0, 6.0])).astype(np.float32)
        if i % 3 == 1:           # a tie group at the top-k boundary region
            grp = rng.choice(V, size=int(rng.integers(2, 60)), replace=False)
            lg[grp] = np.float32(np.sort(lg)[-int(rng.integers(1, 40))])
        if i % 3 == 2:           # a tie group above everything else
            grp = rng.choice(V, size=int(rng.integers(2, 130)), replace=False)
            lg[grp] = lg.max() + np.float32(1.0)
        seen = set(rng.choice(V, size=int(rng.integers(1, 40)), replace=False).tolist()) | {1}
        yield rng, lg, seen


def test_processed_scores_equal_hf_repetition_penalty():
    tr = pytest.importorskip("transformers")
    for rng, lg, seen in _cases(60):
        for pen in (10.0, 1.0, 0.5, 1.3):
            ids = torch.tensor([sorted(seen)], dtype=torch.long)
            hf = tr.RepetitionPenaltyLogitsProcessor(pen)(ids, torch.from_numpy(lg.copy())[None])[0].numpy()
            got = pr.processed_scores(lg, seen, 0, pen, STOP, 0)
            assert np.array_equal(got, hf)
            banned = pr.processed_scores(lg, seen, 2, pen, STOP, 3)
            assert banned[STOP] == -np.inf and np.array_equal(np.delete(banned, STOP), np.delete(hf, STOP))


def test_temperature_form_within_one_ulp_of_hf():
    """The engine multiplies by fp32(1/T); HF's TemperatureLogitsWarper divides: equal up to one fp32 ulp."""
    tr = pytest.importorskip("transformers")
    for rng, lg, seen in _cases(30):
        for t in (0.8, 3.0, 0.5, 1.0):
            hf = tr.TemperatureLogitsWarper(t)(None, torch.from_numpy(lg.copy())[None])[0].numpy()
            got = pr.processed_scores(lg, seen, 0, 1.0, STOP, 0, do_sample=True, temperature=t)
            assert np.all(np.abs(got - hf) <= np.spacing(np.abs(hf)))


def test_kept_sets_equal_hf_top_k_top_p():
    tr = pytest.importorskip("transformers")
    checked = tied_boundaries = 0
    for rng, lg, seen in _cases(150, seed=1):
        s = pr.processed_scores(lg, seen, 0, 10.0, STOP, 0, do_sample=True, temperature=0.8)
        for top_k in (1, 5, 30, 128):
            st = torch.from_numpy(s.copy())[None]
            hk = tr.TopKLogitsWarper(top_k)(None, st.clone())
            cand = pr.top_k_candidates(s, top_k)
            assert set(cand.tolist()) == set(np.flatnonzero(np.isfinite(hk[0].numpy())).tolist())
            tied_boundaries += int(len(cand) > top_k)
            if len(cand) > pr.CMAX:
                continue
            for top_p in (0.3, 0.8, 0.9123, 1.0):
                hp = tr.TopPLogitsWarper(top_p)(None, hk.clone())[0].numpy()
                hf_kept = set(np.flatnonzero(np.isfinite(hp)).tolist())
                w = np.exp(s[cand].astype(np.float64) - s[cand[0]])
                probs = w / w.sum()
                keep = pr.top_p_keep(probs, top_p)
                if keep != pr.top_p_keep(probs, top_p, pr.MARGIN) or keep != pr.top_p_keep(probs, top_p, -pr.MARGIN):
                    continue         # within the fp32 evaluation margin of the top-p boundary
                ours = set(cand[:keep].tolist())
                assert len(ours) == len(hf_kept), (top_k, top_p, len(ours), len(hf_kept))
                # HF's sort leaves the order of tied scores unspecified: only tokens tying the last kept score may differ
                diff = ours ^ hf_kept
                assert all(s[i] == s[cand[keep - 1]] for i in diff)
                checked += 1
    assert checked > 1000 and tied_boundaries > 50


def test_refusal_boundary_is_129_tied_candidates():
    s = np.zeros(V, dtype=np.float32)
    for n_tied, refuse in ((128, False), (129, True)):
        s[:] = -5.0
        s[3:3 + n_tied] = 2.0
        pk = pr.pick(s, {1}, 0, 0, rep_penalty=1.0, stop_tok=STOP, do_sample=True, top_k=30, top_p=1.0, seed=1)
        assert pk.refuse == refuse
        if refuse:
            with pytest.raises(ValueError, match="tie"):
                sample_token(s, 30, 1.0, 1, 0, 0)
        else:
            tok, kept = sample_token(s, 30, 1.0, 1, 0, 0)
            assert len(kept) == 128 and pk.ok == {tok}
    s[:] = -5.0
    s[3:3 + 200] = 2.0          # 200 ties but not at the boundary of top_k = 30: the top-30 scores are distinct
    s[210:240] = np.arange(30, dtype=np.float32) + 10.0
    assert not pr.pick(s, {1}, 0, 0, rep_penalty=1.0, stop_tok=STOP, do_sample=True, top_k=30, seed=1).refuse


def test_pick_agrees_with_oracle_sample_token():
    """A few thousand draws: the fp64 reference and the oracle's fp32 restatement pick the same token outside margins.
    Exactly tied candidates put the top-p tail exactly on its threshold whenever n_tied * (1 - top_p) is an integer;
    the margin rate is bounded on the untied cases only."""
    draws = margins = 0
    plain_draws = plain_margins = 0
    params = [(30, 0.8, 0.8), (1, 1.0, 1.0), (128, 1.0, 3.0), (5, 0.3, 0.5), (60, 0.95, 1.2)]
    for ci, (rng, lg, seen) in enumerate(_cases(320, seed=2)):
        for top_k, top_p, t in params:
            for seq in (0, 3):
                k = int(rng.integers(0, 500))
                pk = pr.pick(lg, seen, k, seq, rep_penalty=10.0, stop_tok=STOP, do_sample=True, top_k=top_k,
                             top_p=top_p, temperature=t, seed=ci + 1)
                sc = pr.processed_scores(lg, seen, k, 10.0, STOP, 0, do_sample=True, temperature=t)
                if pk.refuse:
                    with pytest.raises(ValueError):
                        sample_token(sc, top_k, top_p, ci + 1, k, seq)
                    continue
                tok, _ = sample_token(sc, top_k, top_p, ci + 1, k, seq)
                assert tok in pk.ok, (ci, top_k, top_p, t, tok, sorted(pk.ok))
                if pk.margin:
                    margins += 1
                else:
                    assert pk.ok == {tok}
                draws += 1
                if ci % 3 == 0:
                    plain_draws += 1
                    plain_margins += pk.margin
    print(f"{draws} draws, {margins} within a margin ({plain_margins} of {plain_draws} without ties)")
    assert draws > 3000 and plain_margins <= 0.005 * plain_draws


def test_greedy_pick_is_lowest_index_argmax():
    s = np.full(V, -1.0, dtype=np.float32)
    s[[17, 5, 250]] = 4.0
    assert pr.pick(s, {1}, 0, 0, rep_penalty=10.0, stop_tok=STOP).ok == {5}
    assert pr.pick(s, {1, 5}, 0, 0, rep_penalty=10.0, stop_tok=STOP).ok == {17}
    s[STOP] = 9.0
    assert pr.pick(s, {1}, 0, 0, rep_penalty=10.0, stop_tok=STOP, forbid_stop_before=1).ok == {5}
    assert pr.pick(s, {1}, 1, 0, rep_penalty=10.0, stop_tok=STOP, forbid_stop_before=1).ok == {STOP}
