"""fp64 reference of the GPT decode pick, replayed from the exact fp32 logits a decode path consumed.

Written from the HF processor semantics, independently of `oracle.gpt.sample_token` (which restates the
kernels' fp32 arithmetic).  One step, one sequence:

  RepetitionPenalty  s < 0 ? s * p : s / p on the tokens seen so far, as one fp64 op rounded to fp32.  fp64 carries
                     more than 2 * 24 + 2 bits, so this is the correctly rounded fp32 op bit for bit.
  forbid stop        s[stop] = -inf while k < forbid_stop_before.
  Temperature        (sampling only) s * fp32(1 / T), rounded to fp32.  This is the engine's documented form; HF's
                     TemperatureLogitsWarper divides by T instead, which can differ from it in the last bit.
  greedy             argmax, lowest index among ties.  No tolerance.
  TopK               every token whose score ties the k-th score is kept (TopKLogitsWarper removes only scores
                     strictly below it); more than 128 kept candidates means the engine must refuse the call.
  softmax, TopP      in fp64 over the candidates in descending order (lowest index first among ties); the tail is
                     dropped while its cumulative probability <= 1 - top_p, with that threshold computed in fp32 from
                     the fp32 top_p as the device does; at least one candidate is kept.
  multinomial        u = (philox(seed, k, seq)[0] >> 8) / 2^24; the pick is the first kept candidate whose cumulative
                     weight exceeds u * kt (kt = total kept weight).

The device evaluates softmax, the top-p tail and the cumulative sums in fp32 (expf and at most 128 additions).  When
the top-p tail lies within MARGIN of its threshold, or u * kt within MARGIN * kt of a cumulative boundary, the device's
decision is not determined by the exact values, and the reference returns every pick the fp32 evaluation could make
(`Pick.margin` is True when that is more than one).
"""
from dataclasses import dataclass

import numpy as np

from oracle.gpt import philox4x32_10

CMAX = 128          # candidate slots of the device samplers
MARGIN = 3e-5       # covers expf and <= 128 fp32 additions relative to the fp64 values


@dataclass(frozen=True)
class Pick:
    ok: frozenset       # acceptable picks (one element unless `margin`)
    margin: bool        # a top-p or multinomial decision within MARGIN of its boundary leaves more than one pick
    refuse: bool        # more than CMAX candidates tie at the top-k boundary: the engine must refuse the call


def processed_scores(logits, seen, k, rep_penalty, stop_tok, forbid_stop_before, do_sample=False, temperature=1.0):
    """fp32 scores after RepetitionPenalty, the stop ban and (sampling) the engine's temperature form."""
    s = np.asarray(logits, dtype=np.float32).astype(np.float64)
    p = float(np.float32(rep_penalty))
    idx = np.array(sorted(seen), dtype=np.int64)
    sv = s[idx]
    s[idx] = np.where(sv < 0, sv * p, sv / p)
    s = s.astype(np.float32)
    if k < forbid_stop_before:
        s[stop_tok] = -np.inf
    if do_sample:
        inv_t = np.float32(np.float32(1.0) / np.float32(temperature))
        s = (s.astype(np.float64) * float(inv_t)).astype(np.float32)
    return s


def top_k_candidates(s, top_k):
    """Indices kept by TopK in the device's order: descending score, lowest index first among ties."""
    s = np.asarray(s, dtype=np.float32)
    fin = np.flatnonzero(np.isfinite(s))
    order = fin[np.lexsort((fin, -s[fin]))]
    if len(order) <= top_k:
        return order
    kth = s[order[top_k - 1]]
    return order[s[order] >= kth]


def top_p_keep(probs, top_p, shift=0.0):
    """Number of leading candidates TopP keeps (probs descending, fp64); `shift` moves the threshold."""
    thr = float(np.float32(1.0) - np.float32(top_p)) + shift
    keep = len(probs)
    if top_p < 1.0:
        tail = 0.0
        for i in range(len(probs) - 1, 0, -1):
            tail += probs[i]
            if tail <= thr:
                keep = i
            else:
                break
    return keep


def pick(logits, seen, k, seq, *, rep_penalty, stop_tok, forbid_stop_before=0, do_sample=False, top_k=0,
         top_p=1.0, temperature=1.0, seed=0):
    s = processed_scores(logits, seen, k, rep_penalty, stop_tok, forbid_stop_before, do_sample, temperature)
    if not do_sample:
        return Pick(frozenset([int(np.argmax(s))]), False, False)
    cand = top_k_candidates(s, top_k)
    if len(cand) > CMAX:
        return Pick(frozenset(), False, True)
    sc = s[cand].astype(np.float64)
    w = np.exp(sc - sc[0])
    probs = w / w.sum()
    keep_min, keep_max = top_p_keep(probs, top_p, MARGIN), top_p_keep(probs, top_p, -MARGIN)
    u = (philox4x32_10(seed, k, seq)[0] >> 8) / 16777216.0
    ok = set()
    for keep in range(keep_min, keep_max + 1):
        cum = np.cumsum(w[:keep])
        t, m = u * cum[-1], MARGIN * cum[-1]
        lo = int(np.searchsorted(cum, t - m, side="right"))     # first i with cum[i] > t - m
        hi = int(np.searchsorted(cum, t + m, side="right"))
        # past the last boundary (fp32 rounding of u * kt) the device keeps its last candidate
        ok.update(int(cand[min(i, keep - 1)]) for i in range(lo, hi + 1))
    return Pick(frozenset(ok), len(ok) > 1, False)


@dataclass
class Replay:
    steps: int = 0
    margins: int = 0
    ties: int = 0           # steps whose deciding score was shared by more than one token (see replay_sequence)


def replay_sequence(codes, logits, *, seq, start_tok, stop_tok, max_new, forced=None, tie_tokens=None, **sp):
    """Replay every step of one sequence from the logits it consumed.  Asserts each pick, the termination step and
    (through the Philox counter) the global sequence index `seq`.  `tie_tokens`: count the steps on which at least two
    of these tokens share the greedy maximum / the top-k boundary score."""
    codes = np.asarray(codes)
    seen = {1, start_tok}
    rep = Replay()
    n = len(codes)
    assert len(logits) == n, (len(logits), n)
    for k in range(n):
        pk = pick(logits[k], seen, k, seq, stop_tok=stop_tok, **sp)
        assert not pk.refuse, f"seq {seq} step {k}: more than {CMAX} tied candidates were not refused"
        assert int(codes[k]) in pk.ok, f"seq {seq} step {k}: engine picked {int(codes[k])}, reference {sorted(pk.ok)}"
        rep.margins += pk.margin
        if tie_tokens is not None:
            s = processed_scores(logits[k], seen, k, sp["rep_penalty"], stop_tok, sp.get("forbid_stop_before", 0),
                                 sp.get("do_sample", False), sp.get("temperature", 1.0))
            if sp.get("do_sample", False):
                cand = top_k_candidates(s, sp["top_k"])
                bound = s[cand[-1]]
            else:
                bound = s.max()
            rep.ties += int(np.sum(s[list(tie_tokens)] == bound) >= 2)
        feed = int(codes[k]) if forced is None else int(forced[k])
        seen.add(feed)
        # termination: the device stops at the stop token when free running, else after max_new steps
        last = (forced is None and int(codes[k]) == stop_tok) or k + 1 >= max_new
        assert last == (k == n - 1), f"seq {seq}: engine returned {n} codes, the replay ends at step {k}"
    rep.steps = n
    return rep
