"""Host-side model of the paced weight stream of the batch-1 decode kernel (csrc/gpt_decode1.cuh): on top of the ring
protocol of tests/test_ring_schedule_cpu.py, the producer thread also issues from INSIDE the hand-over polls (`on_spin`)
and after them (`refill`), in instalments of at most `cap` rows and only while fewer than `target` rows are in flight —
issued, phase not yet seen complete.  It finds completed phases with a non-blocking parity test of their `full`
mbarriers, in phase order (`note_landed`).

The model replays the kernel's call sequence with issue attempts at arbitrary points of every poll and copies that land
at arbitrary times (any issued phase may complete; the test in phase order stops at the first incomplete one), for the
H100 grid (132 CTAs) and the B200 grid (148), both model sizes, the ring `idx_gpt_init` sizes on a 227 KB SM and the
smallest ring it accepts.  It checks:

  * every phase is completely issued before its wait (the issuing thread waits too: an incomplete phase would trap);
  * the ring never holds more than R rows; at most NBAR phases (a partly issued one included) are outstanding;
  * every row of the stream is issued exactly once, in order;
  * a paced call never takes the rows in flight above the target, and the in-flight count matches the phases;
  * the parity test is only applied to a phase whose barrier slot has not been re-armed for a later phase;
  * an early exit leaves only phases that can be waited for.

No GPU, no library call: this is the protocol, restated."""
import random

import pytest

from tests.test_ring_schedule_cpu import NBAR, Ring, check_stream, cta_phases, run_decode1

SMEM_OPTIN = 227 * 1024      # cudaDevAttrMaxSharedMemoryPerBlockOptin of H100 and B200
RED1_FLOATS = 2 * 4 * 8 * 16 + 48 + 64 + 8 * 66
PHASE1_BYTES = 14 * 4


def cdiv(a, b):
    return (a + b - 1) // b


def smem_bytes_v2(D, L, V, G, R):
    """gpt_decode.cu: smem_bytes_v2 with idx_gpt_init's bias_cap / ocap."""
    FF = 4 * D
    ocap = cdiv(D, G) + 1
    bias_cap = L * (cdiv(3 * D, G) + 1 + 2 * ocap + cdiv(FF, G) + 1) + cdiv(V, G) + 1
    return (R * D * 2 + FF * 2 + 4 * RED1_FLOATS + 8 * NBAR + 5 * PHASE1_BYTES + 32 + 4 * bias_cap + 4 * ocap
            + 4 * cdiv(V, 32) + 16 + 4 * 4 * D + 64)


def ring_rows(D, L, V, G):
    R = 0
    while smem_bytes_v2(D, L, V, G, R + 1) <= SMEM_OPTIN - 1024:
        R += 1
    return R


def min_ring_rows(D, V, G):
    """The host's refusal bound: the largest phase any CTA can have."""
    FF = 4 * D
    mq, mo, mf, mh = cdiv(3 * D, G) + 1, cdiv(D, G) + 1, cdiv(FF, G) + 1, cdiv(V, G) + 1
    return max(mq, mf, 4 * mo, mh)


class PacedRing(Ring):
    """Ring plus the producer's in-flight bookkeeping: landed / lpidx / inflight, note_landed, issue_paced."""

    def __init__(self, rows, R, nsteps, cap, target, rng):
        super().__init__(rows, R, nsteps, cap)
        self.target, self.rng = target, rng
        self.landed = self.lpidx = self.inflight = 0
        self.arrived = set()       # fully issued phases whose bytes have all landed (their barrier phase completed)

    def issue_fitting(self, budget=0):
        n0 = len(self.issued)
        super().issue_fitting(budget)
        self.inflight += sum(m for (_, _, _, m) in self.issued[n0:])
        self.check_counts()

    def check_counts(self):
        assert self.fill <= self.R
        assert self.tix + (1 if self.part else 0) - self.cons_tile <= NBAR
        assert self.cons_tile <= self.landed <= self.tix
        want = sum(self.rows[n % self.pps] for n in range(self.landed, self.tix)) + self.part
        assert self.inflight == want

    def land_some(self):
        """Copies complete at arbitrary times and in any order."""
        pending = [n for n in range(self.cons_tile, self.tix) if n not in self.arrived]
        for n in pending:
            if self.rng.random() < 0.4:
                self.arrived.add(n)

    def note_landed(self):
        while self.landed < self.tix:
            n = self.landed
            last_armed = self.tix if self.part else self.tix - 1       # highest phase with bytes or an arrive on a slot
            assert n >= self.cons_tile and n + NBAR > last_armed, "parity test of a slot re-armed for a later phase"
            if n not in self.arrived:
                break
            self.inflight -= self.rows[self.lpidx]
            self.landed += 1
            self.lpidx = (self.lpidx + 1) % self.pps
        self.check_counts()

    def issue_paced(self):
        self.land_some()
        self.note_landed()
        before = self.inflight
        budget = min(self.cap, self.target - before)
        if budget > 0:
            n0 = len(self.issued)
            self.issue_fitting(budget)
            got = sum(m for (_, _, _, m) in self.issued[n0:])
            assert got <= budget and self.inflight <= self.target

    def spin(self):
        """A hand-over poll: the producer tries to issue an arbitrary number of times, then once more after it."""
        for _ in range(self.rng.randrange(0, 6)):
            self.issue_paced()
        self.issue_paced()                                   # refill()

    def wait(self):
        super().wait()
        self.arrived.add(self.cons_tile)                     # mbar_wait returns only once the phase has completed

    def advance(self, rows, immediate_all=False):
        if self.landed == self.cons_tile:
            self.inflight -= rows
            self.landed += 1
            self.lpidx = (self.lpidx + 1) % self.pps
        issued = super().advance(rows, immediate_all)
        self.check_counts()
        return issued


def run_paced_decode1(rows, R, nsteps, cap, target, L, seed, stop_after=None):
    """gpt_decode1_kernel's call sequence: issue attempts inside and after every hand-over poll."""
    r = PacedRing(list(rows), R, nsteps, cap, target, random.Random(seed))
    r.issue_fitting(R)                                       # initial fill
    consumed = 0
    for _ in range(nsteps):
        i = 0
        for l in range(L):
            if l > 0:
                r.spin()                                     # P1: x poll + refill
            else:
                r.issue_paced()                              # P1 of layer 0: refill only (the input row is built locally)
            r.wait(); r.advance(rows[i]); i += 1             # QKV
            r.spin()                                         # P3: o poll (or the key-split partials) + refill
            r.wait(); r.advance(rows[i]); i += 1             # O-proj
            r.spin()                                         # P4: x poll + refill
            r.wait(); r.advance(rows[i]); i += 1             # FC
            r.spin()                                         # P5: gelu(fc) poll + refill
            r.wait(); r.advance(rows[i]); i += 1             # PROJ
            consumed += 4
            if stop_after is not None and consumed >= stop_after:
                return r
        r.spin()                                             # head: x poll + refill
        r.wait(); r.advance(rows[i])                         # head
    return r


def drain(r):
    """The kernel's exit: close a partly issued phase with a plain arrive, then wait for every outstanding phase."""
    if r.part > 0:
        r.tix += 1
        r.part = 0
    assert r.tix - r.cons_tile <= NBAR                      # every outstanding phase still owns its slot: waits are unambiguous
    for n in range(r.cons_tile, r.tix):
        # armed with an arrive and all its bytes issued: the phase completes once the copies land
        assert sum(m for (s, p, _, m) in r.issued if s * r.pps + p == n) <= r.rows[n % r.pps]


GEOMS = [(D, V, G, L) for (D, V, L) in ((1280, 8194, 24), (256, 8194, 3)) for G in (132, 148)]


def cta_geometries(D, V, G, L):
    seen = []
    for cta in range(G):
        rows = tuple(cta_phases(D, V, G, cta, L))
        if rows not in seen:
            seen.append(rows)
    return seen


def test_ring_rows_as_the_host_sizes_them():
    # the B200 figure of the 1280-wide model the older model hard-codes, and the H100 grid
    assert ring_rows(1280, 24, 8194, 148) == 72
    assert ring_rows(1280, 24, 8194, 132) == 71


@pytest.mark.parametrize("D,V,G,L", GEOMS)
@pytest.mark.parametrize("cap,target", [(18, 36), (18, 18), (4, 6), (18, 255), (255, 255), (6, 1)])
def test_paced_stream_keeps_the_ring_protocol(D, V, G, L, cap, target):
    R = ring_rows(D, L, V, G)
    for k, rows in enumerate(cta_geometries(D, V, G, L)):
        assert max(rows) <= R
        for nsteps in (1, 2):
            r = run_paced_decode1(rows, R, nsteps, cap, target, L, seed=1000 * k + nsteps)
            check_stream(r, list(rows), nsteps)


@pytest.mark.parametrize("D,V,G,L", GEOMS)
def test_smallest_legal_ring(D, V, G, L):
    R = min_ring_rows(D, V, G)
    Ls = min(L, 3)
    for k, rows in enumerate(cta_geometries(D, V, G, Ls)):
        assert max(rows) <= R
        for cap, target in ((1, 1), (4, 36), (5, 7), (255, 255)):
            r = run_paced_decode1(rows, R, 2, cap, target, Ls, seed=k)
            check_stream(r, list(rows), 2)


@pytest.mark.parametrize("G", [132, 148])
def test_early_exit_leaves_only_waitable_phases(G):
    # the kernel stops consuming when the sequence has finished: what was issued must be drainable
    for stop_after in (1, 2, 5, 11):
        for seed in range(8):
            rows = cta_phases(1280, 8194, G, seed * 7 % G, 24)
            r = run_paced_decode1(rows, ring_rows(1280, 24, 8194, G), 3, 6, 36, 24, seed, stop_after=stop_after)
            drain(r)


@pytest.mark.parametrize("G", [132, 148])
def test_without_spin_issues_and_target_the_old_schedule_is_kept(G):
    # target >= R and no issue attempts inside the polls: exactly the instalment sequence of the previous protocol
    class NoSpin(PacedRing):
        def spin(self):
            self.issue_paced()

    rows = cta_phases(1280, 8194, G, 0, 24)
    R = ring_rows(1280, 24, 8194, G)
    old = run_decode1(list(rows), R, 2, 18, 24)
    r = NoSpin(list(rows), R, 2, 18, 255, random.Random(0))
    r.issue_fitting(R)
    for _ in range(2):
        i = 0
        for _l in range(24):
            r.spin(); r.wait(); r.advance(rows[i]); i += 1
            r.spin(); r.spin(); r.wait(); r.advance(rows[i]); i += 1     # the older model refills twice here
            r.spin(); r.wait(); r.advance(rows[i]); i += 1
            r.spin(); r.wait(); r.advance(rows[i]); i += 1
        r.spin(); r.wait(); r.advance(rows[i])
    assert r.issued == old.issued
