"""Host-side model of the shared-memory weight ring of the GPT decode kernels (csrc/gpt_decode1.cuh, csrc/gpt_decode8.cuh):
phases of consecutive stream rows, issued in instalments by one thread (`issue_fitting`), consumed in order after an mbarrier
wait.  The model replays the kernels' call sequence (the points where `issue_fitting` / `advance` are called) for every CTA
geometry of the two instantiated model sizes and checks the properties the device code relies on:

  * a phase is completely issued before its consumer waits for it (the waiting threads include the issuing thread: a phase
    that is still incomplete at its wait can never complete — the kernel would trap in mbar_wait);
  * the ring never holds more than R rows, at most NBAR phases are outstanding, and a partly issued phase keeps its slot;
  * every row of the stream is issued exactly once, in order, for every step of the launch.

No GPU, no library call: this is the protocol, restated."""
import itertools

import pytest

TROWS, NBAR, MAXIT = 16, 8, 4


def col_begin(n, i, g):
    return (n * i) // g


def cta_phases(D, V, G, cta, L):
    """Rows of the phases of one decode step of CTA `cta` (Sched1::rows): per layer QKV | O | FC | PROJ, then the head."""
    FF, nseg = 4 * D, 4
    nq = col_begin(3 * D, cta + 1, G) - col_begin(3 * D, cta, G)
    no = col_begin(D, cta + 1, G) - col_begin(D, cta, G)
    nf = col_begin(FF, cta + 1, G) - col_begin(FF, cta, G)
    nh = col_begin(V, cta + 1, G) - col_begin(V, cta, G)
    return [nq, no, nf, no * nseg] * L + [nh]


class Ring:
    """issue_fitting / advance of the kernels, line by line."""

    def __init__(self, rows, R, nsteps, cap, minpart=4):
        self.rows, self.R, self.nsteps, self.cap, self.minpart = rows, R, nsteps, cap, minpart
        self.pps = len(rows)
        self.tix = self.cons_tile = 0
        self.fill = self.wpos = self.pstep = self.pidx = self.part = 0
        self.issued = []          # (step, phase, first row, rows) in issue order
        self.uoff = 0
        self.max_fill = 0

    def issue_fitting(self, budget=0):
        if budget <= 0:
            budget = self.cap
        while self.pstep < self.nsteps and self.tix - self.cons_tile < NBAR and budget > 0:
            n = self.rows[self.pidx] - self.part
            avail = min(self.R - self.fill, budget)
            last = avail >= n
            m = n if last else avail
            if not last and m < self.minpart:
                break
            assert m > 0
            self.issued.append((self.pstep, self.pidx, self.part, m))
            self.wpos = (self.wpos + m) % self.R
            self.fill += m
            self.max_fill = max(self.max_fill, self.fill)
            assert self.fill <= self.R
            self.uoff += m
            budget -= m
            if not last:
                self.part += m
                break
            self.part = 0
            self.tix += 1
            self.pidx += 1
            if self.pidx == self.pps:
                self.pidx, self.uoff = 0, 0
                self.pstep += 1

    def wait(self):
        # mbar_wait(full[cons_tile % NBAR]): must already be complete, nobody can issue while the CTA waits
        assert self.tix > self.cons_tile, f"phase {self.cons_tile} waited for before it was completely issued"

    def advance(self, rows, immediate_all=False):
        self.cons_tile += 1
        self.fill -= rows
        assert self.fill >= 0
        if immediate_all or self.tix == self.cons_tile:
            need = self.rows[self.pidx] - self.part if self.pstep < self.nsteps else 0
            self.issue_fitting(max(self.cap, need))
            return True
        return False


def run_decode8(rows, R, nsteps, cap, L):
    r = Ring(rows, R, nsteps, cap)
    r.issue_fitting(R)                                   # initial fill
    for _ in range(nsteps):
        i = 0
        for _l in range(L):
            r.issue_fitting()                            # P1: after the LayerNorm
            r.wait(); r.advance(rows[i]) or r.issue_fitting(); i += 1      # QKV (advance always issues: cap or the remainder)
            r.issue_fitting()                            # grid barrier
            r.issue_fitting()                            # P2: end of the attention phase
            r.issue_fitting()                            # grid barrier
            r.wait(); r.advance(rows[i]) or r.issue_fitting(); i += 1      # O-proj
            r.issue_fitting()                            # grid barrier
            r.issue_fitting()                            # P4: after the LayerNorm
            r.wait(); r.advance(rows[i]) or r.issue_fitting(); i += 1      # FC
            r.issue_fitting()                            # grid barrier
            r.wait(); r.advance(rows[i]) or r.issue_fitting(); i += 1      # PROJ
            r.issue_fitting()                            # grid barrier
        r.wait(); r.advance(rows[i]) or r.issue_fitting()                  # head
        r.issue_fitting()                                # barrier before sampling
        r.issue_fitting()                                # barrier after sampling
    return r


def run_decode1(rows, R, nsteps, cap, L):
    """gpt_decode1_kernel: `advance` issues only when nothing of the next phase is complete; `refill()` after every poll."""
    r = Ring(rows, R, nsteps, cap)
    r.issue_fitting(R)
    for _ in range(nsteps):
        i = 0
        for _l in range(L):
            r.issue_fitting()                            # refill after the x poll
            r.wait(); r.advance(rows[i]); i += 1         # QKV
            r.issue_fitting(); r.issue_fitting()         # O-proj: refill after the o poll (either branch has one or two)
            r.wait(); r.advance(rows[i]); i += 1
            r.issue_fitting()                            # FC: refill after the x poll
            r.wait(); r.advance(rows[i]); i += 1
            r.issue_fitting()                            # PROJ: refill after the f poll
            r.wait(); r.advance(rows[i]); i += 1
        r.issue_fitting()                                # head poll
        r.wait(); r.advance(rows[i])
    return r


def check_stream(r, rows, nsteps):
    # every row exactly once, in order
    exp = []
    for s in range(nsteps):
        for p, n in enumerate(rows):
            exp.append((s, p, n))
    got = {}
    order = []
    for (s, p, first, m) in r.issued:
        k = (s, p)
        assert got.get(k, 0) == first, "instalments of a phase must be consecutive"
        got[k] = first + m
        if not order or order[-1] != k:
            order.append(k)
    assert order == [(s, p) for (s, p, _) in exp]
    for (s, p, n) in exp:
        assert got[(s, p)] == n
    assert r.fill == 0 and r.tix == r.cons_tile == nsteps * len(rows)


# (D, V, G SMs, L, R of the 1-row kernel, R of the 8-row kernel).  For D = 1280 the R are those idx_gpt_init computes
# from a 227 KB shared-memory budget at that SM count: on the 132-SM H100 SXM the 8-row ring is exactly its largest phase
# (the 63-row mel head), with no spare row; at 148 SMs that phase is 56 rows.  The D = 256 rings are deep ones.
GEOMS = [
    (1280, 8194, 132, 24, 71, 63),
    (1280, 8194, 148, 24, 72, 63),
    (256, 8194, 148, 3, 400, 380),
]


@pytest.mark.parametrize("D,V,G,L,R1,R8", GEOMS)
@pytest.mark.parametrize("cap", [4, 6, 12, 18, 24, 255])
def test_every_cta_geometry_never_waits_for_an_unissued_phase(D, V, G, L, R1, R8, cap):
    seen = set()
    for cta in range(G):
        rows = tuple(cta_phases(D, V, G, cta, L))
        if rows in seen:
            continue
        seen.add(rows)
        assert max(rows) <= min(R1, R8)
        for nsteps in (1, 3):
            r = run_decode8(list(rows), R8, nsteps, cap, L)
            check_stream(r, rows, nsteps)
            r = run_decode1(list(rows), R1, nsteps, cap, L)
            check_stream(r, rows, nsteps)


def test_smallest_legal_ring_and_odd_caps():
    # R = the largest phase exactly (the host refuses anything smaller): the ring degenerates to one phase at a time
    rows = cta_phases(1280, 8194, 148, 0, 2)
    R = max(rows)
    for cap, nsteps in itertools.product((1, 4, 5, 7, 255), (1, 2)):
        check_stream(run_decode8(list(rows), R, nsteps, cap, 2), rows, nsteps)
        check_stream(run_decode1(list(rows), R, nsteps, cap, 2), rows, nsteps)


def test_early_exit_leaves_only_waitable_phases():
    # the kernels stop consuming when every sequence has finished: what was issued must be drainable — complete phases are
    # waited for, a partly issued phase is closed with a plain arrive first (its bytes then complete it)
    rows = cta_phases(1280, 8194, 148, 7, 24)
    r = Ring(list(rows), 62, 4, 6)
    r.issue_fitting(62)
    r.wait(); r.advance(rows[0])
    outstanding = r.tix - r.cons_tile
    assert 0 <= outstanding < NBAR
    assert r.part < rows[r.pidx]
    assert r.fill == sum(m for (_, _, _, m) in r.issued) - rows[0]


def test_fragment_order_is_a_permutation_matching_the_mma_layout():
    """frag_idx of gpt_decode8.cuh: element k of an activation row -> position in global memory, such that thread t4 of the
    MMA finds {b0, b1} of k-steps 2j, 2j + 1 in the four consecutive 32-bit words 16 j + 4 t4 .. + 3."""
    def frag_idx(k):
        kk, r = k >> 4, k & 15
        word = (kk >> 1) * 16 + ((r & 7) >> 1) * 4 + (kk & 1) * 2 + (r >> 3)
        return word * 2 + (r & 1)

    D = 1280
    perm = [frag_idx(k) for k in range(D)]
    assert sorted(perm) == list(range(D))
    # m16n8k16 B fragment: b0 = B[k0 + 2 t4 .. + 1][n], b1 = B[k0 + 8 + 2 t4 .. + 1][n]
    for j in range(D // 32):
        for t4 in range(4):
            base = (16 * j + 4 * t4) * 2
            want = []
            for kk in (2 * j, 2 * j + 1):
                want += [16 * kk + 2 * t4, 16 * kk + 2 * t4 + 1, 16 * kk + 8 + 2 * t4, 16 * kk + 8 + 2 * t4 + 1]
            assert [perm.index(base + i) for i in range(8)] == want
