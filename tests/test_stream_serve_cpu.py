"""Scheduling of indextts_b200.streaming.StreamServer against a fake engine that records every call: FIFO admission into
the lowest free slot before each decode call, at most one window per slot per round, `first` on the first window of
every slot occupant, the release of finished and cancelled slots, each request's windows against the solo schedule of
streaming.schedule, and the event rules (one done per request, nothing after a cancel)."""
import numpy as np
import pytest

STOP = 8193
MAX_NEW = 300


class FakeServe:
    """Engine.gpt_serve's GptServe: the request with sequence index i (prompt [[L]]) decodes codes 0, 1, .., L - 1 and
    then the stop code (none when L >= max_new); next() follows the return rules of idx_gpt_serve_next."""

    def __init__(self, log, slots, max_new):
        self.log, self.slots, self.max_new = log, slots, max_new
        self.occupied, self.n_committed, self.finished = [False] * slots, [0] * slots, [False] * slots
        self.seq, self._len, self._codes = [None] * slots, [0] * slots, [np.zeros(0, np.int32)] * slots

    @property
    def codes(self):
        return [c[:n] if o else None for c, n, o in zip(self._codes, self.n_committed, self.occupied)]

    def admit(self, slot, prompt, seq_index):
        assert not self.occupied[slot]
        self.log.append(("admit", slot, seq_index))
        L = int(prompt[0][0])
        self._codes[slot] = np.array(list(range(L)) + [STOP], np.int32)[:self.max_new]
        self.occupied[slot], self.n_committed[slot], self.finished[slot], self.seq[slot] = True, 0, False, seq_index

    def release(self, slot):
        assert self.occupied[slot]
        self.log.append(("release", slot, self.seq[slot], self.finished[slot]))
        self.occupied[slot], self.seq[slot] = False, None

    def next(self, until):
        self.log.append(("next", [s for s in range(self.slots) if not self.occupied[s]]))
        fin0 = list(self.finished)
        while True:
            live = [s for s in range(self.slots) if self.occupied[s] and not self.finished[s]]
            if (not live or any(self.n_committed[s] >= until[s] for s in live)
                    or any(self.occupied[s] and self.finished[s] and not fin0[s] for s in range(self.slots))):
                break
            left = min([32] + [min(until[s], self.max_new) - self.n_committed[s] for s in live])
            for _ in range(left):
                for s in live:
                    if self.finished[s]:
                        continue
                    c = self._codes[s][self.n_committed[s]]
                    self.n_committed[s] += 1
                    self.finished[s] = c == STOP or self.n_committed[s] == self.max_new
        return None, list(self.finished)

    def close(self):
        self.log.append(("close",))


class FakeEngine:
    class gpt_cfg:
        stop_mel_token = STOP

    def __init__(self):
        self.log, self.gen = [], None

    def gpt_serve(self, slots, **kw):
        self.gen = FakeServe(self.log, slots, kw["max_new_tokens"])
        return self.gen

    def stream_vocode_batch(self, calls, n_steps, cfg_rate):
        rec = []
        for c in calls:
            w = None if c["codes"] is None else (int(c["codes"][0]), int(c["codes"][-1]) + 1, c["last"], c["first"])
            rec.append((c["slot"], self.gen.seq[c["slot"]], w))
        self.log.append(("vocode", rec))
        return [dict(pcm=np.zeros(3, np.int16)) for _ in calls]


def _prompt(L):
    return np.array([[L]], np.float32)


def _run(lengths, slots, arrivals, cancels=None, chunk=40, overlap=10):
    """Serve requests of the given code lengths; arrivals[i] is the round before which request i is submitted, cancels
    maps a round to the rids cancelled before it.  Returns (engine log, [(events, log index where the round starts,
    round)], rids)."""
    import torch
    from indextts_b200.streaming import StreamServer
    torch.manual_seed(0)
    eng = FakeEngine()
    srv = StreamServer(eng, slots=slots, chunk_codes=chunk, overlap_codes=overlap, max_new_tokens=MAX_NEW)
    mel = np.zeros((80, 5), np.float32)
    rounds, rids, r, submitted = [], {}, 0, 0
    while submitted < len(lengths) or srv.busy:
        for i, at in enumerate(arrivals):
            if at == r:
                rids[i] = srv.submit(_prompt(lengths[i]), None, mel, None)
                submitted += 1
        for rid in (cancels or {}).get(r, []):
            assert srv.cancel(rid)
        n_log = len(eng.log)
        rounds.append((srv.round(), n_log, r))
        r += 1
        assert r < 10_000
    srv.close()
    return eng.log, rounds, rids


LENGTHS = [95, 0, 40, 250, 31, 130, 70, 70, 299, 12, 160, 55]


@pytest.mark.parametrize("slots", [2, 4, 8])
def test_fifo_admission_into_lowest_free_slot(slots):
    arrivals = [0, 0, 0, 1, 1, 3, 3, 3, 6, 9, 9, 12]
    log, rounds, rids = _run(LENGTHS, slots, arrivals)
    admits = [x for x in log if x[0] == "admit"]
    assert [a[2] for a in admits] == list(range(len(LENGTHS)))              # submission order = sequence index
    occupied = set()
    for x in log:
        if x[0] == "admit":
            assert x[1] == min(set(range(slots)) - occupied)                  # the lowest free slot
            occupied.add(x[1])
        elif x[0] == "release":
            occupied.discard(x[1])
    # before each decode call every waiting request that fits has been admitted
    for k, (events, n_log, r) in enumerate(rounds):
        n_sub = sum(1 for a in arrivals if a <= r)
        end = rounds[k + 1][1] if k + 1 < len(rounds) else len(log)
        for j in range(n_log, end):
            if log[j][0] == "next" and log[j][1]:
                assert len([a for a in log[:j] if a[0] == "admit"]) == n_sub


@pytest.mark.parametrize("slots", [2, 3, 8])
@pytest.mark.parametrize("chunk,overlap", [(40, 10), (30, 0), (7, 3)])
def test_windows_follow_the_solo_schedule(slots, chunk, overlap):
    from indextts_b200.streaming import schedule
    arrivals = [0, 0, 1, 2, 2, 2, 5, 5, 8, 8, 8, 20]
    log, rounds, rids = _run(LENGTHS, slots, arrivals, chunk=chunk, overlap=overlap)
    per_seq = {i: [] for i in range(len(LENGTHS))}
    for x in log:
        if x[0] == "vocode":
            assert len({s for s, _, _ in x[1]}) == len(x[1])                  # at most one window per slot per round
            for s, seq, w in x[1]:
                per_seq[seq].append(w)
    for i, L in enumerate(LENGTHS):
        want = schedule(L, chunk, overlap)
        got = per_seq[i]
        full = [w for w in got if w is not None]
        assert [(a, b, last) for a, b, last, _ in full] == want, i
        assert [f for _, _, _, f in full] == [k == 0 for k in range(len(full))], i     # first on the first window only
        if want and not want[-1][2]:
            assert got[-1] is None and got.count(None) == 1, i                # the flush of a full last window
        else:
            assert None not in got, i
    # every event: one done per request, the silent request (0 codes) done without audio
    done = {}
    for events, _, _ in rounds:
        for rid, pcm, d in events:
            assert rid not in done, "event after done"
            if d:
                done[rid] = pcm
    assert sorted(done) == sorted(rids.values())
    assert done[rids[1]] is None
    # every slot is released once its request is done
    rel = [x for x in log if x[0] == "release"]
    assert sorted(x[2] for x in rel) == list(range(len(LENGTHS))) and all(x[3] for x in rel)


def test_cancel_releases_and_silences():
    arrivals = [0, 0, 0, 0, 1, 1]
    lengths = [250, 200, 90, 120, 60, 60]
    # request 0 (running) is cancelled before round 3, request 5 (waiting: 2 slots) before round 2
    log, rounds, rids = _run(lengths, 2, arrivals, cancels={3: [0], 2: [5]})
    rel = [x for x in log if x[0] == "release"]
    assert (0 in [x[2] for x in rel if not x[3]])                             # released live: a cancel
    assert 5 not in [x[2] for x in log if x[0] == "admit"]                   # never admitted
    for events, _, r in rounds:
        for rid, _, _ in events:
            if rid == 0:
                assert r < 3, "event of request 0 after its cancel"
            assert rid != 5
    dones = [rid for events, _, _ in rounds for rid, _, d in events if d]
    assert sorted(dones) == [1, 2, 3, 4]
    # the slot request 0 left is reused, and its next occupant starts with first=True
    slot0 = [x for x in log if x[0] == "admit" and x[2] == 0][0][1]
    later = [x for x in log if x[0] == "admit" and x[1] == slot0 and x[2] != 0]
    assert later
    ws = [w for x in log if x[0] == "vocode" for s, seq, w in x[1] if seq == later[0][2] and w is not None]
    assert [w[3] for w in ws] == [k == 0 for k in range(len(ws))] and ws
