"""Chunked streaming of one text segment: int16 audio comes out window by window while the segment's speech tokens are
still being decoded.

The design is the one the reference ships in its TensorRT backend (`StreamingDecoder` over `generate_chunks`): whenever
`chunk_codes` codes are committed, the window of the last `chunk_codes` codes is vocoded together with the speaker
prompt, and consecutive windows are cross-faded over `overlap_codes` codes' worth of samples with a Hann window; the
last window is faded out over 512 samples.  Here the decode is the engine's resumable decode (Engine.gpt_stream), each
window runs the engine's tail (Engine.stream_vocode, the tail of codes_to_wav) and the cross-fade is done on the device.
Everything runs serially on the engine stream: the decode kernel is a cooperative launch over every SM.

`IndexTTS2.infer()` / `infer_generator()` are not changed: a chunk from inside a segment cannot come out of the
reference's own generator without restating its front half.  A caller that wants chunks builds the segment's inputs
(Engine.gpt_prepare_inputs and the prompt tensors `infer_generator` caches) and iterates `stream_segment`.
"""
import numpy as np

try:
    import torch
except Exception:  # pragma: no cover
    torch = None

HOP = 256                 # BigVGAN samples per mel frame
CODE_TO_FRAME = 1.72      # mel frames per codec frame (infer_v2_5.py:833); the codec gives 2 frames per code


def window_frames(n_codes, duration_factor=1.0):
    """Mel frames of a window of n codes: int(2 n 1.72 duration_factor), the rule of idx_vocode_request.F."""
    return int(2 * n_codes * CODE_TO_FRAME * duration_factor)


def overlap_samples(overlap_codes, duration_factor=1.0):
    """Cross-fade length in samples.  The frame rule of this codec (2 frames per code), i.e. int(2 n 1.72 df) * 256;
    the TensorRT file's int(n * 1.72) * 256 is the rule of the IndexTTS-2 codec (1 frame per code)."""
    return window_frames(overlap_codes, duration_factor) * HOP


class WindowSchedule:
    """The window schedule of generate_chunks for one sequence: window c covers codes [c stride, c stride + chunk) with
    stride = chunk - overlap and is due as soon as that many codes exist; when the sequence ends, a final partial window
    [c stride, n) covers the codes after the last full window, if any remain."""

    def __init__(self, chunk_codes=100, overlap_codes=20):
        if chunk_codes - overlap_codes <= 0:
            raise ValueError(f"overlap_codes ({overlap_codes}) must be less than chunk_codes ({chunk_codes})")
        self.chunk, self.stride = int(chunk_codes), int(chunk_codes - overlap_codes)
        self.next_end = self.chunk          # end of the next full window

    def ready(self, n_codes):
        """The full windows (start, end) due now that n_codes speech codes exist."""
        out = []
        while n_codes >= self.next_end:
            out.append((self.next_end - self.chunk, self.next_end))
            self.next_end += self.stride
        return out

    def final(self, n_codes):
        """The final partial window (start, n_codes) of a sequence that ended with n_codes speech codes, or None."""
        start = self.next_end - self.chunk
        return (start, n_codes) if start < n_codes else None


def schedule(n_codes, chunk_codes=100, overlap_codes=20):
    """Every window (start, end, last) of a sequence of n_codes speech codes, in the order stream_segment runs them."""
    ws = WindowSchedule(chunk_codes, overlap_codes)
    out = [(a, b, False) for a, b in ws.ready(n_codes)]
    fin = ws.final(n_codes)
    if fin is not None:
        out.append((fin[0], fin[1], True))
    return out


def stream_segments(engine, prompts, prompt_condition, ref_mel, style, *, chunk_codes=100, overlap_codes=20,
                    duration_factor=1.0, n_steps=25, cfg_rate=0.7, **generation_kwargs):
    """Decode several segments as one decode group and yield their audio, round by round, as (audio_list, done_list):
    the shape of the reference's batch StreamingDecoder.generate.  audio_list[i] is request i's int16 array of the round,
    or None when it has nothing this round; done_list[i] is True on the round that emits its last samples (exactly once
    per request; a request that ends without a single code is done with audio None).

    prompts: the [cond][text] rows of Engine.gpt_prepare_inputs, one per request; len(prompts) * num_beams must fit in
    one decode group (max_batch).  prompt_condition, ref_mel, style: one set shared by every request, or lists with one
    per request (P may differ).  Request i has its own window schedule (that of generate_chunks for that sample alone: a
    request's last window runs as soon as that request finishes) and join slot i.

    A round is one Engine.stream_vocode_batch call: after each GptStreamBatch.next (which returns as soon as a request
    reaches its next window end or finishes), every window that is due (full windows, the final partial window of a
    request that finished, the flush of one that ended without one) runs in one call; a request with several due
    windows has them run in consecutive rounds.  Window noise z [80, P_i + F] is drawn with torch.randn on the device of
    ref_mel, one draw per window, in the order the rounds run and, within a round, in request order."""
    n_req = len(prompts)
    per_req = isinstance(ref_mel, (list, tuple))
    pcs, mels, styles = ((list(x) if per_req else [x] * n_req) for x in (prompt_condition, ref_mel, style))
    if len(mels) != n_req or len(pcs) != n_req or len(styles) != n_req:
        raise ValueError("prompt_condition / ref_mel / style: one set, or one per prompt")
    ovlp = overlap_samples(overlap_codes, duration_factor)
    if window_frames(chunk_codes, duration_factor) * HOP < 2 * ovlp:
        raise ValueError("a full window must hold at least twice the overlap: chunk_codes too small for overlap_codes")
    generation_kwargs.setdefault("max_new_tokens", 1500)
    stop = engine.gpt_cfg.stop_mel_token
    scheds = [WindowSchedule(chunk_codes, overlap_codes) for _ in range(n_req)]
    started = [False] * n_req           # a window of the request has run: its slot may keep a tail
    ended = [False] * n_req             # the request's last codes are known
    pending = [[] for _ in range(n_req)]   # due windows: (start, end, last), or None for the flush
    reported = [False] * n_req

    def devof(m):
        return m.device if (torch is not None and isinstance(m, torch.Tensor)) else "cpu"

    def rounds(st):
        while any(pending):
            calls, who = [], []
            for i in range(n_req):
                if not pending[i]:
                    continue
                w = pending[i].pop(0)
                if w is None:
                    calls.append(dict(slot=i, codes=None, last=True))
                else:
                    a, b, last = w
                    F = window_frames(b - a, duration_factor)
                    P = int(mels[i].shape[-1])
                    z = torch.randn(80, P + F, device=devof(mels[i]))
                    if devof(mels[i]) == "cpu":
                        z = z.numpy()
                    calls.append(dict(slot=i, codes=np.ascontiguousarray(st.codes[i][a:b]), prompt_condition=pcs[i],
                                      ref_mel=mels[i], style=styles[i], z=z, F=F, overlap_samples=ovlp,
                                      first=not started[i], last=last))
                    started[i] = True
                who.append(i)
            outs = engine.stream_vocode_batch(calls, n_steps, cfg_rate)
            audio, done = [None] * n_req, [False] * n_req
            for i, o in zip(who, outs):
                audio[i] = o["pcm"]
                if ended[i] and not pending[i]:
                    done[i] = reported[i] = True
            yield audio, done

    with engine.gpt_stream_batch(prompts, **generation_kwargs) as st:
        while not all(ended):
            st.next([1 if ended[i] else scheds[i].next_end for i in range(n_req)])
            silent = [False] * n_req
            for i in range(n_req):
                if ended[i]:
                    continue
                codes = st.codes[i]
                hit = np.flatnonzero(codes == stop)
                n = int(hit[0]) if hit.size else len(codes)
                pending[i] += [(a, b, False) for a, b in scheds[i].ready(n)]
                if st.finished[i] or hit.size:
                    ended[i] = True
                    fin = scheds[i].final(n)
                    if fin is not None:
                        pending[i].append((fin[0], fin[1], True))
                    elif started[i] or pending[i]:
                        pending[i].append(None)
                    else:
                        silent[i] = reported[i] = True
            yield from rounds(st)
            if any(silent):
                yield [None] * n_req, silent


class StreamServer:
    """Chunked streaming for a caller that serves clients: requests are submitted at any time and join a running decode
    group (Engine.gpt_serve) as its slots free up, instead of waiting for a whole stream_segments group to drain.

    submit() queues a request and returns its id; before each decode call the waiting requests are admitted in
    submission order, each into the lowest free slot, which is also its join slot of Engine.stream_vocode_batch.  round()
    runs one round and returns its events (rid, pcm or None, done).  A request's windows, noise draws, first / last
    flags, flush and silent-end rules are those of stream_segments for that request alone: its window schedule cut
    before the stop token, one torch.randn(80, P + F) per window on the device of its ref_mel (within a round in slot
    order), its first window with first=True, done exactly once.  A round runs a decode call only when no window is
    waiting, then at most one window per slot in one stream_vocode_batch call.  A slot is released when its request is
    done or cancelled.

    The sequence index of a request is its id (the submission counter) and the sampling seed is drawn once per server
    from torch's generator unless `seed` is passed, so request i decodes the codes gpt_generate returns for request i of
    all submitted prompts with that seed (when that call decodes it in a group of at least 2 requests).  The slots stay
    in one gpt_decode8_kernel group even when a single request is live."""

    def __init__(self, engine, slots=8, chunk_codes=100, overlap_codes=20, duration_factor=1.0, n_steps=25, cfg_rate=0.7,
                 **generation_kwargs):
        self._ovlp = overlap_samples(overlap_codes, duration_factor)
        WindowSchedule(chunk_codes, overlap_codes)        # refuses overlap_codes >= chunk_codes
        if window_frames(chunk_codes, duration_factor) * HOP < 2 * self._ovlp:
            raise ValueError("a full window must hold at least twice the overlap: chunk_codes too small for overlap_codes")
        generation_kwargs.setdefault("max_new_tokens", 1500)
        if "seed" not in generation_kwargs:
            generation_kwargs["seed"] = int(torch.randint(0, 2 ** 62, (1,)).item())
        self._eng, self._chunk, self._overlap, self._df = engine, chunk_codes, overlap_codes, duration_factor
        self._n_steps, self._cfg_rate = n_steps, cfg_rate
        self._stop = engine.gpt_cfg.stop_mel_token
        self._gen = engine.gpt_serve(slots, **generation_kwargs)
        self._waiting = []                  # rids in submission order
        self._req = {}                      # rid -> request state, from submit until done or cancel
        self._slot = [None] * slots         # rid in each slot
        self._count = 0

    def submit(self, prompt_emb, prompt_condition, ref_mel, style):
        """Queue one request (the arguments of stream_segment); returns its id."""
        rid = self._count
        self._count += 1
        self._req[rid] = dict(prompt=prompt_emb, pc=prompt_condition, mel=ref_mel, style=style, slot=None,
                              sched=WindowSchedule(self._chunk, self._overlap), pending=[], started=False, ended=False)
        self._waiting.append(rid)
        return rid

    def cancel(self, rid):
        """Drop a waiting or running request: no event of it follows.  Returns False when it is unknown or done."""
        r = self._req.pop(rid, None)
        if r is None:
            return False
        if r["slot"] is None:
            self._waiting.remove(rid)
        else:
            self._free(r["slot"])
        return True

    @property
    def busy(self):
        """Whether a request is waiting or running."""
        return bool(self._req)

    def _free(self, slot):
        self._gen.release(slot)
        self._slot[slot] = None

    def _decode(self):
        events = []
        for s in range(len(self._slot)):
            if self._slot[s] is None and self._waiting:
                rid = self._waiting.pop(0)
                self._gen.admit(s, self._req[rid]["prompt"], rid)
                self._req[rid]["slot"], self._slot[s] = s, rid
        live = [s for s, rid in enumerate(self._slot) if rid is not None and not self._req[rid]["ended"]]
        if not live:
            return events
        self._gen.next([self._req[rid]["sched"].next_end if rid is not None else 1 for rid in self._slot])
        for s in live:
            r = self._req[self._slot[s]]
            codes = self._gen.codes[s]
            hit = np.flatnonzero(codes == self._stop)
            n = int(hit[0]) if hit.size else len(codes)
            r["codes"] = codes
            r["pending"] += [(a, b, False) for a, b in r["sched"].ready(n)]
            if self._gen.finished[s] or hit.size:
                r["ended"] = True
                fin = r["sched"].final(n)
                if fin is not None:
                    r["pending"].append((fin[0], fin[1], True))
                elif r["started"] or r["pending"]:
                    r["pending"].append(None)
                else:                       # ended without a single code: done, silent
                    events.append((self._slot[s], None, True))
                    del self._req[self._slot[s]]
                    self._free(s)
        return events

    def round(self):
        """One round: a decode call when no window is waiting (after admitting waiting requests), then every slot's next
        due window in one stream_vocode_batch call.  Returns the round's events (rid, pcm int16 array or None, done)."""
        events = []
        if not any(self._req[rid]["pending"] for rid in self._slot if rid is not None):
            events += self._decode()
        calls, who = [], []
        for s, rid in enumerate(self._slot):
            if rid is None or not self._req[rid]["pending"]:
                continue
            r = self._req[rid]
            w = r["pending"].pop(0)
            if w is None:
                calls.append(dict(slot=s, codes=None, last=True))
            else:
                a, b, last = w
                F = window_frames(b - a, self._df)
                dev = r["mel"].device if (torch is not None and isinstance(r["mel"], torch.Tensor)) else "cpu"
                z = torch.randn(80, int(r["mel"].shape[-1]) + F, device=dev)
                calls.append(dict(slot=s, codes=np.ascontiguousarray(r["codes"][a:b]), prompt_condition=r["pc"],
                                  ref_mel=r["mel"], style=r["style"], z=z.numpy() if dev == "cpu" else z, F=F,
                                  overlap_samples=self._ovlp, first=not r["started"], last=last))
                r["started"] = True
            who.append(s)
        if calls:
            outs = self._eng.stream_vocode_batch(calls, self._n_steps, self._cfg_rate)
            for s, o in zip(who, outs):
                rid = self._slot[s]
                done = self._req[rid]["ended"] and not self._req[rid]["pending"]
                events.append((rid, o["pcm"], done))
                if done:
                    del self._req[rid]
                    self._free(s)
        return events

    def close(self):
        """End the serving group; requests still waiting or running are dropped."""
        self._gen.close()
        self._req.clear()
        self._waiting.clear()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
        return False


def stream_segment(engine, prompt_emb, prompt_condition, ref_mel, style, **kwargs):
    """Decode one segment and yield its audio as int16 arrays, window by window: the one-request case of
    stream_segments.

    prompt_emb: the [cond][text] rows of Engine.gpt_prepare_inputs.  prompt_condition [P, content_dim], ref_mel [80, P],
    style [style_dim]: the tensors infer_generator caches (cache_s2mel_prompt, cache_mel, cache_s2mel_style).
    kwargs: chunk_codes, overlap_codes, duration_factor, n_steps, cfg_rate and those of Engine.gpt_generate
    (max_new_tokens defaults to the reference's 1500).  Each window's codes are cut before the stop token
    (infer_v2_5.py:809-821); its noise z [80, P + F] is drawn with torch.randn, as cfm.inference draws it, on the device
    of ref_mel.  The arrays live where ref_mel lives (numpy for host inputs)."""
    for audio, _ in stream_segments(engine, [prompt_emb], prompt_condition, ref_mel, style, **kwargs):
        if audio[0] is not None:
            yield audio[0]
