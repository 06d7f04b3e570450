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


def stream_segment(engine, prompt_emb, prompt_condition, ref_mel, style, *, chunk_codes=100, overlap_codes=20,
                   duration_factor=1.0, n_steps=25, cfg_rate=0.7, **generation_kwargs):
    """Decode one segment and yield its audio as int16 arrays, window by window.

    prompt_emb: the [cond][text] rows of Engine.gpt_prepare_inputs.  prompt_condition [P, content_dim], ref_mel [80, P],
    style [style_dim]: the tensors infer_generator caches (cache_s2mel_prompt, cache_mel, cache_s2mel_style).
    generation_kwargs: those of Engine.gpt_generate (max_new_tokens defaults to the reference's 1500).  Each window's
    codes are cut before the stop token (infer_v2_5.py:809-821); its noise z [80, P + F] is drawn with torch.randn, as
    cfm.inference draws it, on the device of ref_mel.  The arrays live where ref_mel lives (numpy for host inputs)."""
    ws = WindowSchedule(chunk_codes, overlap_codes)
    ovlp = overlap_samples(overlap_codes, duration_factor)
    if window_frames(chunk_codes, duration_factor) * HOP < 2 * ovlp:
        raise ValueError("a full window must hold at least twice the overlap: chunk_codes too small for overlap_codes")
    generation_kwargs.setdefault("max_new_tokens", 1500)
    stop = engine.gpt_cfg.stop_mel_token
    P = int(ref_mel.shape[-1])
    dev = ref_mel.device if (torch is not None and isinstance(ref_mel, torch.Tensor)) else "cpu"
    first = True

    def window(codes, last):
        nonlocal first
        F = window_frames(len(codes), duration_factor)
        z = torch.randn(80, P + F, device=dev)
        if dev == "cpu":
            z = z.numpy()
        out = engine.stream_vocode(np.ascontiguousarray(codes), prompt_condition, ref_mel, style, z, F,
                                   overlap_samples=ovlp, first=first, last=last, n_steps=n_steps, cfg_rate=cfg_rate)
        first = False
        return out["pcm"]

    with engine.gpt_stream(prompt_emb, **generation_kwargs) as st:
        n = 0
        finished = False
        while not finished:
            _, finished = st.next(ws.next_end)
            codes = st.codes
            hit = np.flatnonzero(codes == stop)
            n = int(hit[0]) if hit.size else len(codes)
            finished = finished or bool(hit.size)
            for a, b in ws.ready(n):
                yield window(codes[a:b], False)
    fin = ws.final(n)
    if fin is not None:
        yield window(st.codes[fin[0]:fin[1]], True)
    elif not first:
        yield engine.stream_vocode(None, last=True)["pcm"]
