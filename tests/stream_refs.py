"""Host model of the window join of idx_stream_vocode (include/idxtts.h): the cross-fade rules of the reference's
StreamingDecoder.generate, restated in numpy.  tests/test_stream_cpu.py checks it against the reference's own output
(tests/golden/stream_join.npz); tests/test_stream_gpu.py checks the device join against it."""
import numpy as np


def _to_int16(x):
    return np.clip(x * 32767, -32767, 32767).astype(np.int16)


def _fade_out(x):
    if len(x) <= 512:
        return x
    x = x.copy()
    x[-512:] *= np.linspace(1.0, 0.0, 512)
    return x


class HostJoin:
    """The join state of one stream: push() takes a window's fp32 waveform and returns the int16 samples it emits."""

    def __init__(self):
        self.tail = None

    def push(self, wav, ovlp, first=False, last=False):
        if first:
            self.tail = None
        wav = np.asarray(wav, np.float32)
        if self.tail is None:
            if last:
                return _to_int16(_fade_out(wav))
            split = len(wav) - ovlp
            self.tail = wav[split:]
            return _to_int16(wav[:split])
        head, rest = wav[:ovlp], wav[ovlp:]
        n = min(len(self.tail), len(head))
        if n:
            w = np.hanning(2 * n)
            blend = self.tail[:n] * w[n:] + head[:n] * w[:n]
        else:
            blend = np.zeros(0, np.float32)
        if last:
            self.tail = None
            return _to_int16(_fade_out(np.concatenate([blend, rest])))
        split = len(rest) - ovlp
        self.tail = rest[split:]
        return _to_int16(np.concatenate([blend, rest[:split]]))

    def flush(self):
        if self.tail is None:
            return None
        out, self.tail = _to_int16(_fade_out(self.tail)), None
        return out
