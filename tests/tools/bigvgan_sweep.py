"""BASELINE config 4: BigVGAN-only throughput sweep on one H100 (mel frames 128-4096, batch 1-16), device-resident
mel and wav, CUDA-event time of idx_bigvgan_forward (engine stream).  Prints samples/s and the fraction of the
measured dense bf16 tensor peak using 1.8037 GFLOP per mel frame (SURVEY section 8d); the GEMMs run in tf32.
    python -m tests.tools.bigvgan_sweep"""
import json
import os

import torch

from indextts_b200 import synth
from indextts_b200.engine import Engine


def main():
    e = Engine(0)
    h = dict(synth.BIGVGAN_V2_22K)
    e.load_state_dict("bigvgan.", synth.make_bigvgan_weights(h, seed=1234))
    e.bigvgan_init(h)
    peaks = {}
    pth = os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))), "MEASURED_PEAKS.json")
    if os.path.exists(pth):
        peaks = json.load(open(pth))
    tf = float(peaks.get("bf16_tflops_sustained", peaks.get("bf16_tflops", 1449.5)))
    g = torch.Generator().manual_seed(0)
    rows = []
    for B in (1, 4, 16):
        for F in (128, 256, 512, 1024, 2048, 4096):
            if B * F > 16384:
                continue
            mel = (torch.randn(B, 80, F, generator=g) * 2.0 - 5.0).clamp(-11.5, 2.0).cuda()
            wav = torch.empty(B, 1, F * 256, device="cuda")
            for _ in range(2):
                e.bigvgan_forward(mel, out=wav)
            ms = []
            for _ in range(3):
                e.bigvgan_forward(mel, out=wav)
                ms.append(e.bigvgan_last_ms())
            t = sorted(ms)[1]
            fl = 1.8037e9 * F * B
            rows.append((B, F, t, B * F * 256 / (t * 1e-3), fl / (t * 1e-3) / 1e12))
            print(f"B={B:3d} F={F:5d}: {t:8.3f} ms  {rows[-1][3] / 1e6:8.2f} Msamples/s  {rows[-1][4]:6.1f} TFLOP/s "
                  f"({100 * rows[-1][4] / tf:4.1f} % of {tf:.0f} bf16 peak)", flush=True)
    e.close()


if __name__ == "__main__":
    main()
