"""Mint tests/golden/tail_full_cfg2.npz: the per-segment tail (codec decode -> length regulator -> cat with the prompt
condition -> CFM 25 Euler steps, CFG 0.7 -> drop the prompt frames -> BigVGAN) at the FULL BASELINE config-2 geometry
(256 codes, P = 861 prompt frames, F = 880, T = 1741, [ASSUMED] 13 x 512 DiT, BigVGAN-v2 22 kHz) in fp32 on the CPU with the
restated oracle chain (oracle/s2mel.py + oracle/bigvgan.py, themselves pinned to the reference's modules and, at the small
geometry, to the executed infer_v2_5.py:827-856 source lines: oracle/make_goldens_tail.py).  Inputs are regenerated from the
seed by the test; only the outputs are stored (wav fp32 225 280 samples, mel 80 x 880).  Build container only; ~10 min on 8 vCPU.
    python -m oracle.make_goldens_tail_full"""
import os
import time

import numpy as np
import torch

from indextts_b200 import synth
from oracle.bigvgan import bigvgan_forward
from oracle.s2mel import cfm_inference, codec_decode, fold_weight_norm, length_regulate

SEED = 20250923
N_CODES, P = 256, 861


def make_inputs(seed=SEED):
    """The test regenerates exactly these (torch CPU generator: identical on every box)."""
    g = torch.Generator().manual_seed(seed)
    cc = dict(synth.CODEC_CFG)
    codes = torch.randint(0, cc["codebook_size"], (1, N_CODES), generator=g)
    prompt_condition = torch.randn(1, P, 512, generator=g)
    ref_mel = torch.randn(1, 80, P, generator=g) * 1.5 - 4.0
    style = torch.randn(1, 192, generator=g)
    F = int(2 * N_CODES * 1.72)
    z = torch.randn(1, 80, P + F, generator=g)
    return codes, prompt_condition, ref_mel, style, z, F


def main():
    torch.set_num_threads(os.cpu_count() or 1)
    c, cc, h = dict(synth.S2MEL_CFG), dict(synth.CODEC_CFG), dict(synth.BIGVGAN_V2_22K)
    ws = fold_weight_norm(synth.make_s2mel_weights(c, seed=1234))
    wc = fold_weight_norm(synth.make_codec_weights(cc, seed=4321))
    wb = synth.make_bigvgan_weights(h, seed=1234)
    codes, pc, ref_mel, style, z, F = make_inputs()
    t0 = time.perf_counter()
    with torch.no_grad():
        S = codec_decode(wc, codes)
        cond = length_regulate(ws, S, F)
        t1 = time.perf_counter()
        mu = torch.cat([pc, cond], 1)
        mel = cfm_inference(ws, c, mu, torch.LongTensor([P + F]), ref_mel, style, z, 25, 0.7)
        t2 = time.perf_counter()
        wav = bigvgan_forward(h, wb, mel[:, :, P:].float())
        t3 = time.perf_counter()
    wav = wav.reshape(-1).numpy().astype(np.float32)
    print(f"codec+regulator {t1 - t0:.1f} s, CFM {t2 - t1:.1f} s, BigVGAN {t3 - t2:.1f} s on {torch.get_num_threads()} threads; "
          f"wav {wav.shape} rms {np.sqrt((wav ** 2).mean()):.4f} max {np.abs(wav).max():.3f}")
    out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "tail_full_cfg2.npz")
    np.savez_compressed(out, seed=SEED, F=F, wav=wav, mel=mel[0, :, P:].numpy().astype(np.float16))   # fp16 mel: printed only, keeps the file < 1 MB
    print("wrote", out, os.path.getsize(out) // 1024, "KiB")


if __name__ == "__main__":
    main()
