"""BASELINE config 3: IndexTTS-2.5, 32 utterances of one speaker, 512 speech tokens each (20.45 s of audio each), full
gpt -> codec -> length regulator -> CFM (25 steps, CFG 0.7, T = 861 + 1761) -> BigVGAN pipeline on ONE H100, synthetic
weights and inputs.  GPT decodes 8 utterances per group (4 groups back to back), the tail runs per utterance.
Prints RTF (= wall / 654 s of audio) and speech-tokens/s (= 16384 / GPT time).
    python -m tests.tools.config3 [n_utt] [n_tokens]"""
import sys
import time

import numpy as np
import torch

from indextts_b200 import synth
from indextts_b200.engine import Engine, fold_weight_norm
from tests.gpt_common import gpt_config, load_gpt, make_gpt_weights, prepare_gpt_inputs, r16


def main():
    n_utt = int(sys.argv[1]) if len(sys.argv) > 1 else 32
    n_tok = int(sys.argv[2]) if len(sys.argv) > 2 else 512
    e = Engine(0)
    cfg = gpt_config()
    w = make_gpt_weights(cfg, seed=2025, bf16=True)
    load_gpt(e, cfg, w, max_batch=8, max_prompt=80)
    c, cc, h = dict(synth.S2MEL_CFG), dict(synth.CODEC_CFG), dict(synth.BIGVGAN_V2_22K)
    ws = fold_weight_norm(synth.make_s2mel_weights(c, seed=1234))
    e.load_state_dict("s2mel.", {k: v for k, v in ws.items() if v.is_floating_point()})
    e.load_state_dict("codec.", fold_weight_norm(synth.make_codec_weights(cc, seed=4321)))
    e.s2mel_init(c); e.codec_init(cc)
    e.load_state_dict("bigvgan.", synth.make_bigvgan_weights(h, seed=1234))
    e.bigvgan_init(h)
    g = torch.Generator().manual_seed(0)
    P = 861
    F = int(2 * n_tok * 1.72)
    style = torch.randn(192, generator=g)
    emo = r16(torch.randn(cfg["model_dim"], generator=g) * 0.5)
    pc = torch.randn(P, 512, generator=g).cuda()
    ref_mel = (torch.randn(80, P, generator=g) * 1.5 - 4.0).cuda()
    sty = style.cuda()
    prompts = []
    for u in range(n_utt):
        L = int(torch.randint(24, 61, (1,), generator=g))
        text = torch.randint(2, 12000, (L,), generator=g)
        prompts.append(prepare_gpt_inputs(w, style, emo, text, lang=1, bf16=True).numpy())
    zs = [torch.randn(80, P + F, generator=g).cuda() for _ in range(2)]
    # warm-up
    e.gpt_generate(prompts[:8], 8, 10.0, forbid_stop_before=8)
    codes0 = np.random.default_rng(0).integers(0, 8192, n_tok).astype(np.int32)
    e.codes_to_wav(codes0, pc, ref_mel, sty, zs[0], F, 25, 0.7, want_wav=False, want_pcm16=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    gpt_ms = 0.0
    all_codes = []
    for g0 in range(0, n_utt, 8):
        grp = prompts[g0:g0 + 8]
        out = e.gpt_generate(grp, n_tok, 10.0, forbid_stop_before=n_tok)
        t = e.gpt_last_timing()
        gpt_ms += t["prefill_ms"] + t["decode_ms"]
        all_codes += out
    t1 = time.perf_counter()
    cfm_ms = voc_ms = 0.0
    for u, codes in enumerate(all_codes):
        e.codes_to_wav(np.minimum(codes, 8191), pc, ref_mel, sty, zs[u & 1], F, 25, 0.7, want_wav=False, want_pcm16=True)
        cfm_ms += e.s2mel_last_ms()["cfm_ms"]
        voc_ms += e.bigvgan_last_ms()
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    audio_s = n_utt * n_tok * (2 * 1.72 * 256 / 22050.0)      # 39.94 ms of audio per speech token
    print(f"config 3: {n_utt} utterances x {n_tok} tokens (T = {P + F}, F = {F}): wall {t2 - t0:.2f} s "
          f"(GPT {t1 - t0:.2f} s, tail {t2 - t1:.2f} s; device: gpt {gpt_ms / 1000:.2f} s, cfm {cfm_ms / 1000:.2f} s, "
          f"bigvgan {voc_ms / 1000:.2f} s) -> RTF {(t2 - t0) / audio_s:.4f}, {n_utt * n_tok / (gpt_ms / 1000):.0f} speech tokens/s (GPT), "
          f"{n_utt * n_tok / (t2 - t0):.0f} tokens/s end to end")
    e.close()


if __name__ == "__main__":
    main()
