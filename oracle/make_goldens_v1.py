"""Mint tests/golden/v1_vocoder_small.npz and (at the IndexTTS-1.5 geometry, synth.v1_5_config) v1_vocoder_full.npz from
the reference's own v1 `BigVGAN` (indextts/BigVGAN/models.py:129-249, which owns the ECAPA-TDNN speaker encoder,
ECAPA_TDNN.py:429-582) with the seeded weights of index-tts_b200/synth.py loaded into it, and v1_gpt_small.npz from its v1
UnifiedVoice.  Needs the reference checkout.
    python -m oracle.make_goldens_v1"""
import os

import numpy as np
import torch

from indextts_b200 import synth
from oracle import refimport, v1


def reference_module(h, w):
    refimport.setup()
    from indextts.BigVGAN.models import BigVGAN
    m = BigVGAN(refimport.AttrDict(dict(h)))
    m.remove_weight_norm()
    m.eval()
    sd = m.state_dict()
    unknown = [k for k in w if k not in sd]
    assert not unknown, unknown
    missing = [k for k in sd if k not in w and not k.endswith("num_batches_tracked")]
    assert not missing, missing
    m.load_state_dict(w, strict=False)
    return m


def main():
    h = synth.small_v1_config()
    seed = 4321
    w = synth.make_bigvgan_v1_weights(h, seed=seed)
    m = reference_module(h, w)
    g = torch.Generator().manual_seed(7)
    latent = torch.randn(1, 9, h["gpt_dim"], generator=g)
    mel_ref = torch.randn(1, 37, h["num_mels"], generator=g) * 1.5 - 4.0
    with torch.no_grad():
        spk_ref = m.speaker_encoder(mel_ref, torch.tensor([1.0]))
        wav_ref, _ = m(latent, mel_ref, torch.tensor([1.0]))
    spk = v1.ecapa_tdnn(w, mel_ref)
    wav = v1.bigvgan_v1_forward(h, w, latent, mel_ref)
    e1, e2 = float((spk - spk_ref).abs().max()), float((wav - wav_ref).abs().max())
    print(f"ECAPA-TDNN embedding max |diff| vs reference {e1:.2e} (std {float(spk_ref.std()):.2f}); wav max |diff| {e2:.2e} "
          f"(rms {float(wav_ref.pow(2).mean().sqrt()):.3f})")
    assert e1 < 1e-4 and e2 < 1e-5
    out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "v1_vocoder_small.npz")
    np.savez_compressed(out, seed=seed, latent=latent.numpy(), mel_ref=mel_ref.numpy(), spk=spk_ref.numpy(), wav=wav_ref.numpy())
    print("wrote", out)


FULL_SEED = 1515


def main_full():
    """The real v1.5 vocoder (1536 channels, x1024, conv_pre K = 7 * 1280) on T = 4 latents (4096 samples) and a 61-frame
    reference mel.  Only the inputs and outputs are stored: the weights are regenerated from the seed."""
    h = synth.v1_5_config()
    w = synth.make_bigvgan_v1_weights(h, seed=FULL_SEED, post_gain=synth.V1_5_POST_GAIN)
    m = reference_module(h, w)
    g = torch.Generator().manual_seed(8)
    latent = torch.randn(1, 4, h["gpt_dim"], generator=g)
    mel_ref = torch.randn(1, 61, h["num_mels"], generator=g) * 1.5 - 4.0
    with torch.no_grad():
        spk_ref = m.speaker_encoder(mel_ref, torch.tensor([1.0]))
        wav_ref, _ = m(latent, mel_ref, torch.tensor([1.0]))
    wav = v1.bigvgan_v1_forward(h, w, latent, mel_ref)
    e = float((wav - wav_ref).abs().max())
    print(f"v1.5 vocoder: wav [{tuple(wav_ref.shape)}] max |diff| vs reference {e:.2e} "
          f"(rms {float(wav_ref.pow(2).mean().sqrt()):.3f})")
    assert wav_ref.shape == (1, 1, 4 * 1024) and e < 1e-5
    out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "v1_vocoder_full.npz")
    np.savez_compressed(out, seed=FULL_SEED, latent=latent.numpy(), mel_ref=mel_ref.numpy(), spk=spk_ref.numpy(),
                        wav=wav_ref.numpy())
    print("wrote", out)


def main_gpt():
    """v1 GPT side against the reference's own v1 UnifiedVoice (kv_cache=False like infer.py:101)."""
    from oracle.gpt import GptOracle
    from oracle.validate_gpt_vs_hf import small_case
    cfg, _, _, text = small_case()
    ccfg = synth.small_v1_cond_cfg(cfg["model_dim"])
    seed = 2468
    w = synth.make_gpt_v1_weights(cfg, ccfg, seed=seed)
    g = refimport.gpt_module_v1(cfg, ccfg, w, kv_cache=False)
    gen = torch.Generator().manual_seed(3)
    mel = torch.randn(1, 100, 61, generator=gen) * 1.5 - 4.0
    with torch.no_grad():
        conds_ref = g.get_conditioning(mel, torch.tensor([61]))[0]
    conds = v1.get_conditioning_v1(w, ccfg, mel[0].t())
    e0 = float((conds - conds_ref).abs().max())
    print(f"get_conditioning (32 latents): max |diff| vs reference {e0:.2e} (std {float(conds_ref.std()):.2f})")
    assert conds.shape == conds_ref.shape == (32, cfg["model_dim"]) and e0 < 2e-4
    rec = {"logits": [], "prompt": None}
    orig_store = g.inference_model.store_mel_emb

    def store(emb):
        rec["prompt"] = emb.detach().clone()
        return orig_store(emb)
    g.inference_model.store_mel_emb = store
    g.inference_model.register_forward_hook(lambda mod, inp, out: rec["logits"].append(out.logits[:, -1, :].detach().float().clone()))
    n = 16
    with torch.no_grad():
        codes = g.inference_speech(mel, text[None], cond_mel_lengths=torch.tensor([61]), do_sample=False, num_beams=1, top_p=0.8,
                                   top_k=30, temperature=1.0, num_return_sequences=1, length_penalty=0.0,
                                   repetition_penalty=10.0, max_generate_length=n)
    codes = codes[0].numpy().astype(np.int32)
    logits = torch.cat(rec["logits"], 0).numpy()
    prompt = v1.prepare_inputs_v1(w, conds, text)
    assert prompt.shape == rec["prompt"][0].shape
    print("prepare_gpt_inputs (v1) max |diff|:", float((prompt - rec["prompt"][0]).abs().max()))
    assert (prompt - rec["prompt"][0]).abs().max() < 2e-4
    o_codes, o_logits = v1.generate_v1(GptOracle(cfg, w, bf16=False), rec["prompt"][0], n, 10.0, kv_cache=False)
    k = len(o_codes)
    print("reference v1 greedy (no KV cache):", codes.tolist())
    print("oracle    v1 greedy (no KV cache):", o_codes.tolist())
    assert codes[:k].tolist() == o_codes.tolist()
    err = float(np.abs(o_logits - logits[:k]).max())
    print(f"logits max |diff| {err:.2e}")
    assert err < 5e-4
    # latents for the vocoder (second forward, model.py:526-589)
    tk = codes[:k]
    tk = tk[tk != cfg["stop_mel_token"]]
    with torch.no_grad():
        lat_ref = g(mel, text[None], torch.tensor([text.shape[0]]), torch.from_numpy(tk.astype(np.int64))[None],
                    torch.tensor([tk.shape[0] * g.mel_length_compression]), cond_mel_lengths=torch.tensor([61]),
                    return_latent=True, clip_inputs=False)[0]
    lat = v1.latents_v1(GptOracle(cfg, w, bf16=False), conds_ref, text, tk)
    e2 = float((lat - lat_ref).abs().max())
    print(f"latents [{tuple(lat_ref.shape)}] max |diff| vs reference {e2:.2e}")
    assert lat.shape == lat_ref.shape and e2 < 5e-4
    out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "v1_gpt_small.npz")
    np.savez_compressed(out, seed=seed, mel=mel.numpy(), text=text.numpy(), conds=conds_ref.numpy(), codes=codes[:k],
                        logits=logits[:k].astype(np.float32), latents=lat_ref.numpy())
    print("wrote", out)


if __name__ == "__main__":
    main()
    main_full()
    main_gpt()
