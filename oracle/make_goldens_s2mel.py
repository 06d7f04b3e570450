"""Mint s2mel / codec golden vectors from the REFERENCE modules (build container only) and pin
the restatement oracle/s2mel.py against them.

    python -m oracle.make_goldens_s2mel

Writes tests/golden/s2mel_small.npz (reduced dims: codec decode, length regulator, one DiT
evaluation, full 6-step CFM solve) and tests/golden/s2mel_full_dit.npz (the [ASSUMED] full
IndexTTS-2.5 dims, one DiT evaluation at T=96 and a codec/length-regulator pass).  Weights are
regenerated from seeds by oracle.s2mel.make_*_weights on the GPU box.

    python -m oracle.make_goldens_s2mel short

writes only tests/golden/s2mel_short.npz: the reference's reflect-padded SConv1d (encodec.py pad1d) at 1, 2 and 3 frames
and one small-dims DiT evaluation at T = 1 and 2, the lengths where pad1d zero-extends before it reflects."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import refimport  # noqa: E402
from oracle.s2mel import (CODEC_CFG, S2MEL_CFG, _reflect_conv, cfm_inference, codec_decode, dit_forward,  # noqa: E402
                          fold_weight_norm, length_regulate, make_codec_weights, make_s2mel_weights, small_codec_cfg,
                          small_s2mel_cfg)

GOLD = os.path.join(ROOT, "tests", "golden")


def ref_s2mel(c, w):
    args = refimport.s2mel_args(hidden=c["hidden"], heads=c["heads"], depth=c["depth"], wn_hidden=c["wn_hidden"],
                                wn_layers=c["wn_layers"], content_dim=c["content_dim"], lr_in=c["lr_in"],
                                style_dim=c["style_dim"])
    m = refimport.s2mel_module(args)
    sd = {"models." + k: v for k, v in w.items()}
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    assert not missing, missing
    return m


def ref_codec(c, w):
    m = refimport.codec_module(**c)
    missing, unexpected = m.load_state_dict(w, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    return m


def inputs(c, T, P, seed):
    g = torch.Generator().manual_seed(seed)
    mu = torch.randn(1, T, c["content_dim"], generator=g)
    prompt = torch.randn(1, 80, P, generator=g) * 1.5 - 4.0
    style = torch.randn(1, c["style_dim"], generator=g)
    z = torch.randn(1, 80, T, generator=g)
    return mu, prompt, style, z


@torch.no_grad()
def main():
    torch.set_num_threads(8)
    out = {}
    # ------------------------------------------------------------------ small dims ----
    c, cc = small_s2mel_cfg(), small_codec_cfg()
    w, wc = make_s2mel_weights(c, seed=1234), make_codec_weights(cc, seed=4321)
    wf, wcf = fold_weight_norm(w), fold_weight_norm(wc)
    m, mc = ref_s2mel(c, w), ref_codec(cc, wc)
    g = torch.Generator().manual_seed(5)
    codes = torch.randint(0, cc["codebook_size"], (1, 23), generator=g)
    S_ref = mc.decode(codes)
    S_or = codec_decode(wcf, codes)
    print("codec decode: max|ref-oracle| =", (S_ref - S_or).abs().max().item(), tuple(S_ref.shape))
    assert (S_ref - S_or).abs().max() < 1e-5
    ylen = int(S_ref.shape[1] * 1.72)
    lr_in = torch.randn(1, 46, c["lr_in"], generator=g)
    cond_ref = m.models["length_regulator"](lr_in, ylens=torch.LongTensor([ylen]), n_quantizers=3, f0=None)[0]
    cond_or = length_regulate(wf, lr_in, ylen)
    print("length regulator: max|ref-oracle| =", (cond_ref - cond_or).abs().max().item(), tuple(cond_ref.shape))
    assert (cond_ref - cond_or).abs().max() < 1e-5
    T, P = 61, 17
    mu, prompt, style, z = inputs(c, T, P, 7)
    x_lens = torch.LongTensor([T])
    est = m.models["cfm"].estimator
    prompt_x = torch.zeros(1, 80, T)
    prompt_x[..., :P] = prompt
    tt = torch.tensor([0.32])
    d_ref = est(z, prompt_x, x_lens, tt, style, mu)
    d_or = dit_forward(wf, c, z, prompt_x, x_lens, tt, style, mu)
    print("DiT forward: max|ref-oracle| =", (d_ref - d_or).abs().max().item(), "out std", d_ref.std().item())
    assert (d_ref - d_or).abs().max() < 2e-4
    nst = 6
    cfm = m.models["cfm"]
    mel_ref = cfm.solve_euler(z.clone(), x_lens, prompt, mu.clone(), style, None, torch.linspace(0, 1, nst + 1), 0.7)
    mel_or = cfm_inference(wf, c, mu, x_lens, prompt, style, z, nst, 0.7)
    print("CFM 6 steps: max|ref-oracle| =", (mel_ref - mel_or).abs().max().item(), "mel std", mel_ref.std().item())
    assert (mel_ref - mel_or).abs().max() < 1e-3
    np.savez_compressed(os.path.join(GOLD, "s2mel_small.npz"), codes=codes.numpy(), S_infer=S_ref.numpy(),
                        lr_in=lr_in.numpy(), ylen=ylen, cond=cond_ref.numpy(), mu=mu.numpy(), prompt=prompt.numpy(),
                        style=style.numpy(), z=z.numpy(), t=tt.numpy(), dit=d_ref.numpy(), n_steps=nst,
                        mel=mel_ref.numpy(), seed_s2mel=1234, seed_codec=4321)
    # ------------------------------------------------------------------- full dims ----
    c, cc = dict(S2MEL_CFG), dict(CODEC_CFG)
    w, wc = make_s2mel_weights(c, seed=1234), make_codec_weights(cc, seed=4321)
    wf, wcf = fold_weight_norm(w), fold_weight_norm(wc)
    m, mc = ref_s2mel(c, w), ref_codec(cc, wc)
    assert sum(p.numel() for p in m.models["cfm"].parameters()) == 98187344          # SURVEY A.2
    assert sum(p.numel() for p in m.models["length_regulator"].parameters()) == 4988416
    assert sum(p.numel() for p in mc.parameters()) == 50583312
    codes = torch.randint(0, 8192, (1, 16), generator=g)
    S_ref = mc.decode(codes)
    assert (S_ref - codec_decode(wcf, codes)).abs().max() < 1e-4
    ylen = int(S_ref.shape[1] * 1.72)
    cond_ref = m.models["length_regulator"](S_ref, ylens=torch.LongTensor([ylen]), n_quantizers=3, f0=None)[0]
    assert (cond_ref - length_regulate(wf, S_ref, ylen)).abs().max() < 1e-4
    T, P = 96, 41
    mu, prompt, style, z = inputs(c, T, P, 9)
    x_lens = torch.LongTensor([T])
    prompt_x = torch.zeros(1, 80, T)
    prompt_x[..., :P] = prompt
    tt = torch.tensor([0.6])
    d_ref = m.models["cfm"].estimator(z, prompt_x, x_lens, tt, style, mu)
    d_or = dit_forward(wf, c, z, prompt_x, x_lens, tt, style, mu)
    print("full DiT forward: max|ref-oracle| =", (d_ref - d_or).abs().max().item(), "out std", d_ref.std().item())
    assert (d_ref - d_or).abs().max() < 5e-4
    np.savez_compressed(os.path.join(GOLD, "s2mel_full_dit.npz"), codes=codes.numpy(), S_infer=S_ref.numpy(),
                        ylen=ylen, cond=cond_ref.numpy(), mu=mu.numpy(), prompt=prompt.numpy(), style=style.numpy(),
                        z=z.numpy(), t=tt.numpy(), dit=d_ref.numpy(), seed_s2mel=1234, seed_codec=4321)
    print("wrote s2mel goldens")
    short_goldens()


@torch.no_grad()
def short_goldens():
    refimport.setup()
    from indextts.s2mel.modules.encodec import SConv1d
    out = {}
    g = torch.Generator().manual_seed(21)
    conv = SConv1d(6, 5, kernel_size=5, pad_mode="reflect")     # the WaveNet in-layer's padding, (2, 2)
    with torch.no_grad():
        for p in conv.parameters():
            p.copy_(torch.randn(p.shape, generator=g))
    out["sconv_weight"], out["sconv_bias"] = conv.conv.conv.weight.numpy(), conv.conv.conv.bias.numpy()
    for T in (1, 2, 3):
        x = torch.randn(1, 6, T, generator=g)
        y = conv(x)
        assert (y - _reflect_conv(x, conv.conv.conv.weight, conv.conv.conv.bias, 5)).abs().max() < 1e-5
        out[f"sconv_x{T}"], out[f"sconv_y{T}"] = x.numpy(), y.numpy()
    c = small_s2mel_cfg()
    w = make_s2mel_weights(c, seed=1234)
    est = ref_s2mel(c, w).models["cfm"].estimator
    for T in (1, 2):
        mu, _, style, z = inputs(c, T, 0, 30 + T)
        px = torch.zeros(1, 80, T)
        tt = torch.tensor([0.45])
        d_ref = est(z, px, torch.LongTensor([T]), tt, style, mu)
        d_or = dit_forward(fold_weight_norm(w), c, z, px, torch.LongTensor([T]), tt, style, mu)
        print(f"DiT forward T={T}: max|ref-oracle| =", (d_ref - d_or).abs().max().item())
        assert (d_ref - d_or).abs().max() < 2e-4
        out.update({f"dit{T}_mu": mu.numpy(), f"dit{T}_style": style.numpy(), f"dit{T}_z": z.numpy(), f"dit{T}_t": tt.numpy(),
                    f"dit{T}": d_ref.numpy()})
    np.savez_compressed(os.path.join(GOLD, "s2mel_short.npz"), seed_s2mel=1234, **out)
    print("wrote s2mel_short.npz")


if __name__ == "__main__":
    if sys.argv[1:] == ["short"]:
        short_goldens()
    else:
        main()
