"""Pin oracle/emo.py against the reference ConformerEncoder / PerceiverResampler modules and mint
tests/golden/emo_small.npz, emo_full.npz and emo_full_t750.npz (build container only).   python -m oracle.make_goldens_emo

emo_full_t750 is a 15 s prompt (T = 750 feature rows, T' = 374 after the subsampling).  It stores the reference's outputs
(ctx, latent, emovec) and the seed of the features, not the features: the test re-draws them from the seed."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import refimport  # noqa: E402
from oracle.emo import EMO_CFG, conformer_encode, get_emovec, make_emo_weights, perceiver_resample, small_emo_cfg  # noqa: E402


@torch.no_grad()
def check(c, T, seed, name, store_feats=True):
    refimport.setup()
    from indextts.gpt.conformer_encoder import ConformerEncoder
    from indextts.gpt.perceiver import PerceiverResampler
    w = make_emo_weights(c, seed=777)
    enc = ConformerEncoder(input_size=c["idim"], output_size=c["odim"], linear_units=c["linear_units"],
                           attention_heads=c["heads"], num_blocks=c["blocks"], input_layer="conv2d2")
    per = PerceiverResampler(c["p_dim"], dim_context=c["odim"], ff_mult=c["p_ff_mult"], heads=c["p_heads"], num_latents=1)
    sd_e = {k[len("emo_conditioning_encoder."):]: v for k, v in w.items() if k.startswith("emo_conditioning_encoder.")}
    miss, unexp = enc.load_state_dict(sd_e, strict=False)
    assert not unexp and all("pos_enc.pe" in m for m in miss), (miss, unexp)
    sd_p = {k[len("emo_perceiver_encoder."):]: v for k, v in w.items() if k.startswith("emo_perceiver_encoder.")}
    miss, unexp = per.load_state_dict(sd_p, strict=False)
    assert not unexp and not miss, (miss, unexp)
    enc.eval(); per.eval()
    g = torch.Generator().manual_seed(seed)
    feats = torch.randn(T, c["idim"], generator=g)
    # the reference call chain incl. its length quirk (trap P10): lengths = feature dim, mask all-valid
    ctx_ref, mask = enc(feats[None], torch.tensor([c["idim"]]))
    assert bool(mask.all())
    conds_mask = torch.nn.functional.pad(mask.squeeze(1), (1, 0), value=True)
    lat_ref = per(ctx_ref, conds_mask)[0, 0]
    ctx = conformer_encode(w, c, feats)
    lat = perceiver_resample(w, c, ctx)
    print(f"{name}: conformer max|ref-oracle| {float((ctx_ref[0] - ctx).abs().max()):.2e} (T'={ctx.shape[0]}), "
          f"perceiver {float((lat_ref - lat).abs().max()):.2e}")
    assert (ctx_ref[0] - ctx).abs().max() < 2e-4 and (lat_ref - lat).abs().max() < 2e-4
    ev = get_emovec(w, c, feats)
    ev_ref = torch.nn.functional.linear(torch.nn.functional.linear(lat_ref[None], w["emovec_layer.weight"], w["emovec_layer.bias"]),
                                        w["emo_layer.weight"], w["emo_layer.bias"])[0]
    out = dict(ctx=ctx_ref[0].numpy(), latent=lat_ref.numpy(), emovec=ev_ref.numpy(), seed=777)
    if store_feats:
        out.update(feats=feats.numpy())
    else:
        out.update(feats_seed=seed, T=T)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", name + ".npz"), **out)
    assert (ev - ev_ref).abs().max() < 5e-4


if __name__ == "__main__":
    torch.set_num_threads(8)
    check(small_emo_cfg(), 37, 1, "emo_small")
    check(dict(EMO_CFG), 60, 2, "emo_full")
    check(dict(EMO_CFG), 750, 3, "emo_full_t750", store_feats=False)
    print("wrote emo goldens")
