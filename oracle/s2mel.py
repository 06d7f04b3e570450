"""CPU restatement of the v2/v2.5 s2mel stage: semantic-codec decode → length regulator →
flow-matching CFM (DiT + WaveNet) Euler solver.

TEST INFRASTRUCTURE ONLY (see oracle/gpt.py header).  Pinned against the reference's own
modules (EnhancedCodec, InterpolateRegulator, CFM/DiT/WN imported from /root/reference) by
oracle/make_goldens_s2mel.py; the reference tests pin nothing here (SURVEY.md §8c).

Restated (reference file:line):
  EnhancedCodec.decode               indextts/codec/models.py:205-231
    FVQ vq2emb                       codec/amphion_codec/quantize/factorized_vector_quantize.py:96-127
    VocosBackbone / ConvNeXtBlock    codec/kmeans/vocos.py:468-527,719-783
  InterpolateRegulator.forward       s2mel/modules/length_regulator.py:90-141
  BASECFM.inference / solve_euler    s2mel/modules/flow_matching.py:30-115
  DiT.forward                        s2mel/modules/diffusion_transformer.py:186-257
  TimestepEmbedder / FinalLayer      diffusion_transformer.py:19-101
  Transformer / Block / Attention / FeedForward / AdaptiveLayerNorm / RMSNorm / rotary
                                     s2mel/modules/gpt_fast/model.py:20-39,121-360
  WN (+ SConv1d reflect padding)     s2mel/modules/wavenet.py:103-166, encodec.py:192-229

All fp32 (the reference disables autocast for this stage: infer_v2_5.py:827-828, trap P5).
Weights: dict keyed by the reference state-dict names with weight norm already folded
(`fold_weight_norm`), e.g. "cfm.estimator.wavenet.in_layers.0.conv.conv.weight".
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from indextts_b200.synth import (CODEC_CFG, S2MEL_CFG, make_codec_weights, make_s2mel_weights,  # noqa: F401,E402
                                  small_codec_cfg, small_s2mel_cfg)







def fold_weight_norm(sd):
    """torch.nn.utils.weight_norm (dim=0): w = g * v / ||v||, norm over all dims but 0."""
    out = {}
    for k, v in sd.items():
        if k.endswith("weight_g"):
            base = k[: -len("weight_g")]
            vv = sd[base + "weight_v"]
            norm = vv.reshape(vv.shape[0], -1).norm(dim=1).reshape(-1, *([1] * (vv.dim() - 1)))
            out[base + "weight"] = v * vv / norm
        elif k.endswith("weight_v"):
            continue
        else:
            out[k] = v
    return out


# ------------------------------------------------------------------------------ weights --




# -------------------------------------------------------------------------------- codec --
@torch.no_grad()
def codec_decode(w, codes):
    """codes [B, n] int64 → S_infer [B, 2n, hidden] (codec/models.py:205-231)."""
    q = "quantizer.quantizers.0."
    emb = F.embedding(codes, w[q + "codebook.weight"]).transpose(1, 2)          # [B, 8, n]
    x = F.conv1d(emb, w[q + "out_project.weight"], w[q + "out_project.bias"])   # [B, H, n]
    b = "decoder.0."
    x = F.conv1d(x, w[b + "embed.weight"], w[b + "embed.bias"], padding=3)
    Vd = x.shape[1]
    x = F.layer_norm(x.transpose(1, 2), (Vd,), w[b + "norm.weight"], w[b + "norm.bias"], 1e-6).transpose(1, 2)
    l = 0
    while (b + f"convnext.{l}.dwconv.weight") in w:
        p = b + f"convnext.{l}."
        r = x
        y = F.conv1d(x, w[p + "dwconv.weight"], w[p + "dwconv.bias"], padding=3, groups=Vd).transpose(1, 2)
        y = F.layer_norm(y, (Vd,), w[p + "norm.weight"], w[p + "norm.bias"], 1e-6)
        y = F.gelu(F.linear(y, w[p + "pwconv1.weight"], w[p + "pwconv1.bias"]))
        y = F.linear(y, w[p + "pwconv2.weight"], w[p + "pwconv2.bias"]) * w[p + "gamma"]
        x = r + y.transpose(1, 2)
        l += 1
    x = F.layer_norm(x.transpose(1, 2), (Vd,), w[b + "final_layer_norm.weight"], w[b + "final_layer_norm.bias"], 1e-6)
    x = F.linear(x, w["decoder.1.weight"], w["decoder.1.bias"])                 # [B, n, H]
    x = F.interpolate(x.transpose(1, 2), scale_factor=2, mode="nearest")
    return F.conv1d(x, w["up.weight"], w["up.bias"], padding=1).transpose(1, 2)


# --------------------------------------------------------------------- length regulator --
@torch.no_grad()
def length_regulate(w, x, ylen, n_convs=4):
    """x [B, 2n, in] → [B, ylen, C] (length_regulator.py:90-141; continuous input, no f0)."""
    r = "length_regulator."
    x = F.linear(x, w[r + "content_in_proj.weight"], w[r + "content_in_proj.bias"])
    x = F.interpolate(x.transpose(1, 2).contiguous(), size=int(ylen), mode="nearest")
    C = x.shape[1]
    for i in range(n_convs):
        x = F.conv1d(x, w[r + f"model.{3 * i}.weight"], w[r + f"model.{3 * i}.bias"], padding=1)
        x = F.group_norm(x, 1, w[r + f"model.{3 * i + 1}.weight"], w[r + f"model.{3 * i + 1}.bias"], 1e-5)
        x = F.mish(x)
    k = 3 * n_convs
    x = F.conv1d(x, w[r + f"model.{k}.weight"], w[r + f"model.{k}.bias"])
    return x.transpose(1, 2).contiguous()   # mask is all-ones for a single full-length sequence


# ---------------------------------------------------------------------------------- DiT --
def _t_embed(w, pfx, t):
    args = 1000 * t[:, None].float() * w[pfx + ".freqs"][None]
    emb = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    h = F.silu(F.linear(emb, w[pfx + ".mlp.0.weight"], w[pfx + ".mlp.0.bias"]))
    return F.linear(h, w[pfx + ".mlp.2.weight"], w[pfx + ".mlp.2.bias"])


def _rms(x, weight, eps=1e-5):
    return x * torch.rsqrt(torch.mean(x * x, dim=-1, keepdim=True) + eps) * weight


def _adaln(w, pfx, x, c):
    wb = F.linear(c, w[pfx + ".project_layer.weight"], w[pfx + ".project_layer.bias"])
    d = x.shape[-1]
    return wb[..., :d] * _rms(x, w[pfx + ".norm.weight"]) + wb[..., d:]


def _rope(x, hd):
    """x [B,T,H,hd]; interleaved pairs, base 1e4 (gpt_fast/model.py:336-360)."""
    T = x.shape[1]
    freqs = 1.0 / (10000 ** (torch.arange(0, hd, 2)[: hd // 2].float() / hd))
    ang = torch.outer(torch.arange(T).float(), freqs)
    cos, sin = torch.cos(ang)[None, :, None, :], torch.sin(ang)[None, :, None, :]
    xs = x.float().reshape(*x.shape[:-1], -1, 2)
    o = torch.stack([xs[..., 0] * cos - xs[..., 1] * sin, xs[..., 1] * cos + xs[..., 0] * sin], -1)
    return o.flatten(3)


def pad1d_reflect(x, left, right):
    """encodec.py pad1d(mode='reflect'): an input no longer than the larger pad is zero-extended to max(left, right) + 1
    frames, reflected, and the extension cropped off again (F.pad alone refuses such short inputs)."""
    extra = max(max(left, right) + 1 - x.shape[-1], 0)
    x = F.pad(x, (0, extra))
    y = F.pad(x, (left, right), mode="reflect")
    return y[..., :y.shape[-1] - extra]


def _reflect_conv(x, weight, bias, k):
    if k > 1:
        pt = k - 1
        x = pad1d_reflect(x, pt - pt // 2, pt // 2)             # encodec.py:214-229 (stride 1)
    return F.conv1d(x, weight, bias)


@torch.no_grad()
def dit_forward(w, c, x, prompt_x, x_lens, t, style, cond):
    """DiT.forward (diffusion_transformer.py:186-257). x,prompt_x [B,80,T]; cond [B,T,content]."""
    e = "cfm.estimator."
    H, nh, Dn, WH, NL = c["hidden"], c["heads"], c["depth"], c["wn_hidden"], c["wn_layers"]
    hd = H // nh
    B, _, T = x.shape
    t1 = _t_embed(w, e + "t_embedder", t)
    cond = F.linear(cond, w[e + "cond_projection.weight"], w[e + "cond_projection.bias"])
    xt, pt = x.transpose(1, 2), prompt_x.transpose(1, 2)
    x_in = torch.cat([xt, pt, cond, style[:, None, :].repeat(1, T, 1)], dim=-1)
    h = F.linear(x_in, w[e + "cond_x_merge_linear.weight"], w[e + "cond_x_merge_linear.bias"])
    key_mask = (torch.arange(T)[None, :] < x_lens[:, None])          # [B,T]
    attn_mask = key_mask[:, None, None, :].expand(B, 1, T, T)
    cvec = t1[:, None, :]
    skips = []
    for l in range(Dn):
        p = e + f"transformer.layers.{l}."
        if l > Dn // 2:
            h = F.linear(torch.cat([h, skips.pop(-1)], dim=-1), w[p + "skip_in_linear.weight"], w[p + "skip_in_linear.bias"])
        a = _adaln(w, p + "attention_norm", h, cvec)
        qkv = F.linear(a, w[p + "attention.wqkv.weight"])
        q, k, v = qkv.split([H, H, H], dim=-1)
        q = _rope(q.view(B, T, nh, hd), hd).transpose(1, 2)
        k = _rope(k.view(B, T, nh, hd), hd).transpose(1, 2)
        v = v.view(B, T, nh, hd).transpose(1, 2)
        y = F.scaled_dot_product_attention(q, k, v, attn_mask=attn_mask)
        y = y.transpose(1, 2).contiguous().view(B, T, H)
        h = h + F.linear(y, w[p + "attention.wo.weight"])
        f = _adaln(w, p + "ffn_norm", h, cvec)
        f = F.linear(F.silu(F.linear(f, w[p + "feed_forward.w1.weight"])) * F.linear(f, w[p + "feed_forward.w3.weight"]),
                     w[p + "feed_forward.w2.weight"])
        h = h + f
        if l < Dn // 2:
            skips.append(h)
    h = _adaln(w, e + "transformer.norm", h, cvec)
    x_res = F.linear(torch.cat([h, xt], dim=-1), w[e + "skip_linear.weight"], w[e + "skip_linear.bias"])
    y = F.linear(x_res, w[e + "conv1.weight"], w[e + "conv1.bias"]).transpose(1, 2)        # [B,WH,T]
    t2 = _t_embed(w, e + "t_embedder2", t)
    mask = key_mask[:, None, :].float()
    # WN (wavenet.py:132-166)
    g = F.conv1d(t2[:, :, None], w[e + "wavenet.cond_layer.conv.conv.weight"], w[e + "wavenet.cond_layer.conv.conv.bias"])
    out = torch.zeros_like(y)
    K = c["wn_kernel"]
    for i in range(NL):
        xin = _reflect_conv(y, w[e + f"wavenet.in_layers.{i}.conv.conv.weight"], w[e + f"wavenet.in_layers.{i}.conv.conv.bias"], K)
        gl = g[:, i * 2 * WH:(i + 1) * 2 * WH, :]
        ia = xin + gl
        acts = torch.tanh(ia[:, :WH]) * torch.sigmoid(ia[:, WH:])
        rs = F.conv1d(acts, w[e + f"wavenet.res_skip_layers.{i}.conv.conv.weight"], w[e + f"wavenet.res_skip_layers.{i}.conv.conv.bias"])
        if i < NL - 1:
            y = (y + rs[:, :WH]) * mask
            out = out + rs[:, WH:]
        else:
            out = out + rs
    wn_out = (out * mask).transpose(1, 2) + F.linear(x_res, w[e + "res_projection.weight"], w[e + "res_projection.bias"])
    # FinalLayer (diffusion_transformer.py:84-101)
    mod = F.linear(F.silu(t1), w[e + "final_layer.adaLN_modulation.1.weight"], w[e + "final_layer.adaLN_modulation.1.bias"])
    shift, scale = mod.chunk(2, dim=1)
    z = F.layer_norm(wn_out, (WH,), None, None, 1e-6) * (1 + scale[:, None]) + shift[:, None]
    z = F.linear(z, w[e + "final_layer.linear.weight"], w[e + "final_layer.linear.bias"]).transpose(1, 2)
    return F.conv1d(z, w[e + "conv2.weight"], w[e + "conv2.bias"])


@torch.no_grad()
def cfm_inference(w, c, mu, x_lens, prompt, style, z, n_timesteps=25, inference_cfg_rate=0.7):
    """BASECFM.inference with the noise z supplied by the caller (flow_matching.py:30-115, P6)."""
    x = z.clone()
    t_span = torch.linspace(0, 1, n_timesteps + 1)
    t = t_span[0]
    P = prompt.size(-1)
    prompt_x = torch.zeros_like(x)
    prompt_x[..., :P] = prompt[..., :P]
    x[..., :P] = 0
    for step in range(1, len(t_span)):
        dt = t_span[step] - t_span[step - 1]
        if inference_cfg_rate > 0:
            sx = torch.cat([x, x], 0)
            sp = torch.cat([prompt_x, torch.zeros_like(prompt_x)], 0)
            ss = torch.cat([style, torch.zeros_like(style)], 0)
            sm = torch.cat([mu, torch.zeros_like(mu)], 0)
            st = torch.stack([t, t])
            d = dit_forward(w, c, sx, sp, torch.cat([x_lens, x_lens]), st, ss, sm)
            dphi, cfg_dphi = d.chunk(2, dim=0)
            dphi = (1.0 + inference_cfg_rate) * dphi - inference_cfg_rate * cfg_dphi
        else:
            dphi = dit_forward(w, c, x, prompt_x, x_lens, t[None], style, mu)
        x = x + dt * dphi
        t = t + dt
        x[:, :, :P] = 0
    return x
