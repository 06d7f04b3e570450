"""CPU restatement of the emotion-vector path of UnifiedVoice (SURVEY.md §8a row a7).

TEST INFRASTRUCTURE ONLY.  Pinned against the reference's own ConformerEncoder / PerceiverResampler
modules (importable from /root/reference) by oracle/make_goldens_emo.py.

Restated (reference file:line):
  merge_emovec / get_emovec / get_emo_conditioning   indextts/gpt/model_v2.py:827-838,588-593
  ConformerEncoder.forward (all-valid mask, trap P10) indextts/gpt/conformer_encoder.py:389-437
  Conv2dSubsampling2 + RelPositionalEncoding          gpt/conformer/subsampling.py:135-187, embedding.py:35-141
  ConformerEncoderLayer / ConvolutionModule / FFN     gpt/conformer_encoder.py:20-55,56-167,232-313
  RelPositionMultiHeadedAttention (no rel_shift)      gpt/conformer/attention.py:189-312
  PerceiverResampler / Attention / GEGLU / RMSNorm    gpt/perceiver.py:140-317
fp32 throughout (the reference runs this under bf16 autocast; the result is rounded to bf16 by the
caller before it enters the GPT prompt, see DESIGN.md §5).
"""
import math

import torch
import torch.nn.functional as F

from indextts_b200.synth import EMO_CFG, make_emo_weights, small_emo_cfg  # noqa: F401


def _ln(x, w, p, eps=1e-5):
    return F.layer_norm(x, (x.shape[-1],), w[p + ".weight"], w[p + ".bias"], eps)


def _lin(x, w, p):
    return F.linear(x, w[p + ".weight"], w.get(p + ".bias"))


def pos_table(T, d, device=None, dtype=None):
    """RelPositionalEncoding.pe (embedding.py:47-53), computed in fp32 on the CPU as the reference computes it, then moved
    to `device` / `dtype` (the values do not change)."""
    pe = torch.zeros(T, d)
    position = torch.arange(0, T).unsqueeze(1)
    div = torch.exp(torch.arange(0, d, 2) * -(math.log(10000.0) / d))
    pe[:, 0::2] = torch.sin(position * div)
    pe[:, 1::2] = torch.cos(position * div)
    return pe.to(device=device, dtype=dtype)


def rel_attention(q, k, v, pp, pos_bias_u, pos_bias_v, H):
    """RelPositionMultiHeadedAttention without rel_shift (attention.py:189-312) after its linears: q, k, v, pp (linear_pos of
    the table) [T, od] -> [T, od]."""
    T2, od = q.shape
    dk = od // H
    q = q.view(T2, H, dk)
    k, v, pp = (t.view(T2, H, dk).transpose(0, 1) for t in (k, v, pp))
    qu = (q + pos_bias_u).transpose(0, 1)
    qv = (q + pos_bias_v).transpose(0, 1)
    sc = (qu @ k.transpose(1, 2) + qv @ pp.transpose(1, 2)) / math.sqrt(dk)
    return (torch.softmax(sc, -1) @ v).transpose(0, 1).reshape(T2, od)


def latent_attention(q, kv, hh):
    """The perceiver's Attention (perceiver.py:224-274) after to_q / to_kv: q [nl, inner], kv [n, 2 inner] -> [nl, inner]."""
    nl, inner = q.shape
    dh = inner // hh
    k, v = kv.chunk(2, -1)
    qq = q.view(nl, hh, dh).transpose(0, 1)
    k = k.reshape(-1, hh, dh).transpose(0, 1)
    v = v.reshape(-1, hh, dh).transpose(0, 1)
    att = torch.softmax(qq @ k.transpose(1, 2) * dh ** -0.5, -1) @ v
    return att.transpose(0, 1).reshape(nl, inner)


@torch.no_grad()
def conformer_encode(w, c, x, prefix="emo_conditioning_encoder."):
    """x [T, idim] → [T', odim]  (ConformerEncoder with conv2d2 front-end, rel-pos attention)."""
    e = prefix
    od, H = c["odim"], c["heads"]
    y = F.relu(F.conv2d(x[None, None], w[e + "embed.conv.0.weight"], w[e + "embed.conv.0.bias"], stride=2))
    _, C, T2, Fs = y.shape
    y = y.transpose(1, 2).contiguous().view(1, T2, C * Fs)
    y = _lin(y, w, e + "embed.out.0")[0]
    y = y * math.sqrt(od)
    pe = pos_table(T2, od, device=x.device, dtype=x.dtype)
    for i in range(c["blocks"]):
        p = e + f"encoders.{i}."
        h = _ln(y, w, p + "norm_mha")
        a = rel_attention(_lin(h, w, p + "self_attn.linear_q"), _lin(h, w, p + "self_attn.linear_k"),
                          _lin(h, w, p + "self_attn.linear_v"), F.linear(pe, w[p + "self_attn.linear_pos.weight"]),
                          w[p + "self_attn.pos_bias_u"], w[p + "self_attn.pos_bias_v"], H)
        y = y + _lin(a, w, p + "self_attn.linear_out")
        h = _ln(y, w, p + "norm_conv").t()[None]
        h = F.glu(F.conv1d(h, w[p + "conv_module.pointwise_conv1.weight"], w[p + "conv_module.pointwise_conv1.bias"]), dim=1)
        h = F.conv1d(h, w[p + "conv_module.depthwise_conv.weight"], w[p + "conv_module.depthwise_conv.bias"],
                     padding=(c["cnn_kernel"] - 1) // 2, groups=od)
        h = F.silu(_ln(h[0].t(), w, p + "conv_module.norm")).t()[None]
        h = F.conv1d(h, w[p + "conv_module.pointwise_conv2.weight"], w[p + "conv_module.pointwise_conv2.bias"])[0].t()
        y = y + h
        h = _ln(y, w, p + "norm_ff")
        y = y + _lin(F.silu(_lin(h, w, p + "feed_forward.w_1")), w, p + "feed_forward.w_2")
        y = _ln(y, w, p + "norm_final")
    return _ln(y, w, e + "after_norm")


@torch.no_grad()
def perceiver_resample(w, c, ctx, prefix="emo_perceiver_encoder.", squeeze=True):
    """ctx [T', odim] → [p_dim] (1 latent; `squeeze=False`: [n_latents, p_dim], the v1 32-latent prompt)."""
    q = prefix
    hh = c["p_heads"]
    x = _lin(ctx, w, q + "proj_context")
    lat = w[q + "latents"].clone()
    for i in range(c["p_depth"]):
        a = q + f"layers.{i}.0."
        context = torch.cat([lat, x], 0)
        att = latent_attention(F.linear(lat, w[a + "to_q.weight"]), F.linear(context, w[a + "to_kv.weight"]), hh)
        lat = F.linear(att, w[a + "to_out.weight"]) + lat
        f = q + f"layers.{i}.1."
        h = _lin(lat, w, f + "0")
        xg, gate = h.chunk(2, -1)
        lat = _lin(F.gelu(gate) * xg, w, f + "2") + lat
    out = F.normalize(lat, dim=-1) * (c["p_dim"] ** 0.5) * w[q + "norm.gamma"]
    return out[0] if squeeze else out


@torch.no_grad()
def get_emovec(w, c, feats):
    """feats [T, idim] (w2v-BERT features) → emo_vec [model_dim]  (model_v2.py:827-831)."""
    lat = perceiver_resample(w, c, conformer_encode(w, c, feats))
    return _lin(_lin(lat[None], w, "emovec_layer"), w, "emo_layer")[0]


def merge_emovec(w, c, spk_feats, emo_feats, alpha=1.0):
    base = get_emovec(w, c, spk_feats)
    emo = get_emovec(w, c, emo_feats)
    return base + alpha * (emo - base)
