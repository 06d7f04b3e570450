"""Plain-torch restatement of IndexTTS2.get_emb (infer_v2_5.py:281-290) over transformers' Wav2Vec2BertModel
(models/wav2vec2_bert/modeling_wav2vec2_bert.py, position_embeddings_type "relative_key", eval mode), without importing
transformers, so GPU tests can run it.

    get_emb(sd, cfg, feats, mask) = (hidden_states[cfg["layers"]] - semantic_mean) / semantic_std

sd holds the HF state-dict names (feature_projection.*, encoder.layers.N.*) plus semantic_mean / semantic_std.
`make_weights(cfg, seed)` draws a seeded state dict in a fixed order: the goldens store only the seed.
"""
import math

import torch
import torch.nn.functional as F

FULL = dict(feat_dim=160, hidden=1024, heads=16, ffn=4096, layers=17, conv_kernel=31, left_max=64, right_max=8, eps=1e-5)
SMALL = dict(feat_dim=160, hidden=128, heads=2, ffn=256, layers=2, conv_kernel=31, left_max=64, right_max=8, eps=1e-5)


def layer_names(i):
    p = f"encoder.layers.{i}."
    names = []
    for ln in ("ffn1_layer_norm", "self_attn_layer_norm", "conv_module.layer_norm", "conv_module.depthwise_layer_norm",
               "ffn2_layer_norm", "final_layer_norm"):
        names += [p + ln + ".weight", p + ln + ".bias"]
    for lin in ("ffn1.intermediate_dense", "ffn1.output_dense", "ffn2.intermediate_dense", "ffn2.output_dense",
                "self_attn.linear_q", "self_attn.linear_k", "self_attn.linear_v", "self_attn.linear_out"):
        names += [p + lin + ".weight", p + lin + ".bias"]
    names += [p + "self_attn.distance_embedding.weight", p + "conv_module.pointwise_conv1.weight",
              p + "conv_module.depthwise_conv.weight", p + "conv_module.pointwise_conv2.weight"]
    return names


def shapes(cfg, n_layers):
    """name -> shape of every tensor get_emb reads, for n_layers encoder layers."""
    C, Fd, Ff, K = cfg["hidden"], cfg["feat_dim"], cfg["ffn"], cfg["conv_kernel"]
    out = {"feature_projection.layer_norm.weight": (Fd,), "feature_projection.layer_norm.bias": (Fd,),
           "feature_projection.projection.weight": (C, Fd), "feature_projection.projection.bias": (C,)}
    for i in range(n_layers):
        for n in layer_names(i):
            leaf = n.split(".", 3)[3]
            if leaf.endswith("layer_norm.weight") or leaf.endswith("layer_norm.bias"):
                out[n] = (C,)
            elif "intermediate_dense" in leaf:
                out[n] = (Ff, C) if leaf.endswith("weight") else (Ff,)
            elif "output_dense" in leaf:
                out[n] = (C, Ff) if leaf.endswith("weight") else (C,)
            elif "linear_" in leaf:
                out[n] = (C, C) if leaf.endswith("weight") else (C,)
            elif "distance_embedding" in leaf:
                out[n] = (cfg["left_max"] + cfg["right_max"] + 1, C // cfg["heads"])
            elif "pointwise_conv1" in leaf:
                out[n] = (2 * C, C, 1)
            elif "depthwise_conv" in leaf:
                out[n] = (C, 1, K)
            elif "pointwise_conv2" in leaf:
                out[n] = (C, C, 1)
    out["semantic_mean"] = (C,)
    out["semantic_std"] = (C,)
    return out


def make_weights(cfg, seed, n_layers=None):
    """Seeded state dict (fp32, CPU) in a fixed draw order.  Linear / conv weights ~ N(0, 1/fan_in), biases N(0, 0.02^2),
    LayerNorm weights 1 + N(0, 0.1^2) and biases N(0, 0.1^2), distance embeddings N(0, 1), the normalisation statistics
    mean ~ N(0, 0.1^2), std ~ U(0.5, 1.5)."""
    g = torch.Generator().manual_seed(int(seed))
    sd = {}
    for n, shp in shapes(cfg, cfg["layers"] if n_layers is None else n_layers).items():
        if n == "semantic_std":
            sd[n] = 0.5 + torch.rand(shp, generator=g)
        elif n == "semantic_mean":
            sd[n] = 0.1 * torch.randn(shp, generator=g)
        elif "layer_norm" in n:
            sd[n] = (1.0 if n.endswith("weight") else 0.0) + 0.1 * torch.randn(shp, generator=g)
        elif "distance_embedding" in n:
            sd[n] = torch.randn(shp, generator=g)
        elif n.endswith("bias"):
            sd[n] = 0.02 * torch.randn(shp, generator=g)
        else:
            fan_in = shp[1] * (shp[2] if len(shp) == 3 else 1)
            if "depthwise" in n:
                fan_in = shp[2]
            sd[n] = torch.randn(shp, generator=g) / math.sqrt(fan_in)
    return sd


def _ln(x, sd, name, eps):
    return F.layer_norm(x, x.shape[-1:], sd[name + ".weight"], sd[name + ".bias"], eps)


def _lin(x, sd, name):
    return F.linear(x, sd[name + ".weight"], sd.get(name + ".bias"))


def get_emb(sd, cfg, feats, mask):
    """feats [B, T, feat_dim], mask [B, T] (0/1) -> [B, T, hidden], in the dtype / device of feats."""
    eps, C, H = cfg["eps"], cfg["hidden"], cfg["heads"]
    L, R, K = cfg["left_max"], cfg["right_max"], cfg["conv_kernel"]
    dt, dev = feats.dtype, feats.device
    sd = {k: v.to(dev, dt) for k, v in sd.items()}
    B, T, _ = feats.shape
    keep = mask.to(dev).bool()
    x = _lin(_ln(feats, sd, "feature_projection.layer_norm", eps), sd, "feature_projection.projection")
    x = x.masked_fill(~keep[..., None], 0.0)
    bias = (1.0 - keep[:, None, None, :].to(dt)) * torch.finfo(dt).min
    pos = torch.arange(T, device=dev)
    dist = torch.clamp(pos[None, :] - pos[:, None], -L, R) + L

    def ffn(x, p):
        h = F.silu(_lin(_ln(x, sd, p + "_layer_norm", eps), sd, p + ".intermediate_dense"))
        return _lin(h, sd, p + ".output_dense")

    for i in range(cfg["layers"]):
        p = f"encoder.layers.{i}."
        x = 0.5 * ffn(x, p + "ffn1") + x
        h = _ln(x, sd, p + "self_attn_layer_norm", eps)
        q, k, v = (_lin(h, sd, p + "self_attn.linear_" + n).view(B, T, H, -1).transpose(1, 2) for n in "qkv")
        d = q.shape[-1]
        E = sd[p + "self_attn.distance_embedding.weight"][dist]                         # [T, T, d]
        s = (q @ k.transpose(-2, -1) + torch.einsum("bhld,lrd->bhlr", q, E)) / math.sqrt(d) + bias
        a = (torch.softmax(s, dim=-1) @ v).transpose(1, 2).reshape(B, T, C)
        x = _lin(a, sd, p + "self_attn.linear_out") + x
        h = _ln(x, sd, p + "conv_module.layer_norm", eps).masked_fill(~keep[..., None], 0.0)
        h = F.glu(F.conv1d(h.transpose(1, 2), sd[p + "conv_module.pointwise_conv1.weight"]), dim=1)
        h = F.conv1d(F.pad(h, (K - 1, 0)), sd[p + "conv_module.depthwise_conv.weight"], groups=C)
        h = F.silu(_ln(h.transpose(1, 2), sd, p + "conv_module.depthwise_layer_norm", eps))
        h = F.conv1d(h.transpose(1, 2), sd[p + "conv_module.pointwise_conv2.weight"]).transpose(1, 2)
        x = x + h
        x = 0.5 * ffn(x, p + "ffn2") + x
        x = _ln(x, sd, p + "final_layer_norm", eps)
    return (x - sd["semantic_mean"]) / sd["semantic_std"]
