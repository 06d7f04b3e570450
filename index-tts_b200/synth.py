"""Deterministic synthetic weights and inputs at the reference shapes (there are no checkpoints
offline: bench.py, the tests and the oracle all regenerate the same tensors from a seed with the
torch CPU generator).  State-dict names follow the reference modules.  No compute path here."""
import math

import numpy as np
import torch


def r16(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.bfloat16).to(torch.float32)



def gpt_config(layers=24, model_dim=1280, heads=20, number_mel_codes=8194, start_mel_token=8192,
               stop_mel_token=8193, max_mel_tokens=1815, max_text_tokens=600,
               number_text_tokens=12000, n_langs=8):
    return dict(layers=layers, model_dim=model_dim, heads=heads, number_mel_codes=number_mel_codes,
                start_mel_token=start_mel_token, stop_mel_token=stop_mel_token,
                max_mel_tokens=max_mel_tokens, max_text_tokens=max_text_tokens,
                number_text_tokens=number_text_tokens, n_langs=n_langs,
                max_mel_positions=max_mel_tokens + 2 + 1)  # model_v2.py:398-400


def make_gpt_weights(cfg, seed=1234, bf16=True, head_gain=4.0):
    """Deterministic synthetic weights under the reference's state-dict names.

    Init follows transformers_gpt2.py:689-714 (normal std 0.02, c_proj std 0.02/sqrt(2L)) and
    model_v2.py:249,413-417 (embeddings std 0.02), except that biases / LayerNorm affine get
    small random values so the bias paths are exercised, and the mel head is scaled by
    `head_gain` so that greedy decisions are not dominated by ties of near-flat logits.
    """
    g = torch.Generator().manual_seed(seed)
    L, D, V = cfg["layers"], cfg["model_dim"], cfg["number_mel_codes"]
    w = {}

    def n(*shape, std=0.02):
        return torch.randn(*shape, generator=g) * std

    for l in range(L):
        p = f"gpt.h.{l}."
        w[p + "ln_1.weight"] = 1.0 + n(D, std=0.1)
        w[p + "ln_1.bias"] = n(D, std=0.05)
        w[p + "attn.c_attn.weight"] = n(D, 3 * D)
        w[p + "attn.c_attn.bias"] = n(3 * D)
        w[p + "attn.c_proj.weight"] = n(D, D, std=0.02 / math.sqrt(2 * L))
        w[p + "attn.c_proj.bias"] = n(D)
        w[p + "ln_2.weight"] = 1.0 + n(D, std=0.1)
        w[p + "ln_2.bias"] = n(D, std=0.05)
        w[p + "mlp.c_fc.weight"] = n(D, 4 * D)
        w[p + "mlp.c_fc.bias"] = n(4 * D)
        w[p + "mlp.c_proj.weight"] = n(4 * D, D, std=0.02 / math.sqrt(2 * L))
        w[p + "mlp.c_proj.bias"] = n(D)
    w["gpt.ln_f.weight"] = 1.0 + n(D, std=0.1)
    w["gpt.ln_f.bias"] = n(D, std=0.05)
    w["final_norm.weight"] = 1.0 + n(D, std=0.1)
    w["final_norm.bias"] = n(D, std=0.05)
    w["mel_head.weight"] = n(V, D, std=head_gain / math.sqrt(D))
    w["mel_head.bias"] = n(V, std=0.1)
    w["mel_embedding.weight"] = n(V, D)
    w["mel_pos_embedding.emb.weight"] = n(cfg["max_mel_positions"], D)
    w["text_embedding.weight"] = n(cfg["number_text_tokens"] + 1, D)
    w["text_pos_embedding.emb.weight"] = n(cfg["max_text_tokens"] + 2, D)
    w["lang_embedding.weight"] = n(cfg["n_langs"] + 1, D)
    w["spk_emb_proj.weight"] = n(D, 192, std=1.0 / math.sqrt(192))
    w["spk_emb_proj.bias"] = n(D)
    if bf16:
        w = {k: r16(v) for k, v in w.items()}
    return w


BIGVGAN_V2_22K = dict(  # s2mel/modules/bigvgan/config.json:11-21
    num_mels=80, upsample_rates=[4, 4, 2, 2, 2, 2], upsample_kernel_sizes=[8, 8, 4, 4, 4, 4],
    upsample_initial_channel=1536, resblock_kernel_sizes=[3, 7, 11],
    resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]], use_tanh_at_final=False,
    use_bias_at_final=False, activation="snakebeta", snake_logscale=True, resblock="1")


def small_config(ch=64, rates=(4, 2), ksz=(8, 4)):
    h = dict(BIGVGAN_V2_22K)
    h.update(upsample_initial_channel=ch, upsample_rates=list(rates), upsample_kernel_sizes=list(ksz))
    return h


def kaiser_sinc_filter1d(cutoff=0.25, half_width=0.3, kernel_size=12):  # filter.py:30-70
    half_size = kernel_size // 2
    delta_f = 4 * half_width
    A = 2.285 * (half_size - 1) * math.pi * delta_f + 7.95
    if A > 50.0:
        beta = 0.1102 * (A - 8.7)
    elif A >= 21.0:
        beta = 0.5842 * (A - 21) ** 0.4 + 0.07886 * (A - 21.0)
    else:
        beta = 0.0
    window = torch.kaiser_window(kernel_size, beta=beta, periodic=False)
    time = torch.arange(-half_size, half_size) + 0.5
    filt = 2 * cutoff * window * torch.sinc(2 * cutoff * time)
    filt = filt / filt.sum()
    return filt.view(1, 1, kernel_size)


def make_bigvgan_weights(h, seed=1234, post_gain=0.06):
    """Seeded synthetic generator weights under the reference state-dict names (weight norm
    already removed).  Conv weights are scaled to 1/sqrt(fan_in) so activations neither vanish
    nor explode through the 6 stages (the reference's std 0.01 init, bigvgan/utils.py:45-48,
    would drive everything to ~0); alpha/beta ~ N(0, 0.3) in log scale."""
    g = torch.Generator().manual_seed(seed)
    w = {}

    def conv(name, co, ci, k, bias=True, gain=1.0):
        w[name + ".weight"] = torch.randn(co, ci, k, generator=g) * (gain / math.sqrt(ci * k))
        if bias:
            w[name + ".bias"] = torch.randn(co, generator=g) * 0.05

    def act(name, c):
        w[name + ".act.alpha"] = torch.randn(c, generator=g) * 0.3
        w[name + ".act.beta"] = torch.randn(c, generator=g) * 0.3
        filt = kaiser_sinc_filter1d()
        w[name + ".upsample.filter"] = filt.clone()
        w[name + ".downsample.lowpass.filter"] = filt.clone()

    ch = h["upsample_initial_channel"]
    conv("conv_pre", ch, h["num_mels"], 7)
    nk = len(h["resblock_kernel_sizes"])
    for i, (u, k) in enumerate(zip(h["upsample_rates"], h["upsample_kernel_sizes"])):
        # ConvTranspose1d weight is [in, out, k]; each output sees k/u taps
        w[f"ups.{i}.0.weight"] = torch.randn(ch, ch // 2, k, generator=g) * (1.0 / math.sqrt(ch * k / u))
        w[f"ups.{i}.0.bias"] = torch.randn(ch // 2, generator=g) * 0.05
        ch //= 2
        for j, ks in enumerate(h["resblock_kernel_sizes"]):
            rb = i * nk + j
            for m in range(3):
                conv(f"resblocks.{rb}.convs1.{m}", ch, ch, ks, gain=0.7)
                conv(f"resblocks.{rb}.convs2.{m}", ch, ch, ks, gain=0.5)
            for q in range(6):
                act(f"resblocks.{rb}.activations.{q}", ch)
    act("activation_post", ch)
    conv("conv_post", 1, ch, 7, bias=h.get("use_bias_at_final", True), gain=post_gain)
    return w


def synthetic_mel(B, F_, seed=0, num_mels=80):
    """log-mel shaped input: N(-5, 2^2) clipped to [-11.5, 2] (SURVEY.md §8d config 4)."""
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, num_mels, F_, generator=g) * 2.0 - 5.0).clamp(-11.5, 2.0)


S2MEL_CFG = dict(hidden=512, heads=8, depth=13, wn_hidden=512, wn_layers=8, wn_kernel=5,
                 in_channels=80, content_dim=512, style_dim=192, lr_in=1024, lr_convs=4)


CODEC_CFG = dict(codebook_size=8192, hidden_size=1024, codebook_dim=8, vocos_dim=384,
                 vocos_intermediate_dim=2048, vocos_num_layers=12)


def small_s2mel_cfg():
    c = dict(S2MEL_CFG)
    c.update(hidden=128, heads=2, depth=5, wn_hidden=128, wn_layers=3, content_dim=64, lr_in=96)  # FinalLayer needs wn_hidden == hidden
    return c


def small_codec_cfg():
    return dict(codebook_size=64, hidden_size=96, codebook_dim=8, vocos_dim=48,
                vocos_intermediate_dim=128, vocos_num_layers=3)


def make_s2mel_weights(c, seed=1234):
    """Seeded synthetic weights under the reference names (as stored in a checkpoint: weight-norm
    layers keep weight_g/weight_v).  1/sqrt(fan_in) scaling keeps activations O(1); adaLN
    projections are biased to (scale~1, shift~0) like a trained model."""
    g = torch.Generator().manual_seed(seed)
    w = {}
    H, Dn, WH, NL, C = c["hidden"], c["depth"], c["wn_hidden"], c["wn_layers"], c["in_channels"]
    inter = ((int(2 * 4 * H / 3) + 255) // 256) * 256

    def lin(name, co, ci, bias=True, gain=1.0):
        w[name + ".weight"] = torch.randn(co, ci, generator=g) * (gain / math.sqrt(ci))
        if bias:
            w[name + ".bias"] = torch.randn(co, generator=g) * 0.05

    def wn(name, shape, bias=True, gain=1.0):
        v = torch.randn(*shape, generator=g) * (1.0 / math.sqrt(np.prod(shape[1:])))
        w[name + ".weight_v"] = v
        w[name + ".weight_g"] = (v.reshape(shape[0], -1).norm(dim=1) * gain *
                                 (1.0 + 0.1 * torch.randn(shape[0], generator=g))).reshape(shape[0], *([1] * (len(shape) - 1)))
        if bias:
            w[name + ".bias"] = torch.randn(shape[0], generator=g) * 0.05

    def adaln(name, dim):
        w[name + ".project_layer.weight"] = torch.randn(2 * dim, dim, generator=g) * (0.3 / math.sqrt(dim))
        b = torch.randn(2 * dim, generator=g) * 0.05
        b[:dim] += 1.0
        w[name + ".project_layer.bias"] = b
        w[name + ".norm.weight"] = 1.0 + 0.1 * torch.randn(dim, generator=g)

    e = "cfm.estimator."
    for l in range(Dn):
        p = e + f"transformer.layers.{l}."
        lin(p + "attention.wqkv", 3 * H, H, bias=False)
        lin(p + "attention.wo", H, H, bias=False, gain=0.5)
        lin(p + "feed_forward.w1", inter, H, bias=False)
        lin(p + "feed_forward.w3", inter, H, bias=False)
        lin(p + "feed_forward.w2", H, inter, bias=False, gain=0.5)
        adaln(p + "ffn_norm", H)
        adaln(p + "attention_norm", H)
        lin(p + "skip_in_linear", H, 2 * H)
    adaln(e + "transformer.norm", H)
    wn(e + "x_embedder", (H, C))                      # present in checkpoints, unused by forward
    w[e + "cond_embedder.weight"] = torch.randn(1024, H, generator=g) * 0.02
    lin(e + "cond_projection", H, c["content_dim"])
    for te, dim in (("t_embedder", H), ("t_embedder2", WH)):
        half = 128
        w[e + te + ".freqs"] = torch.exp(-math.log(10000) * torch.arange(0, half, dtype=torch.float32) / half)
        lin(e + te + ".mlp.0", dim, 256)
        lin(e + te + ".mlp.2", dim, dim)
    lin(e + "conv1", WH, H)
    w[e + "conv2.weight"] = torch.randn(C, WH, 1, generator=g) * (1.0 / math.sqrt(WH))
    w[e + "conv2.bias"] = torch.randn(C, generator=g) * 0.05
    for i in range(NL):
        wn(e + f"wavenet.in_layers.{i}.conv.conv", (2 * WH, WH, c["wn_kernel"]))
        co = 2 * WH if i < NL - 1 else WH
        wn(e + f"wavenet.res_skip_layers.{i}.conv.conv", (co, WH, 1), gain=0.5)
    wn(e + "wavenet.cond_layer.conv.conv", (2 * WH * NL, WH, 1))
    wn(e + "final_layer.linear", (WH, WH))
    lin(e + "final_layer.adaLN_modulation.1", 2 * WH, WH, gain=0.3)
    lin(e + "res_projection", WH, H)
    w[e + "content_mask_embedder.weight"] = torch.zeros(1, H)
    lin(e + "skip_linear", H, H + C)
    lin(e + "cond_x_merge_linear", H, H + 2 * C + c["style_dim"])
    w[e + "input_pos"] = torch.arange(16384)
    # length regulator
    r = "length_regulator."
    ch = c["content_dim"]
    w[r + "mask_token"] = torch.zeros(1, ch)
    w[r + "embedding.weight"] = torch.randn(2048, ch, generator=g) * 0.02
    lin(r + "content_in_proj", ch, c["lr_in"])
    for i in range(c["lr_convs"]):
        w[r + f"model.{3 * i}.weight"] = torch.randn(ch, ch, 3, generator=g) * (1.0 / math.sqrt(3 * ch))
        w[r + f"model.{3 * i}.bias"] = torch.randn(ch, generator=g) * 0.05
        w[r + f"model.{3 * i + 1}.weight"] = 1.0 + 0.1 * torch.randn(ch, generator=g)
        w[r + f"model.{3 * i + 1}.bias"] = torch.randn(ch, generator=g) * 0.05
    k = 3 * c["lr_convs"]
    w[r + f"model.{k}.weight"] = torch.randn(ch, ch, 1, generator=g) * (1.0 / math.sqrt(ch))
    w[r + f"model.{k}.bias"] = torch.randn(ch, generator=g) * 0.05
    return w


def make_codec_weights(c, seed=4321):
    g = torch.Generator().manual_seed(seed)
    w = {}
    Hs, Cd, Vd, Vi = c["hidden_size"], c["codebook_dim"], c["vocos_dim"], c["vocos_intermediate_dim"]

    def t(*shape, std):
        return torch.randn(*shape, generator=g) * std

    q = "quantizer.quantizers.0."
    w[q + "codebook.weight"] = t(c["codebook_size"], Cd, std=1.0)
    for nm, (co, ci) in (("in_project", (Cd, Hs)), ("out_project", (Hs, Cd))):
        v = t(co, ci, 1, std=1.0 / math.sqrt(ci))
        w[q + nm + ".weight_v"] = v
        w[q + nm + ".weight_g"] = v.reshape(co, -1).norm(dim=1).reshape(co, 1, 1) * (1 + 0.1 * torch.randn(co, generator=g)).reshape(co, 1, 1)
        w[q + nm + ".bias"] = t(co, std=0.05)
    for part in ("encoder", "decoder"):
        b = part + ".0."
        w[b + "embed.weight"] = t(Vd, Hs, 7, std=1.0 / math.sqrt(7 * Hs))
        w[b + "embed.bias"] = t(Vd, std=0.05)
        for nm in ("norm", "final_layer_norm"):
            w[b + nm + ".weight"] = 1.0 + t(Vd, std=0.1)
            w[b + nm + ".bias"] = t(Vd, std=0.05)
        for l in range(c["vocos_num_layers"]):
            p = b + f"convnext.{l}."
            w[p + "dwconv.weight"] = t(Vd, 1, 7, std=1.0 / math.sqrt(7))
            w[p + "dwconv.bias"] = t(Vd, std=0.05)
            w[p + "norm.weight"] = 1.0 + t(Vd, std=0.1)
            w[p + "norm.bias"] = t(Vd, std=0.05)
            w[p + "pwconv1.weight"] = t(Vi, Vd, std=1.0 / math.sqrt(Vd))
            w[p + "pwconv1.bias"] = t(Vi, std=0.05)
            w[p + "pwconv2.weight"] = t(Vd, Vi, std=1.0 / math.sqrt(Vi))
            w[p + "pwconv2.bias"] = t(Vd, std=0.05)
            w[p + "gamma"] = 0.3 + t(Vd, std=0.05)
        w[part + ".1.weight"] = t(Hs, Vd, std=1.0 / math.sqrt(Vd))
        w[part + ".1.bias"] = t(Hs, std=0.05)
    for nm in ("down", "up"):
        w[nm + ".weight"] = t(Hs, Hs, 3, std=1.0 / math.sqrt(3 * Hs))
        w[nm + ".bias"] = t(Hs, std=0.05)
    return w


EMO_CFG = dict(idim=1024, odim=512, linear_units=1024, heads=4, blocks=4, cnn_kernel=15,
               p_dim=1024, p_heads=4, p_dim_head=64, p_depth=2, p_ff_mult=2, model_dim=1280)


def small_emo_cfg():
    return dict(idim=40, odim=32, linear_units=48, heads=2, blocks=2, cnn_kernel=15,
                p_dim=64, p_heads=2, p_dim_head=64, p_depth=2, p_ff_mult=2, model_dim=256)


def make_emo_weights(c, seed=777, enc_prefix="emo_conditioning_encoder.", per_prefix="emo_perceiver_encoder.", n_latents=1,
                     heads_out=True):
    """Emotion path of UnifiedVoice (gpt/model_v2.py:375-392): emo_conditioning_encoder (Conformer),
    emo_perceiver_encoder (1 latent), emovec_layer, emo_layer — reference state-dict names."""
    g = torch.Generator().manual_seed(seed)
    w = {}

    def t(*shape, std):
        return torch.randn(*shape, generator=g) * std

    def lin(name, co, ci, bias=True, gain=1.0):
        w[name + ".weight"] = t(co, ci, std=gain / math.sqrt(ci))
        if bias:
            w[name + ".bias"] = t(co, std=0.05)

    def ln(name, d):
        w[name + ".weight"] = 1.0 + t(d, std=0.1)
        w[name + ".bias"] = t(d, std=0.05)

    od, H = c["odim"], c["heads"]
    e = enc_prefix
    w[e + "embed.conv.0.weight"] = t(od, 1, 3, 3, std=1.0 / 3.0)
    w[e + "embed.conv.0.bias"] = t(od, std=0.05)
    fsub = (c["idim"] - 1) // 2
    lin(e + "embed.out.0", od, od * fsub, gain=1.5)
    for i in range(c["blocks"]):
        p = e + f"encoders.{i}."
        for nm in ("linear_q", "linear_k", "linear_v", "linear_out"):
            lin(p + "self_attn." + nm, od, od)
        lin(p + "self_attn.linear_pos", od, od, bias=False)
        w[p + "self_attn.pos_bias_u"] = t(H, od // H, std=0.1)
        w[p + "self_attn.pos_bias_v"] = t(H, od // H, std=0.1)
        lin(p + "feed_forward.w_1", c["linear_units"], od)
        lin(p + "feed_forward.w_2", od, c["linear_units"], gain=0.5)
        w[p + "conv_module.pointwise_conv1.weight"] = t(2 * od, od, 1, std=1.0 / math.sqrt(od))
        w[p + "conv_module.pointwise_conv1.bias"] = t(2 * od, std=0.05)
        w[p + "conv_module.depthwise_conv.weight"] = t(od, 1, c["cnn_kernel"], std=1.0 / math.sqrt(c["cnn_kernel"]))
        w[p + "conv_module.depthwise_conv.bias"] = t(od, std=0.05)
        ln(p + "conv_module.norm", od)
        w[p + "conv_module.pointwise_conv2.weight"] = t(od, od, 1, std=0.5 / math.sqrt(od))
        w[p + "conv_module.pointwise_conv2.bias"] = t(od, std=0.05)
        for nm in ("norm_ff", "norm_mha", "norm_conv", "norm_final"):
            ln(p + nm, od)
    ln(e + "after_norm", od)
    q = per_prefix
    pd, inner = c["p_dim"], c["p_heads"] * c["p_dim_head"]
    lin(q + "proj_context", pd, od)
    w[q + "latents"] = t(n_latents, pd, std=0.02 if n_latents == 1 else 1.0)
    di = int(pd * c["p_ff_mult"] * 2 / 3)
    for i in range(c["p_depth"]):
        lin(q + f"layers.{i}.0.to_q", inner, pd, bias=False)
        lin(q + f"layers.{i}.0.to_kv", 2 * inner, pd, bias=False)
        lin(q + f"layers.{i}.0.to_out", pd, inner, bias=False, gain=0.5)
        lin(q + f"layers.{i}.1.0", 2 * di, pd)
        lin(q + f"layers.{i}.1.2", pd, di, gain=0.5)
    w[q + "norm.gamma"] = 1.0 + t(pd, std=0.1)
    if heads_out:
        lin("emovec_layer", c["model_dim"], pd)
        lin("emo_layer", c["model_dim"], c["model_dim"])
    return w


# ------------------------------------------------------------------ IndexTTS v1 / v1.5 vocoder (row a13) --
def small_v1_config():
    """A tiny latent-conditioned BigVGAN (indextts/BigVGAN/models.py:129-199) for tests; the ECAPA-TDNN speaker encoder
    inside it is always the full 512/1536-channel network (ECAPA_TDNN.py:470-541 defaults)."""
    return dict(gpt_dim=32, upsample_rates=[4, 2], upsample_kernel_sizes=[8, 4], upsample_initial_channel=32,
                resblock="1", resblock_kernel_sizes=[3, 7], resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5]],
                activation="snakebeta", snake_logscale=True, feat_upsample=False,
                cond_d_vector_in_each_upsampling_layer=True, speaker_embedding_dim=24, num_mels=20)


def v1_5_config():
    """The IndexTTS-1.5 vocoder: 1280-d GPT latents -> 1536 channels, six upsamples (x1024, 24 kHz), AMPBlock1 with
    kernels 3/7/11, snakebeta, the speaker embedding added after conv_pre and after every upsample.

    [ASSUMED] from the published IndexTTS-1.5 checkpoints/config.yaml, which the reference checkout does not carry;
    consistent with SURVEY section 8 row a13 (1280-d latents, x1024, 24 kHz).  Its GPT is
    gpt_config(max_mel_tokens=605, max_text_tokens=402) with the V1_COND_CFG conditioning encoder, also [ASSUMED]."""
    return dict(gpt_dim=1280, upsample_rates=[4, 4, 4, 4, 2, 2], upsample_kernel_sizes=[8, 8, 4, 4, 4, 4],
                upsample_initial_channel=1536, resblock="1", resblock_kernel_sizes=[3, 7, 11],
                resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]], activation="snakebeta", snake_logscale=True,
                feat_upsample=False, cond_d_vector_in_each_upsampling_layer=True, speaker_embedding_dim=512, num_mels=100)


V1_5_POST_GAIN = 0.012      # conv_post gain of the v1.5 test weights (make_bigvgan_v1_weights)


# v1 / v1.5 conditioning encoder (gpt/model.py:352-363): conformer over a 100-bin mel (512 dims, 2048 FF units, 8 heads,
# 6 blocks) and a 32-latent perceiver at p_dim = model_dim = 1280
V1_COND_CFG = dict(idim=100, odim=512, linear_units=2048, heads=8, blocks=6, cnn_kernel=15, p_dim=1280, p_heads=8,
                   p_dim_head=64, p_depth=2, p_ff_mult=2, model_dim=1280)


def make_ecapa_weights(n_mels, emb_dim, seed=99, prefix="speaker_encoder.", channels=(512, 512, 512, 512, 1536),
                       kernel_sizes=(5, 3, 3, 3, 1), scale=8, se_channels=128, attention_channels=128):
    """Seeded ECAPA-TDNN weights under the reference state-dict names (ECAPA_TDNN.py:470-541), BatchNorm running
    statistics included (eval mode)."""
    g = torch.Generator().manual_seed(seed)
    w = {}

    def conv(name, co, ci, k, gain=1.0):
        w[name + ".weight"] = torch.randn(co, ci, k, generator=g) * (gain / math.sqrt(ci * k))
        w[name + ".bias"] = torch.randn(co, generator=g) * 0.05

    def bn(name, c):
        w[name + ".weight"] = 1.0 + torch.randn(c, generator=g) * 0.1
        w[name + ".bias"] = torch.randn(c, generator=g) * 0.05
        w[name + ".running_mean"] = torch.randn(c, generator=g) * 0.1
        w[name + ".running_var"] = 0.6 + torch.rand(c, generator=g) * 0.8

    def tdnn(name, ci, co, k):
        conv(name + ".conv.conv", co, ci, k, gain=1.4)      # ReLU halves the power
        bn(name + ".norm.norm", co)

    q = prefix
    tdnn(q + "blocks.0", n_mels, channels[0], kernel_sizes[0])
    for i in range(1, len(channels) - 1):
        p = q + f"blocks.{i}"
        if channels[i - 1] != channels[i]:
            conv(p + ".shortcut.conv", channels[i], channels[i - 1], 1)
        tdnn(p + ".tdnn1", channels[i - 1], channels[i], 1)
        for j in range(scale - 1):
            tdnn(p + f".res2net_block.blocks.{j}", channels[i] // scale, channels[i] // scale, kernel_sizes[i])
        tdnn(p + ".tdnn2", channels[i], channels[i], 1)
        conv(p + ".se_block.conv1.conv", se_channels, channels[i], 1)
        conv(p + ".se_block.conv2.conv", channels[i], se_channels, 1)
    tdnn(q + "mfa", channels[-2] * (len(channels) - 2), channels[-1], kernel_sizes[-1])
    tdnn(q + "asp.tdnn", channels[-1] * 3, attention_channels, 1)
    conv(q + "asp.conv.conv", channels[-1], attention_channels, 1)
    bn(q + "asp_bn.norm", channels[-1] * 2)
    conv(q + "fc.conv", emb_dim, channels[-1] * 2, 1)
    return w


def make_bigvgan_v1_weights(h, seed=4321, post_gain=0.06):
    """Seeded weights of the latent-conditioned v1 BigVGAN under the reference state-dict names (weight norm removed).
    `post_gain` scales conv_post: at the v1.5 geometry the default drives 1/3 of the samples into tanh saturation, where
    the waveform hides the generator's errors; V1_5_POST_GAIN keeps it in the near-linear range."""
    h2 = dict(h, num_mels=h["gpt_dim"], use_bias_at_final=True)
    w = make_bigvgan_weights(h2, seed=seed, post_gain=post_gain)   # same generator layout: conv_pre takes gpt_dim channels
    g = torch.Generator().manual_seed(seed + 1)
    E, ch = h["speaker_embedding_dim"], h["upsample_initial_channel"]
    w["cond_layer.weight"] = torch.randn(ch, E, 1, generator=g) * (0.5 / math.sqrt(E))
    w["cond_layer.bias"] = torch.randn(ch, generator=g) * 0.05
    for i in range(len(h["upsample_rates"])):
        ch //= 2
        w[f"conds.{i}.weight"] = torch.randn(ch, E, 1, generator=g) * (0.5 / math.sqrt(E))
        w[f"conds.{i}.bias"] = torch.randn(ch, generator=g) * 0.05
    w.update(make_ecapa_weights(h["num_mels"], E, seed=seed + 2))
    return w


def small_v1_cond_cfg(model_dim=256):
    """v1 conditioning encoder (gpt/model.py:352-363) at test size: conformer over a 100-bin mel + 32-latent perceiver."""
    return dict(idim=100, odim=32, linear_units=48, heads=2, blocks=2, cnn_kernel=15, p_dim=model_dim, p_heads=2,
                p_dim_head=64, p_depth=2, p_ff_mult=2, model_dim=model_dim)


def make_gpt_v1_weights(cfg, ccfg, seed=1234):
    """Seeded v1 UnifiedVoice weights (reference state-dict names): the GPT stack of make_gpt_weights without the v2-only
    tensors, plus conditioning_encoder.* / perceiver_encoder.* (32 latents)."""
    w = make_gpt_weights(cfg, seed=seed, bf16=False)
    for k in ("spk_emb_proj.weight", "spk_emb_proj.bias", "lang_embedding.weight"):
        w.pop(k, None)
    w.update(make_emo_weights(ccfg, seed=seed + 7, enc_prefix="conditioning_encoder.", per_prefix="perceiver_encoder.",
                              n_latents=32, heads_out=False))
    return w
