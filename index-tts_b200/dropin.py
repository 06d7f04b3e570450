"""Drop-in binding for the reference pipeline classes.

`attach(tts)` takes a live reference object — `indextts.infer_v2_5.IndexTTS2` built by the reference's own
constructor, i.e. with its own config/checkpoint loaders (`indextts.infer_v2.IndexTTS2` is NOT covered: its
`inference_speech` call passes no `campplus_embedding` and consumes the returned conditioning latent,
infer_v2.py:583-662 — `attach` raises for it) — registers the
weights of its modules with the CUDA engine and rebinds the module-level seams of `infer_generator`
(SURVEY.md §8b) to the C-ABI:

    tts.gpt.merge_emovec              → idx_merge_emovec                            (model_v2.py:827-838)
    tts.gpt.inference_speech          → idx_gpt_prepare_inputs + idx_gpt_generate   (model_v2.py:716-825)
    tts.semantic_codec.decode         → idx_codec_decode                            (codec/models.py:205-231)
    tts.s2mel.models['length_regulator'](…)  → idx_length_regulate                  (length_regulator.py:90-141)
    tts.s2mel.models['cfm'].inference → idx_cfm_solve                               (flow_matching.py:30-115)
    tts.bigvgan(mel)                  → idx_bigvgan_forward                         (bigvgan.py:360-386)
    tts.get_emb                       → idx_semantic_encode                         (infer_v2_5.py:281-290)

`infer_v2_5.py` itself is not modified: `.infer()` keeps its signature, text front-end, prompt caching,
segment loop and timing prints, and simply reaches these callables instead of the PyTorch modules.  Tensors
stay torch tensors (containers) ON THE DEVICE: the engine receives their raw device pointers and writes its results into
torch CUDA tensors (no `.cpu().numpy()` bounce at any seam; only the few dozen text ids and the generated codes cross
the host).  The engine stream is ordered after torch's current stream before every call (include/idxtts.h, stream
contract).  Nothing here falls back to PyTorch compute: if the engine cannot be created the call raises.
"""
import types

import numpy as np
import torch

from .engine import Engine, fold_weight_norm


def _sd(module):
    # `inference_model.*` re-exports the same tensors (GPT2InferenceModel shares the blocks, model_v2.py:466-474)
    return {k: v.detach() for k, v in module.state_dict().items()
            if torch.is_floating_point(v) and not k.startswith("inference_model.")}


def load_reference_weights(engine: Engine, tts, max_batch: int = 1):
    """Register the weights the reference loaded (checkpoint.py:22-35, commons.py:579-635,
    codec/models.py:233-247, bigvgan.py:413-492) and size the engine from the modules' own shapes."""
    gpt = tts.gpt
    sd = _sd(gpt)
    engine.load_state_dict("gpt.", sd)
    layers = len(gpt.gpt.h)
    D = gpt.model_dim
    engine.gpt_init(layers, D, gpt.heads, gpt.number_mel_codes, gpt.start_mel_token, gpt.stop_mel_token,
                    sd["mel_pos_embedding.emb.weight"].shape[0],
                    max_prompt=sd["text_pos_embedding.emb.weight"].shape[0] + 8, max_batch=max_batch,
                    weights_bf16=True)
    # emotion conformer + perceiver (model_v2.py:378-398), sized from the tensors; absent on stand-ins without them
    E, Q = "emo_conditioning_encoder.", "emo_perceiver_encoder."
    if E + "embed.out.0.weight" in sd:
        od = sd[E + "embed.out.0.weight"].shape[0]
        blocks = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith(E + "encoders."))
        lat = sd[Q + "latents"]
        inner = sd[Q + "layers.0.0.to_q.weight"].shape[0]
        heads = sd[E + "encoders.0.self_attn.pos_bias_u"].shape[0]
        p_heads = int(getattr(getattr(gpt, "emo_perceiver_encoder", None), "heads", 0)) or max(1, inner // 64)
        # Conv2dSubsampling2 (conformer/subsampling.py:144-160): out Linear takes od * ((idim - 1) // 2) features;
        # the w2v-BERT feature width is even (1024), hence 2 * fsub + 2
        fsub = sd[E + "embed.out.0.weight"].shape[1] // od
        engine.emo_init(dict(idim=int(getattr(gpt, "emo_input_size", 0)) or 2 * fsub + 2, odim=od, linear_units=sd[E + "encoders.0.feed_forward.w_1.weight"].shape[0], heads=heads,
                             blocks=blocks, cnn_kernel=sd[E + "encoders.0.conv_module.depthwise_conv.weight"].shape[-1],
                             p_dim=lat.shape[-1], p_heads=p_heads, p_dim_head=inner // p_heads,
                             p_depth=1 + max(int(k.split(".")[2]) for k in sd if k.startswith(Q + "layers.")),
                             p_ff_mult=max(1, round(sd[Q + "layers.0.1.0.weight"].shape[0] * 3 / (4 * lat.shape[-1]))),
                             model_dim=D))
    # s2mel (weight-norm parametrised layers are folded: g * v / ||v||)
    s2 = {k[len("models."):]: v for k, v in _sd(tts.s2mel).items()}
    s2 = fold_weight_norm(s2)
    engine.load_state_dict("s2mel.", s2)
    est = "cfm.estimator."
    H = s2[est + "cond_projection.weight"].shape[0]
    depth = 1 + max(int(k.split(".")[4]) for k in s2 if k.startswith(est + "transformer.layers."))
    wn_layers = 1 + max(int(k.split(".")[4]) for k in s2 if k.startswith(est + "wavenet.in_layers."))
    lr_convs = sum(1 for k in s2 if k.startswith("length_regulator.model.") and k.endswith(".weight")
                   and s2[k].dim() == 3 and s2[k].shape[-1] == 3)
    engine.s2mel_init(dict(hidden=H, heads=H // 64, depth=depth, wn_hidden=s2[est + "conv1.weight"].shape[0],
                           wn_layers=wn_layers, wn_kernel=s2[est + "wavenet.in_layers.0.conv.conv.weight"].shape[-1],
                           in_channels=s2[est + "conv2.weight"].shape[0],
                           content_dim=s2[est + "cond_projection.weight"].shape[1],
                           style_dim=s2[est + "cond_x_merge_linear.weight"].shape[1] - H - 2 * s2[est + "conv2.weight"].shape[0],
                           lr_in=s2["length_regulator.content_in_proj.weight"].shape[1], lr_convs=lr_convs))
    cd = fold_weight_norm(_sd(tts.semantic_codec))
    engine.load_state_dict("codec.", cd)
    q = "quantizer.quantizers.0."
    engine.codec_init(dict(codebook_size=cd[q + "codebook.weight"].shape[0], hidden_size=cd["decoder.1.weight"].shape[0],
                           codebook_dim=cd[q + "codebook.weight"].shape[1], vocos_dim=cd["decoder.1.weight"].shape[1],
                           vocos_intermediate_dim=cd["decoder.0.convnext.0.pwconv1.weight"].shape[0],
                           vocos_num_layers=1 + max(int(k.split(".")[3]) for k in cd if k.startswith("decoder.0.convnext."))))
    bv = fold_weight_norm(_sd(tts.bigvgan))
    engine.load_state_dict("bigvgan.", bv)
    engine.bigvgan_init(dict(tts.bigvgan.h))
    return engine


# get_emb reads hidden_states[17] of the w2v-BERT 2.0 encoder (infer_v2_5.py:288): the feature projection and the first 17
# conformer layers; layers 17..23 are never read.
SEMANTIC_LAYERS = 17


def attach_semantic(tts, engine: Engine):
    """Register the w2v-BERT weights get_emb uses (feature_projection.*, encoder.layers.0..16.*, semantic_mean / std) under
    "semantic.", size the encoder from the tensors and semantic_model.config, and rebind tts.get_emb to the engine."""
    sm = tts.semantic_model
    keep = ("feature_projection.",) + tuple(f"encoder.layers.{i}." for i in range(SEMANTIC_LAYERS))
    sd = {k: v for k, v in _sd(sm).items() if k.startswith(keep)}
    sd["semantic_mean"] = torch.as_tensor(tts.semantic_mean).reshape(-1)
    sd["semantic_std"] = torch.as_tensor(tts.semantic_std).reshape(-1)
    engine.load_state_dict("semantic.", sd)
    c = sm.config
    p = "encoder.layers.0."
    engine.semantic_init(dict(feat_dim=sd["feature_projection.projection.weight"].shape[1],
                              hidden=sd["feature_projection.projection.weight"].shape[0], heads=c.num_attention_heads,
                              ffn=sd[p + "ffn1.intermediate_dense.weight"].shape[0], layers=SEMANTIC_LAYERS,
                              conv_kernel=sd[p + "conv_module.depthwise_conv.weight"].shape[-1],
                              left_max=c.left_max_position_embeddings, right_max=c.right_max_position_embeddings,
                              eps=c.layer_norm_eps))
    dev = torch.device("cuda", engine.device)

    def get_emb(input_features, attention_mask):
        # infer_v2_5.py:281-290: (hidden_states[17] - semantic_mean) / semantic_std, [B, T, 1024] on the device
        return torch.as_tensor(engine.get_emb(input_features, attention_mask)).to(dev)

    tts.get_emb = get_emb
    return tts


def _fresh_seed():
    """A new Philox key per generate call, drawn from torch's global generator: `torch.manual_seed(s)` before `.infer()`
    reproduces a take, and successive calls / segments differ — like the reference's torch.multinomial draws, which
    advance the global generator on every call (ADVICE r1: a constant torch.initial_seed() replayed one stream forever)."""
    return int(torch.randint(0, 2 ** 31 - 1, (1,)).item())


def _check_hf_kwargs(num_return_sequences, typical_sampling, hf):
    if typical_sampling:
        raise NotImplementedError("typical_sampling=True (TypicalLogitsWarper, model_v2.py:798-800) is not built on the engine path")
    if int(num_return_sequences or 1) != 1:
        raise NotImplementedError("num_return_sequences must be 1 (what infer_v2_5.py:771-791 / infer.py pass)")
    nb = int(hf.get("num_beams", 1) or 1)
    if nb > 4:
        raise NotImplementedError("num_beams <= 4 (the reference default is 3)")
    if hf.get("do_sample", False):
        tk = int(hf.get("top_k", 0) or 0)
        if tk <= 0 or tk > 128:
            raise NotImplementedError("do_sample needs 1 <= top_k <= 128 on the engine path (the reference default is 30, the "
                                      "webui allows up to 100); top_k=0 / larger values are rejected, never silently capped")
    return nb


def attach(tts, engine: Engine = None, device: int = 0):
    """Rebind the compute seams of a reference IndexTTS2 (infer_v2_5) instance to the CUDA engine (see module doc)."""
    if type(tts).__module__.endswith("infer_v2"):
        raise NotImplementedError("attach() covers indextts.infer_v2_5.IndexTTS2; infer_v2.IndexTTS2 (row f3) is not built")
    engine = engine or Engine(device)
    load_reference_weights(engine, tts, max_batch=4)      # room for the default 3 beams
    if hasattr(tts, "semantic_model"):
        attach_semantic(tts, engine)
    dev = torch.device("cuda", engine.device)
    gpt = tts.gpt

    def inference_speech(self, speech_condition, text_inputs, langs=None, emo_speech_condition=None, cond_lengths=None,
                         emo_cond_lengths=None, emo_vec=None, use_speed=False, campplus_embedding=None, wav=None,
                         input_tokens=None, num_return_sequences=1, max_generate_length=None, typical_sampling=False,
                         typical_mass=.9, **hf):
        # same argument meaning as gpt/model_v2.py:716-825; emo_vec comes from merge_emovec (:833-838)
        if emo_vec is None or campplus_embedding is None:
            raise ValueError("the engine path needs emo_vec and campplus_embedding (what infer_v2_5.py:759-791 passes)")
        nb = _check_hf_kwargs(num_return_sequences, typical_sampling, hf)
        sampling = dict(do_sample=bool(hf.get("do_sample", False)), top_k=int(hf.get("top_k", 0) or 0),
                        top_p=float(hf.get("top_p", 1.0)), temperature=float(hf.get("temperature", 1.0)),
                        seed=_fresh_seed(), num_beams=nb,
                        length_penalty=float(hf.get("length_penalty", 0.0)))
        lang = int(langs.reshape(-1)[0]) if langs is not None else 0
        outs = []
        styles = campplus_embedding.reshape(-1, 192)
        for i in range(text_inputs.shape[0]):
            # device tensors go in as device pointers; the prompt rows stay on the device for idx_gpt_generate
            prompt = engine.gpt_prepare_inputs(styles[min(i, styles.shape[0] - 1)], emo_vec.reshape(-1, self.model_dim)[0],
                                               text_inputs[i], lang)
            max_new = max_generate_length if max_generate_length is not None else self.max_mel_tokens - 1
            (codes,) = engine.gpt_generate([prompt], int(max_new),
                                           repetition_penalty=float(hf.get("repetition_penalty", 1.0)), **sampling)
            outs.append(torch.from_numpy(codes.astype(np.int64)))
        n = max(len(o) for o in outs)
        pad = torch.full((len(outs), n), self.stop_mel_token, dtype=torch.long)
        for i, o in enumerate(outs):
            pad[i, : len(o)] = o
        return pad.to(dev), None

    gpt.inference_speech = types.MethodType(inference_speech, gpt)

    if getattr(engine, "emo_cfg", None) is not None:
        def merge_emovec(self, speech_condition, emo_speech_condition, cond_lengths=None, emo_cond_lengths=None, alpha=1.0):
            # model_v2.py:827-838; features [1, T, 1024] (or [1, 1024, T], transposed like get_emo_conditioning :588-593)
            def feats(x, lengths, what):
                x = x[0].float()
                x = (x.t() if x.shape[0] == engine.emo_cfg.idim and x.shape[1] != engine.emo_cfg.idim else x).contiguous()
                # The conformer masks rows at or beyond the given length; the engine encodes every row.  infer_v2_5.py passes
                # the feature dim (1024, trap P10), which masks nothing for T <= 1024.
                if lengths is not None and int(torch.as_tensor(lengths).reshape(-1).min()) < x.shape[0]:
                    raise RuntimeError(f"merge_emovec: {what} {torch.as_tensor(lengths).reshape(-1).tolist()} is below the "
                                       f"{x.shape[0]} feature rows; the engine does not mask rows")
                return x
            v = engine.merge_emovec(feats(speech_condition, cond_lengths, "cond_lengths"),
                                    feats(emo_speech_condition, emo_cond_lengths, "emo_cond_lengths"), float(alpha))
            return torch.as_tensor(v)[None].to(dev)

        gpt.merge_emovec = types.MethodType(merge_emovec, gpt)

    def codec_decode(self, codes):
        c = codes.reshape(-1, codes.shape[-1])
        out = [torch.as_tensor(engine.codec_decode(c[i])) for i in range(c.shape[0])]
        return torch.stack(out).to(dev)

    tts.semantic_codec.decode = types.MethodType(codec_decode, tts.semantic_codec)

    class _LengthRegulator(torch.nn.Module):
        def forward(self, x, ylens=None, n_quantizers=None, f0=None):
            y = engine.length_regulate(x[0].float().contiguous(), int(ylens.max()))
            return torch.as_tensor(y)[None].to(dev), ylens, None, None, None

    tts.s2mel.models["length_regulator"] = _LengthRegulator()

    cfm = tts.s2mel.models["cfm"]

    def cfm_inference(self, mu, x_lens, prompt, style, f0, n_timesteps, temperature=1.0, inference_cfg_rate=0.5):
        B, T = mu.size(0), mu.size(1)
        z = torch.randn([B, self.in_channels, T], device=mu.device) * temperature   # same RNG call (trap P6)
        out = engine.cfm_solve(mu[0].float().contiguous(), prompt[0].float().contiguous(), style[0].float().contiguous(),
                               z[0].contiguous(), n_timesteps, inference_cfg_rate)
        return torch.as_tensor(out)[None].to(mu.device)

    cfm.inference = types.MethodType(cfm_inference, cfm)

    def bigvgan_forward(mel):
        return engine.bigvgan_forward(mel.float().contiguous())

    tts.bigvgan.forward = bigvgan_forward
    tts._b200_engine = engine
    return tts


# ------------------------------------------------------------------ IndexTTS v1 / v1.5 (indextts/infer.py) --
def attach_v1(tts, engine: Engine = None, device: int = 0):
    """Rebind the compute seams of a reference `indextts.infer.IndexTTS` instance (v1 / v1.5, SURVEY section 8 row a13):

        tts.gpt.inference_speech(mel, text, ...)          → idx_v1_get_conditioning + idx_gpt_prepare_inputs_v1 + idx_gpt_generate
                                                             (gpt/model.py:661-713; positions follow kv_cache, infer.py:101)
        tts.gpt(mel, text, ..., return_latent=True)       → idx_gpt_latents_v1                      (gpt/model.py:526-589)
        tts.bigvgan(latent, mel_ref)                      → idx_v1_vocode                            (BigVGAN/models.py:201-249)

    The strict fp32 GPT path is used (the reference's CPU configuration, BASELINE config 1)."""
    engine = engine or Engine(device)
    gpt = tts.gpt
    sd = _sd(gpt)
    engine.load_state_dict("gpt.", sd)
    D = gpt.model_dim
    engine.gpt_init(len(gpt.gpt.h), D, gpt.heads, gpt.number_mel_codes, gpt.start_mel_token, gpt.stop_mel_token,
                    sd["mel_pos_embedding.emb.weight"].shape[0],
                    max_prompt=sd["text_pos_embedding.emb.weight"].shape[0] + sd["perceiver_encoder.latents"].shape[0] + 8,
                    max_batch=4, weights_bf16=False)      # room for the default 3 beams
    E, Q = "conditioning_encoder.", "perceiver_encoder."
    od = sd[E + "embed.out.0.weight"].shape[0]
    fsub = sd[E + "embed.out.0.weight"].shape[1] // od
    inner = sd[Q + "layers.0.0.to_q.weight"].shape[0]
    p_heads = sd[E + "encoders.0.self_attn.pos_bias_u"].shape[0]
    n_lat = sd[Q + "latents"].shape[0]
    engine.v1_cond_init(dict(idim=2 * fsub + 2, odim=od, linear_units=sd[E + "encoders.0.feed_forward.w_1.weight"].shape[0],
                             heads=p_heads, blocks=1 + max(int(k.split(".")[2]) for k in sd if k.startswith(E + "encoders.")),
                             cnn_kernel=sd[E + "encoders.0.conv_module.depthwise_conv.weight"].shape[-1], p_dim=D, p_heads=p_heads,
                             p_dim_head=inner // p_heads,
                             p_depth=1 + max(int(k.split(".")[2]) for k in sd if k.startswith(Q + "layers.")),
                             p_ff_mult=max(1, round(sd[Q + "layers.0.1.0.weight"].shape[0] * 3 / (4 * D))), model_dim=D), n_lat)
    bv = fold_weight_norm({k: v for k, v in tts.bigvgan.state_dict().items() if torch.is_floating_point(v)})
    engine.load_state_dict("bigvgan_v1.", bv)
    engine.v1_vocoder_init(dict(tts.bigvgan.h))
    dev = torch.device("cuda", engine.device)
    kv_cache = bool(getattr(gpt.inference_model, "kv_cache", False))

    def _conds(mel):                                     # mel [1, 100, T] as infer.py passes it
        return engine.v1_get_conditioning(mel[0].float().t().contiguous().cpu().numpy())

    def inference_speech(self, speech_conditioning_mel, text_inputs, cond_mel_lengths=None, input_tokens=None,
                         num_return_sequences=1, max_generate_length=None, typical_sampling=False, typical_mass=.9, **hf):
        nb = _check_hf_kwargs(num_return_sequences, typical_sampling, hf)
        conds = _conds(speech_conditioning_mel)
        outs = []
        for i in range(text_inputs.shape[0]):
            prompt = engine.gpt_prepare_inputs_v1(conds, text_inputs[i].cpu().numpy())
            max_new = max_generate_length if max_generate_length is not None else self.max_mel_tokens - 1
            (codes,) = engine.gpt_generate([prompt], int(max_new), repetition_penalty=float(hf.get("repetition_penalty", 1.0)),
                                           do_sample=bool(hf.get("do_sample", False)), top_k=int(hf.get("top_k", 0) or 0),
                                           top_p=float(hf.get("top_p", 1.0)), temperature=float(hf.get("temperature", 1.0)),
                                           num_beams=nb, length_penalty=float(hf.get("length_penalty", 0.0)),
                                           seed=_fresh_seed(), mel_pos_mode=0 if kv_cache else 1)
            outs.append(torch.from_numpy(codes.astype(np.int64)))
        n = max(len(o) for o in outs)
        pad = torch.full((len(outs), n), self.stop_mel_token, dtype=torch.long)
        for i, o in enumerate(outs):
            pad[i, : len(o)] = o
        return pad.to(dev)

    gpt.inference_speech = types.MethodType(inference_speech, gpt)

    def forward(speech_conditioning_latent, text_inputs, text_lengths, mel_codes, wav_lengths, cond_mel_lengths=None, types=None,
                text_first=True, raw_mels=None, return_attentions=False, return_latent=False, clip_inputs=False):
        if not return_latent:
            raise NotImplementedError("the engine path implements the inference use of forward(): return_latent=True (infer.py:~640)")
        conds = _conds(speech_conditioning_latent)
        lat = engine.gpt_latents_v1(conds, text_inputs[0, : int(text_lengths[0])].cpu().numpy(), mel_codes[0].cpu().numpy())
        return torch.from_numpy(lat)[None].to(dev)

    gpt.forward = forward

    def bigvgan_forward(x, mel_ref, lens=None):
        wav = engine.v1_vocode(x[0].float().contiguous().cpu().numpy(), mel_ref[0].float().contiguous().cpu().numpy())
        return torch.from_numpy(wav)[None, None].to(dev), None

    tts.bigvgan.forward = bigvgan_forward
    tts._b200_engine = engine
    return tts
