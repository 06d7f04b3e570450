"""TEST INFRASTRUCTURE ONLY: CPU restatement of the IndexTTS v1 / v1.5 vocoder side (SURVEY.md section 8 row a13,
BASELINE config 1): the ECAPA-TDNN speaker encoder and the latent-conditioned BigVGAN.

  ECAPA_TDNN.forward                 indextts/BigVGAN/ECAPA_TDNN.py:543-582
    TDNNBlock (conv -> ReLU -> BN)   :79-128      Conv1d "same" + reflect padding: indextts/BigVGAN/nnet/CNN.py:411-470
    Res2NetBlock                     :131-191
    SEBlock                          :194-242
    AttentiveStatisticsPooling       :245-338
    SERes2NetBlock                   :341-426
  BigVGAN.forward (v1)               indextts/BigVGAN/models.py:201-249  (speaker embedding -> cond_layer / conds[i],
                                     latents [B, T, gpt_dim] in, tanh out)
  AMPBlock1 / Activation1d           models.py:33-125, alias_free_torch/* (same arithmetic as the v2 copy restated in
                                     oracle/bigvgan.py)

Pinned against the reference's own `indextts.BigVGAN.models.BigVGAN` (which owns the ECAPA encoder) by
oracle/make_goldens_v1.py -> tests/golden/v1_vocoder_small.npz and, at the IndexTTS-1.5 geometry,
tests/golden/v1_vocoder_full.npz.  The CUDA side (csrc/bigvgan.cu, csrc/ecapa.cu) is checked against it by
tests/test_v1_gpu.py and, at full size in float64 on the GPU, tests/test_v1_full_gpu.py.  The GPT-side functions below
run on whatever device and dtype the weights are on."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle.bigvgan import activation1d


def _conv_same(x, w, b, dilation=1):
    """speechbrain-style Conv1d(padding="same", padding_mode="reflect") for odd kernels (nnet/CNN.py:458-470)."""
    k = w.shape[-1]
    pad = dilation * (k - 1) // 2
    if pad:
        x = F.pad(x, (pad, pad), mode="reflect")
    return F.conv1d(x, w, b, dilation=dilation)


def _bn(x, w, p, eps=1e-5):
    return F.batch_norm(x, w[p + ".norm.running_mean"], w[p + ".norm.running_var"], w[p + ".norm.weight"], w[p + ".norm.bias"],
                        training=False, eps=eps)


def _tdnn(x, w, p, dilation=1):
    return _bn(F.relu(_conv_same(x, w[p + ".conv.conv.weight"], w[p + ".conv.conv.bias"], dilation)), w, p + ".norm")


def weighted_stats(x, m):
    """_compute_statistics of AttentiveStatisticsPooling (ECAPA_TDNN.py:299-304): x [B, C, L], weights m [B, 1 or C, L]
    summing to 1 over L -> (mean, std) [B, C], std = sqrt(clamp(sum m (x - mean)^2, 1e-12))."""
    mean = (m * x).sum(2)
    std = torch.sqrt((m * (x - mean.unsqueeze(2)).pow(2)).sum(2).clamp(1e-12))
    return mean, std


@torch.no_grad()
def ecapa_tdnn(w, mel, prefix="speaker_encoder.", channels=(512, 512, 512, 512, 1536), kernel_sizes=(5, 3, 3, 3, 1),
               dilations=(1, 2, 3, 4, 1), scale=8):
    """mel [B, T, n_mels] (full-length utterances: lengths = 1) -> speaker embedding [B, 1, lin_neurons]."""
    q = prefix
    x = mel.transpose(1, 2)
    xl = []
    x = _tdnn(x, w, q + "blocks.0", dilations[0])
    xl.append(x)
    for i in range(1, len(channels) - 1):
        p = q + f"blocks.{i}"
        res = x
        if (p + ".shortcut.conv.weight") in w:
            res = _conv_same(x, w[p + ".shortcut.conv.weight"], w[p + ".shortcut.conv.bias"])
        y = _tdnn(x, w, p + ".tdnn1")
        parts, prev = [], None
        for j, c in enumerate(torch.chunk(y, scale, dim=1)):                # Res2NetBlock (:179-191)
            if j == 0:
                prev = c
            elif j == 1:
                prev = _tdnn(c, w, p + f".res2net_block.blocks.{j - 1}", dilations[i])
            else:
                prev = _tdnn(c + prev, w, p + f".res2net_block.blocks.{j - 1}", dilations[i])
            parts.append(prev)
        y = torch.cat(parts, dim=1)
        y = _tdnn(y, w, p + ".tdnn2")
        s = y.mean(dim=2, keepdim=True)                                     # SEBlock (:228-242), lengths = 1
        s = F.relu(F.conv1d(s, w[p + ".se_block.conv1.conv.weight"], w[p + ".se_block.conv1.conv.bias"]))
        s = torch.sigmoid(F.conv1d(s, w[p + ".se_block.conv2.conv.weight"], w[p + ".se_block.conv2.conv.bias"]))
        x = s * y + res
        xl.append(x)
    x = _tdnn(torch.cat(xl[1:], dim=1), w, q + "mfa", dilations[-1])
    # AttentiveStatisticsPooling with global context (:282-338)
    L = x.shape[-1]
    mean, std = weighted_stats(x, torch.full((x.shape[0], 1, L), 1.0 / L, dtype=x.dtype, device=x.device))
    attn = torch.cat([x, mean.unsqueeze(2).repeat(1, 1, L), std.unsqueeze(2).repeat(1, 1, L)], dim=1)
    attn = torch.tanh(_tdnn(attn, w, q + "asp.tdnn"))
    attn = F.conv1d(attn, w[q + "asp.conv.conv.weight"], w[q + "asp.conv.conv.bias"])
    mean, std = weighted_stats(x, F.softmax(attn, dim=2))
    pooled = torch.cat((mean, std), dim=1).unsqueeze(2)
    pooled = F.batch_norm(pooled, w[q + "asp_bn.norm.running_mean"], w[q + "asp_bn.norm.running_var"],
                          w[q + "asp_bn.norm.weight"], w[q + "asp_bn.norm.bias"], training=False, eps=1e-5)
    out = F.conv1d(pooled, w[q + "fc.conv.weight"], w[q + "fc.conv.bias"])
    return out.transpose(1, 2)


@torch.no_grad()
def bigvgan_v1_forward(h, w, latent, mel_ref):
    """latent [B, T, gpt_dim], mel_ref [B, Tm, n_mels] -> wav [B, 1, T * prod(rates)]  (models.py:201-249,
    feat_upsample = False, cond_d_vector_in_each_upsampling_layer as configured)."""
    ls = h.get("snake_logscale", True)
    spk = ecapa_tdnn(w, mel_ref).transpose(1, 2)                            # [B, emb, 1]

    def act(name, x):
        return activation1d(x, w[name + ".act.alpha"], w[name + ".act.beta"], w[name + ".upsample.filter"], ls)

    x = latent.transpose(1, 2)
    x = F.conv1d(x, w["conv_pre.weight"], w["conv_pre.bias"], padding=3)
    x = x + F.conv1d(spk, w["cond_layer.weight"], w["cond_layer.bias"])
    nk = len(h["resblock_kernel_sizes"])
    for i, (u, k) in enumerate(zip(h["upsample_rates"], h["upsample_kernel_sizes"])):
        x = F.conv_transpose1d(x, w[f"ups.{i}.0.weight"], w[f"ups.{i}.0.bias"], stride=u, padding=(k - u) // 2)
        if h.get("cond_d_vector_in_each_upsampling_layer", True):
            x = x + F.conv1d(spk, w[f"conds.{i}.weight"], w[f"conds.{i}.bias"])
        xs = None
        for j, (ks, dil) in enumerate(zip(h["resblock_kernel_sizes"], h["resblock_dilation_sizes"])):
            rb = i * nk + j
            xb = x
            for mi, d in enumerate(dil):
                xt = act(f"resblocks.{rb}.activations.{2 * mi}", xb)
                xt = F.conv1d(xt, w[f"resblocks.{rb}.convs1.{mi}.weight"], w[f"resblocks.{rb}.convs1.{mi}.bias"],
                              dilation=d, padding=int((ks * d - d) / 2))
                xt = act(f"resblocks.{rb}.activations.{2 * mi + 1}", xt)
                xt = F.conv1d(xt, w[f"resblocks.{rb}.convs2.{mi}.weight"], w[f"resblocks.{rb}.convs2.{mi}.bias"],
                              padding=int((ks - 1) / 2))
                xb = xt + xb
            xs = xb if xs is None else xs + xb
        x = xs / nk
    x = act("activation_post", x)
    x = F.conv1d(x, w["conv_post.weight"], w["conv_post.bias"], padding=3)
    return torch.tanh(x)


# ------------------------------------------------------------------------------------------------
# GPT side of v1 / v1.5 (indextts/gpt/model.py).  Same GPT-2 stack and head as v2 (oracle/gpt.py); what differs:
#   get_conditioning ("conformer_perceiver")  model.py:493-503: ConformerEncoder(100-bin mel, conv2d2) -> PerceiverResampler
#                                             with 32 latents -> conds [32, D]
#   prepare_gpt_inputs                         model.py:597-660: [conds(32)][text_emb(start, text, stop) + text_pos(arange)]
#   decode positions                           model.py:139-161: with the KV cache step k>=1 sits at mel position k+1
#                                              (trap P1); WITHOUT it (infer.py:101, the CPU default) the whole suffix
#                                              [start, t1..tk] is re-embedded at positions 0..k every step
#   latents for the vocoder                    model.py:526-589 (return_latent=True): one teacher-forced pass over
#                                              [conds][start_text, text, stop_text][start_mel, codes, stop_mel],
#                                              final_norm(ln_f hidden) of the mel part, last two positions dropped
# Pinned against the reference's own v1 UnifiedVoice by oracle/make_goldens_v1.py (tests/golden/v1_gpt_small.npz).
def get_conditioning_v1(w, ccfg, mel):
    """mel [T, 100] -> conds [32, D]."""
    from oracle.emo import conformer_encode, perceiver_resample
    ctx = conformer_encode(w, ccfg, mel, prefix="conditioning_encoder.")
    return perceiver_resample(w, ccfg, ctx, prefix="perceiver_encoder.", squeeze=False)


def prepare_inputs_v1(w, conds, text_ids):
    """[conds][text_embedding(start, text.., stop) + text_pos_embedding(0..L+1)]  (model.py:597-660, batch 1, no padding)."""
    ids = torch.as_tensor(text_ids, dtype=torch.long)
    ids = ids[(ids != 0) & (ids != 1)]
    ids = F.pad(F.pad(ids, (1, 0), value=0), (0, 1), value=1)
    emb = w["text_embedding.weight"][ids] + w["text_pos_embedding.emb.weight"][: ids.shape[0]]
    return torch.cat([conds, emb], dim=0)


@torch.no_grad()
def generate_v1(oracle, prompt, max_new, repetition_penalty=10.0, kv_cache=False):
    """Greedy decode of the v1 model.  `oracle` is an oracle.gpt.GptOracle (fp32).  kv_cache=False reproduces the CPU
    default of infer.py:101: every step re-runs the whole sequence with mel positions 0..k."""
    if kv_cache:
        return oracle.generate(prompt, max_new, repetition_penalty, 0)
    w, cfg = oracle.w, oracle.cfg
    start, stop = cfg["start_mel_token"], cfg["stop_mel_token"]
    prompt = torch.as_tensor(prompt, dtype=torch.float32).to(w["mel_embedding.weight"])
    toks, codes, logits = [start], [], []
    seen = {1, start}
    for k in range(max_new):
        oracle.reset()
        t = torch.tensor(toks, device=prompt.device)
        emb = w["mel_embedding.weight"][t] + w["mel_pos_embedding.emb.weight"][: len(toks)]
        hidden = oracle.forward_rows(torch.cat([prompt, emb], 0))[-1:]
        lg = oracle.logits(hidden)[0]
        logits.append(lg.clone())
        s = lg.clone()
        idx = torch.tensor(sorted(seen), device=s.device)
        sv = s[idx]
        s[idx] = torch.where(sv < 0, sv * repetition_penalty, sv / repetition_penalty)
        tok = int(torch.argmax(s))
        codes.append(tok)
        if tok == stop:
            break
        toks.append(tok)
        seen.add(tok)
    return np.array(codes, dtype=np.int32), torch.stack(logits).cpu().numpy()


@torch.no_grad()
def latents_v1(oracle, conds, text_ids, codes):
    """UnifiedVoice.forward(..., return_latent=True) (model.py:526-589) for one utterance: final_norm(ln_f(hidden)) at the
    mel positions [start_mel, codes..., stop_mel] minus the last two -> [len(codes), D]  (what BigVGAN v1 consumes)."""
    w, cfg = oracle.w, oracle.cfg
    dev = w["mel_embedding.weight"].device
    ids = torch.as_tensor(np.asarray(text_ids), dtype=torch.long, device=dev)
    ids = F.pad(F.pad(ids, (0, 1), value=1), (1, 0), value=0)            # stop appended, then start prepended (:565-569)
    text_emb = w["text_embedding.weight"][ids] + w["text_pos_embedding.emb.weight"][: ids.shape[0]]
    mel = torch.as_tensor(np.asarray(codes), dtype=torch.long, device=dev)
    mel = F.pad(F.pad(mel, (0, 1), value=cfg["stop_mel_token"]), (1, 0), value=cfg["start_mel_token"])
    mel_emb = w["mel_embedding.weight"][mel] + w["mel_pos_embedding.emb.weight"][: mel.shape[0]]
    oracle.reset()
    hidden = oracle.forward_rows(torch.cat([conds, text_emb, mel_emb], 0))
    h = F.layer_norm(hidden, (hidden.shape[-1],), w["gpt.ln_f.weight"], w["gpt.ln_f.bias"], 1e-5)
    h = F.layer_norm(h, (h.shape[-1],), w["final_norm.weight"], w["final_norm.bias"], 1e-5)
    return h[-mel.shape[0]:][:-2]
