"""CPU restatement of the IndexTTS v2/v2.5 GPT speech-token path.

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  The product path (index-tts_b200/) never imports it.

Parity status: PINNED against the reference itself.  The reference's own tests pin no numbers for
this path (SURVEY.md §4, §8c), so the restatement is checked against outputs of the reference's own
`UnifiedVoice.inference_speech` (gpt/model_v2.py:716-825: its prepare_gpt_inputs, vendored GPT2 blocks,
vendored generate()/_beam_search and BeamSearchScorer) run on CPU in this container with the same
seeded weights — oracle/make_goldens_gpt_ref.py → tests/golden/gpt_ref_wrapper.npz: prompt embeddings,
greedy tokens and logits (6.4e-6), plain beam search, beam-sample with the RNG contract substituted.
In addition the blocks are checked against stock `transformers.GPT2Model` in fp32 and under CPU
autocast bf16 (oracle/validate_gpt_vs_hf.py → tests/golden/gpt_small.npz), which is what anchors the
bf16 rounding-point model.

What is restated (reference file:line):
  prepare_gpt_inputs                       indextts/gpt/model_v2.py:648-714 (+ :754-768 conds)
  GPT2InferenceModel.forward               indextts/gpt/model_v2.py:121-198
      prefill: cat(prompt_emb, mel_emb[start] + mel_pos[0])             :146-156, :244-256
      cached step k>=1: mel_emb[tok] + mel_pos[mask_len - S] = pos k+1  :158-161   (trap P1)
  GPT2Block / Attention / MLP              indextts/gpt/transformers_gpt2.py:189-227,571-667
      ln eps 1e-5, Conv1D weight [in,out], gelu_new                     (trap P4)
  ln_f then lm_head = Sequential(final_norm, mel_head)  model_v2.py:54,186 (trap P3)
  greedy _sample + RepetitionPenalty over ALL input_ids incl. the fake prompt [1..1, 8192]
      indextts/gpt/transformers_generation_utils.py:3196-3265; model_v2.py:705-713 (trap P2)
  logits upcast to fp32 before processors   transformers_generation_utils.py:3220 (trap P5)

bf16 policy (`bf16=True`, the reference's use_bf16 path: infer_v2_5.py:143-146,758): weights
are bf16 values; every tensor autocast materialises in bf16 is rounded to bf16 (after each
Conv1D / Linear, after every elementwise op of NewGELUActivation); LayerNorm runs
fp32-in/fp32-out; attention keeps fp32 scores/softmax and rounds its output.
Trap P12 (found while pinning against HF): the RESIDUAL STREAM IS FP32 even on the bf16 path —
`null_position_embeddings` returns fp32 zeros (model_v2.py:23-24), GPT2Model adds them to the
bf16 inputs_embeds (transformers_gpt2.py:1037-1038) and type promotion makes hidden_states
fp32; every later `attn_output + residual` (:639, :664) adds a bf16 branch to the fp32 stream
and stays fp32.  So residual adds are NOT rounded; only the branch outputs are.
"""
import math

import numpy as np
import torch


from indextts_b200.synth import gpt_config, make_gpt_weights, r16  # noqa: F401,E402






def prepare_gpt_inputs(w, style, emo_vec, text_ids, lang, bf16=True):
    """[cond(3)][start_text, text…, stop_text] embeddings (model_v2.py:648-714, :754-768).
    style [192], emo_vec [D], text_ids 1-D ints (start/stop tokens inside are dropped, :674)."""
    rr = r16 if bf16 else (lambda x: x)
    style = torch.as_tensor(style, dtype=torch.float32).reshape(-1)
    emo_vec = torch.as_tensor(emo_vec, dtype=torch.float32).reshape(-1)
    ids = torch.as_tensor(np.asarray(text_ids), dtype=torch.long).reshape(-1)
    ids = ids[(ids != 0) & (ids != 1)]
    spk = rr(rr(style) @ w["spk_emb_proj.weight"].t() + w["spk_emb_proj.bias"])  # :754
    cond0 = rr(spk + emo_vec)                                                      # :768
    D = cond0.shape[0]
    ids = torch.cat([torch.tensor([0]), ids, torch.tensor([1])])                   # :676-677
    pos = torch.arange(ids.shape[0])
    temb = rr(w["text_embedding.weight"][ids] + w["text_pos_embedding.emb.weight"][pos])  # :679
    if lang is not None:
        temb = rr(temb + w["lang_embedding.weight"][lang])                         # :681
    return torch.cat([cond0[None], torch.zeros(2, D), temb], dim=0)


def _gelu_new(x, bf16):
    if not bf16:
        return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * torch.pow(x, 3.0))))
    # NewGELUActivation on a bf16 tensor: every op materialises a bf16 tensor
    t1 = r16(x * x * x)
    t2 = r16(0.044715 * t1)
    t3 = r16(x + t2)
    t4 = r16(math.sqrt(2.0 / math.pi) * t3)
    t5 = r16(torch.tanh(t4))
    t6 = r16(1.0 + t5)
    t7 = r16(0.5 * x)
    return r16(t7 * t6)


def _ln(x, w, b):
    return torch.nn.functional.layer_norm(x, (x.shape[-1],), w, b, 1e-5)


def philox4x32_10(seed, c0, c1):
    """Philox4x32-10 with counter (c0, c1, 0, 0) and 64-bit key `seed` — the device sampler's RNG."""
    M0, M1 = 0xD2511F53, 0xCD9E8D57
    k0, k1 = seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF
    x0, x1, x2, x3 = c0 & 0xFFFFFFFF, c1 & 0xFFFFFFFF, 0, 0
    for _ in range(10):
        p0, p1 = M0 * x0, M1 * x2
        x0, x1, x2, x3 = ((p1 >> 32) ^ x1 ^ k0) & 0xFFFFFFFF, p1 & 0xFFFFFFFF, ((p0 >> 32) ^ x3 ^ k1) & 0xFFFFFFFF, p0 & 0xFFFFFFFF
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return x0, x1, x2, x3


CMAX = 128     # candidate slots of the device samplers (csrc/gpt_decode.cu)


def sample_token(scores, top_k, top_p, seed, step, seq):
    """Temperature is already applied.  TopK (1 <= top_k <= CMAX = 128 — the device sampler refuses anything else; ties at
    the k-th value kept, and more than CMAX of them raise ValueError, as the device refuses them) → TopP → multinomial by
    inverse CDF over the descending candidates with one Philox draw (transformers logits_process order,
    transformers_generation_utils.py:1035-1047; RNG contract of the device sampler)."""
    s = np.asarray(scores, dtype=np.float32)
    order = np.lexsort((np.arange(len(s)), -s))            # descending, lowest index first among ties
    kk = min(top_k, CMAX) if top_k > 0 else CMAX      # top_k = 0: warper disabled (the device refuses it; kept for the checker's own tests)
    cand = []
    kth = None
    for idx in order:
        if not np.isfinite(s[idx]):
            break
        if len(cand) >= CMAX:
            if top_k > 0 and s[idx] == kth:
                raise ValueError("more than 128 tokens tie at the top-k boundary")
            break
        if len(cand) < kk:
            cand.append(int(idx))
            kth = s[idx]
        elif s[idx] == kth:
            cand.append(int(idx))
        else:
            break
    cv = np.exp((s[cand] - s[cand[0]]).astype(np.float32)).astype(np.float32)
    tot = np.float32(0)
    for v in cv:
        tot = np.float32(tot + v)
    keep = len(cand)
    if top_p < 1.0:
        tail = np.float32(0)
        for i in range(len(cand) - 1, 0, -1):
            tail = np.float32(tail + np.float32(cv[i] / tot))
            if tail <= np.float32(1.0 - top_p):
                keep = i
            else:
                break
    kt = np.float32(0)
    for i in range(keep):
        kt = np.float32(kt + cv[i])
    r0 = philox4x32_10(seed, step, seq)[0]
    u = np.float32(np.float32(r0 >> 8) * np.float32(1.0 / 16777216.0) * kt)
    acc = np.float32(0)
    pick = keep - 1
    for i in range(keep):
        acc = np.float32(acc + cv[i])
        if u < acc:
            pick = i
            break
    return cand[pick], cand[:keep]


class GptOracle:
    def __init__(self, cfg, weights, bf16=True):
        self.cfg, self.w, self.bf16 = cfg, weights, bf16
        self.rr = r16 if bf16 else (lambda x: x)
        self.reset()

    def reset(self):
        L = self.cfg["layers"]
        self.k = [None] * L
        self.v = [None] * L

    def forward_rows(self, x):
        """x [T, D] new positions (appended to the KV cache, causal) → final hidden [T, D]."""
        cfg, w, rr = self.cfg, self.w, self.rr
        H = cfg["heads"]
        T, D = x.shape
        hd = D // H
        for l in range(cfg["layers"]):
            p = f"gpt.h.{l}."
            h = _ln(x, w[p + "ln_1.weight"], w[p + "ln_1.bias"])
            qkv = rr(rr(h) @ w[p + "attn.c_attn.weight"] + w[p + "attn.c_attn.bias"])
            q, k, v = qkv.split(D, dim=-1)
            self.k[l] = k if self.k[l] is None else torch.cat([self.k[l], k], 0)
            self.v[l] = v if self.v[l] is None else torch.cat([self.v[l], v], 0)
            K, Vv = self.k[l], self.v[l]
            S = K.shape[0]
            qh = q.view(T, H, hd).transpose(0, 1)
            kh = K.view(S, H, hd).transpose(0, 1)
            vh = Vv.view(S, H, hd).transpose(0, 1)
            sc = (qh @ kh.transpose(1, 2)) / math.sqrt(hd)          # transformers_gpt2.py:199-203
            qpos = torch.arange(S - T, S, device=x.device)[:, None]
            mask = torch.arange(S, device=x.device)[None, :] <= qpos
            sc = sc.masked_fill(~mask[None], float("-inf"))
            a = rr((torch.softmax(sc, dim=-1) @ vh).transpose(0, 1).reshape(T, D))
            o = rr(a @ w[p + "attn.c_proj.weight"] + w[p + "attn.c_proj.bias"])
            x = x + o            # residual stream stays fp32 (trap P12, see module docstring)
            h = _ln(x, w[p + "ln_2.weight"], w[p + "ln_2.bias"])
            f = rr(rr(h) @ w[p + "mlp.c_fc.weight"] + w[p + "mlp.c_fc.bias"])
            f = _gelu_new(f, self.bf16)
            m = rr(f @ w[p + "mlp.c_proj.weight"] + w[p + "mlp.c_proj.bias"])
            x = x + m
        return x

    def logits(self, hidden):
        w, rr = self.w, self.rr
        h = _ln(hidden, w["gpt.ln_f.weight"], w["gpt.ln_f.bias"])            # GPT2Model ln_f
        h = _ln(h, w["final_norm.weight"], w["final_norm.bias"])              # lm_head[0]  (P3)
        return rr(rr(h) @ w["mel_head.weight"].t() + w["mel_head.bias"])      # .float()    (P5)

    @torch.no_grad()
    def generate(self, prompt_emb, max_new_tokens, repetition_penalty=10.0, forbid_stop_before=0,
                 forced=None, do_sample=False, top_k=0, top_p=1.0, temperature=1.0, seed=0, seq=0):
        """Greedy (or sampled) decode. Returns (codes incl. stop token, raw logits [n, V])."""
        cfg, w, rr = self.cfg, self.w, self.rr
        start, stop = cfg["start_mel_token"], cfg["stop_mel_token"]
        self.reset()
        prompt_emb = torch.as_tensor(prompt_emb, dtype=torch.float32).to(w["mel_embedding.weight"])
        first = rr(w["mel_embedding.weight"][start] + w["mel_pos_embedding.emb.weight"][0])
        x = torch.cat([prompt_emb, first[None]], dim=0)                       # model_v2.py:146-156
        hidden = self.forward_rows(x)[-1:]
        seen = {1, start}                                                     # fake ids (P2)
        codes, all_logits = [], []
        for k in range(max_new_tokens):
            lg = self.logits(hidden)[0]
            all_logits.append(lg.clone())
            s = lg.clone()
            idx = torch.tensor(sorted(seen), device=s.device)
            sv = s[idx]
            s[idx] = torch.where(sv < 0, sv * repetition_penalty, sv / repetition_penalty)
            if k < forbid_stop_before:
                s[stop] = float("-inf")
            if do_sample:
                sc = (s.cpu().numpy().astype(np.float32) * np.float32(1.0 / temperature)).astype(np.float32)
                tok, _ = sample_token(sc, top_k, top_p, seed, k, seq)
            else:
                tok = int(torch.argmax(s))  # first maximal index on CPU
            codes.append(tok)
            feed = tok if forced is None else int(forced[k])
            if forced is None and tok == stop:
                break
            if k + 1 >= max_new_tokens:
                break
            seen.add(feed)
            emb = rr(w["mel_embedding.weight"][feed] + w["mel_pos_embedding.emb.weight"][k + 2])
            hidden = self.forward_rows(emb[None])                             # position k+2 (P1)
        return np.array(codes, dtype=np.int32), torch.stack(all_logits).cpu().numpy()
