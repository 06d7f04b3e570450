"""GPU: the w2v-BERT 2.0 prompt encoder behind IndexTTS2.get_emb (idx_semantic_encode).

  * the relative_key flash attention alone against float64 on the same fp16 q / k / v / E, with the five query-row kinds of
    tests/test_flash_attention_gpu.py (the masked keys here are real rows that would win row kind 3 and carry v = 100);
  * the fused conv-module kernel against float64, each entry's rows between NaN rows;
  * get_emb end to end against the goldens minted from transformers, and against the float64 oracle at T = 750 (a 15 s
    prompt: 1500 fbank frames stacked in pairs; the last row masked as the extractor masks an odd frame count);
  * padding: the valid rows of each entry of a B = 2 call are bitwise equal to that entry's own B = 1 call;
  * the drop-in: a stand-in tts gets get_emb rebound, and its CUDA output matches the oracle.
End to end, the default path (fp16 GEMM operands) is held to 2e-2 and the strict fp32 path to 2e-3 max abs on outputs of
O(1), the bounds of the emotion encoder (tests/test_emo.py)."""
import math
import os
import types

import numpy as np
import pytest
import torch

from indextts_b200.dropin import SEMANTIC_LAYERS, attach_semantic
from oracle import w2v_bert
from tests import w2v_bert_refs as kr
from tests.test_flash_attention_gpu import make_qkv

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
L, R = 64, 8
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def relkey_case(B, H, T, lens, seed):
    q, k, v = (x.astype(np.float64) for x in make_qkv(B, H, T, seed))
    rng = np.random.default_rng(seed + 1)
    E = 0.1 * rng.standard_normal((L + R + 1, 64))
    kind = np.arange(T) % 5
    for bh in range(B * H):
        n = lens[bh // H]
        klast = k[bh, n - 1]
        q[bh, kind == 1] = 40.0 * klast / (klast ** 2).sum()             # score ~40 with the last valid key
        u = -2.0 * q[bh, kind == 3].mean(axis=0) if (kind == 3).any() else np.zeros(64)
        k[bh, n:] = -8.0 * u                                             # masked keys would win row kind 3 ...
        v[bh, n:] = 100.0                                                # ... and pull the output far off
    return tuple(x.astype(np.float16) for x in (q, k, v, E))


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("T", [1, 2, 7, 72, 127, 128, 129, 750, 1741])
def test_relkey_flash_attention(engine, T, B):
    H = 16
    lens = [max(1, T - 1), max(1, (2 * T) // 3)][:B]
    q, k, v, E = relkey_case(B, H, T, lens, seed=T * 13 + B)
    ref, vmag, smag = kr.relkey_attention(q, k, v, E, lens, H, L, R)
    # fp16 rounding of P (1e-3 of the weighted |v|), the fp32 sums of q.k and q.E in the exponent, the fp16 output
    bound = vmag * (1e-3 + 4 * math.log(2.0) * 64 * U * smag) + 2.0 ** -11 * np.abs(ref)
    to_out = lambda x: x.reshape(B, H, T, 64).transpose(0, 2, 1, 3).reshape(B, T, H * 64)
    ref, bound = to_out(ref), to_out(bound)
    got = engine.debug_flash_attention_relkey(q, k, v, E, lens, B, H, L, R).astype(np.float64)
    assert np.all(np.isfinite(got))
    err = np.abs(got - ref)
    print(f"relkey T={T} B={B} lens={lens}: max err {err.max():.2e}, max err / bound {(err / bound).max():.3f}")
    assert np.all(err <= bound)


def conv_module_ref(x, lens, dw, lw, lb, eps):
    x = x.astype(np.float64)
    B, T, C2 = x.shape
    C, K = C2 // 2, dw.shape[1]
    g = x[..., :C] / (1.0 + np.exp(-x[..., C:]))
    for b in range(B):
        g[b, lens[b]:] = 0.0
    gp = np.concatenate([np.zeros((B, K - 1, C)), g], axis=1)
    y = sum(gp[:, k:k + T] * dw[:, k] for k in range(K))
    y = (y - y.mean(-1, keepdims=True)) / np.sqrt(y.var(-1, keepdims=True) + eps) * lw + lb
    return y / (1.0 + np.exp(-y))


@pytest.mark.parametrize("C,K,T,lens", [(1024, 31, 75, [74, 40]), (128, 31, 9, [9, 1]), (256, 15, 130, [130])])
def test_conv_module_kernel(engine, C, K, T, lens):
    rng = np.random.default_rng(C + K + T)
    B = len(lens)
    x = rng.standard_normal((B, T, 2 * C)).astype(np.float32)
    dw = (rng.standard_normal((C, K)) / math.sqrt(K)).astype(np.float32)
    lw = (1 + 0.1 * rng.standard_normal(C)).astype(np.float32)
    lb = (0.1 * rng.standard_normal(C)).astype(np.float32)
    ref = conv_module_ref(x, lens, dw.astype(np.float64), lw, lb, 1e-5)
    out, out16 = engine.debug_conv_module(x, lens, dw, lw, lb, 1e-5)
    e32 = np.abs(out - ref).max()
    e16 = (np.abs(out16.astype(np.float64) - ref) - 2.0 ** -11 * np.abs(ref)).max()
    print(f"conv module C={C} K={K} T={T} lens={lens}: fp32 max err {e32:.2e}, fp16 max err beyond rounding {e16:.2e}")
    assert np.all(np.isfinite(out)) and e32 <= 1e-4 and e16 <= 1e-4


def load(engine, cfg, sd):
    engine.load_state_dict("semantic.", sd)
    engine.semantic_init(cfg)


def run_both(engine, x, mask):
    out = engine.get_emb(x, mask)
    engine.set_option("gemm_backend", 1)
    try:
        out32 = engine.get_emb(x, mask)
    finally:
        engine.set_option("gemm_backend", 0)
    return out, out32


@pytest.mark.parametrize("name", ["w2v_small.npz", "w2v_full.npz"])
def test_get_emb_matches_golden(engine, name):
    z = np.load(os.path.join(GOLD, name))
    cfg = dict(w2v_bert.FULL, hidden=int(z["hidden"]), heads=int(z["heads"]), ffn=int(z["ffn"]), layers=int(z["layers"]))
    load(engine, cfg, w2v_bert.make_weights(cfg, int(z["seed"]), n_layers=int(z["model_layers"])))
    out, out32 = run_both(engine, z["input_features"], z["attention_mask"])
    e, e32 = np.abs(out - z["out"]).max(), np.abs(out32 - z["out"]).max()
    print(f"{name}: default max abs {e:.2e}, strict fp32 max abs {e32:.2e}")
    assert e <= 2e-2 and e32 <= 2e-3


@pytest.fixture(scope="module")
def full_case():
    cfg = w2v_bert.FULL
    sd = w2v_bert.make_weights(cfg, 2024)
    g = torch.Generator().manual_seed(7)
    T = 750
    x = torch.randn(2, T, cfg["feat_dim"], generator=g)
    lens = torch.tensor([T - 1, 413])
    mask = (torch.arange(T)[None, :] < lens[:, None]).to(torch.int32)
    ref = w2v_bert.get_emb(sd, cfg, x.double().cuda(), mask.cuda()).cpu().numpy()
    return cfg, sd, x.numpy(), mask.numpy(), ref


def test_get_emb_matches_oracle_15s(engine, full_case):
    cfg, sd, x, mask, ref = full_case
    load(engine, cfg, sd)
    out, out32 = run_both(engine, x[:1], mask[:1])
    e, e32 = np.abs(out - ref[:1]).max(), np.abs(out32 - ref[:1]).max()
    print(f"T=750 (749 valid): default max abs {e:.2e}, strict fp32 max abs {e32:.2e}, output rms {np.sqrt((ref ** 2).mean()):.2f}")
    assert e <= 2e-2 and e32 <= 2e-3


def test_padding_is_bitwise_solo(engine, full_case):
    cfg, sd, x, mask, ref = full_case
    load(engine, cfg, sd)
    both = engine.get_emb(x, mask)
    n = [int(m.sum()) for m in mask]
    for b in range(2):
        solo = engine.get_emb(np.ascontiguousarray(x[b:b + 1, :n[b]]), np.ones((1, n[b]), np.int32))
        assert np.array_equal(both[b, :n[b]].view(np.uint32), solo[0].view(np.uint32)), b
    e = np.abs(both - ref).max()
    print(f"B=2, lens {n}: default max abs vs oracle {e:.2e} (all rows)")
    assert e <= 2e-2


def test_get_emb_refuses_bad_masks(engine):
    cfg = w2v_bert.SMALL
    load(engine, cfg, w2v_bert.make_weights(cfg, 5))
    x = np.zeros((1, 4, cfg["feat_dim"]), np.float32)
    with pytest.raises(RuntimeError):
        engine.get_emb(x, np.array([[1, 0, 1, 1]]))
    with pytest.raises(RuntimeError):
        engine.get_emb(x, np.zeros((1, 4), np.int32))


def test_dropin_rebinds_get_emb(engine):
    cfg = dict(w2v_bert.SMALL, layers=SEMANTIC_LAYERS)
    sd = w2v_bert.make_weights(cfg, 11, n_layers=SEMANTIC_LAYERS + 1)
    mean, std = sd.pop("semantic_mean"), sd.pop("semantic_std")

    class _Model:
        config = types.SimpleNamespace(num_attention_heads=cfg["heads"], left_max_position_embeddings=L,
                                       right_max_position_embeddings=R, layer_norm_eps=cfg["eps"])

        def state_dict(self):
            return sd

    tts = types.SimpleNamespace(semantic_model=_Model(), semantic_mean=mean, semantic_std=std)
    attach_semantic(tts, engine)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1, 61, cfg["feat_dim"], generator=g).cuda()
    mask = torch.ones(1, 61, dtype=torch.int32).cuda()
    mask[0, -1] = 0
    out = tts.get_emb(x, mask)
    assert isinstance(out, torch.Tensor) and out.is_cuda and out.shape == (1, 61, cfg["hidden"])
    ref = w2v_bert.get_emb(dict(sd, semantic_mean=mean, semantic_std=std), cfg, x.double(), mask)
    e = float((out.double() - ref).abs().max())
    print(f"drop-in get_emb: default max abs {e:.2e}")
    assert e <= 2e-2
