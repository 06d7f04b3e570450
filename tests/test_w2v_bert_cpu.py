"""CPU: the w2v-BERT 2.0 oracle behind get_emb (oracle/w2v_bert.py) against the goldens minted from transformers'
Wav2Vec2BertModel (oracle/make_goldens_w2v.py) and against transformers directly; the float64 relative-key attention
reference of the encoder's flash kernel (tests/w2v_bert_refs.py); and the constants of the reference's get_emb that the
drop-in relies on."""
import ast
import importlib.util
import math
import os

import numpy as np
import pytest
import torch

from oracle import w2v_bert
from oracle.refimport import REF
from tests import w2v_bert_refs as kr

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def golden(name):
    z = np.load(os.path.join(GOLD, name))
    cfg = dict(w2v_bert.FULL, hidden=int(z["hidden"]), heads=int(z["heads"]), ffn=int(z["ffn"]), layers=int(z["layers"]))
    sd = w2v_bert.make_weights(cfg, int(z["seed"]), n_layers=int(z["model_layers"]))
    return z, cfg, sd


@pytest.mark.parametrize("name", ["w2v_small.npz", "w2v_full.npz"])
def test_oracle_matches_golden(name):
    z, cfg, sd = golden(name)
    got = w2v_bert.get_emb(sd, cfg, torch.from_numpy(z["input_features"]).double(), torch.from_numpy(z["attention_mask"]))
    err = float((got.float() - torch.from_numpy(z["out"])).abs().max())
    print(f"{name}: oracle vs golden max abs {err:.2e}")
    assert err <= 1e-4


def test_oracle_matches_transformers():
    if importlib.util.find_spec("transformers") is None:
        pytest.skip("transformers is not installed")
    from oracle.make_goldens_w2v import hf_model
    cfg = w2v_bert.SMALL
    sd = w2v_bert.make_weights(cfg, 99, n_layers=cfg["layers"])
    m = hf_model(cfg, cfg["layers"], sd).double()
    g = torch.Generator().manual_seed(5)
    feats = torch.randn(3, 41, cfg["feat_dim"], generator=g, dtype=torch.float64)
    mask = (torch.arange(41)[None, :] < torch.tensor([41, 20, 1])[:, None]).to(torch.int32)
    with torch.no_grad():
        hs = m(input_features=feats, attention_mask=mask, output_hidden_states=True).hidden_states[cfg["layers"]]
    ref = (hs - sd["semantic_mean"].double()) / sd["semantic_std"].double()
    err = float((w2v_bert.get_emb(sd, cfg, feats, mask) - ref).abs().max())
    print(f"oracle vs transformers (float64) max abs {err:.2e}")
    assert err <= 1e-9


def test_relkey_reference_matches_direct_formula():
    """w2v_bert_refs.relkey_attention against the score formula of modeling_wav2vec2_bert.py:305-326 written out per element."""
    rng = np.random.default_rng(3)
    B, H, T, L, R = 2, 2, 19, 5, 3
    q, k, v = (rng.standard_normal((B * H, T, 64)) for _ in range(3))
    E = rng.standard_normal((L + R + 1, 64))
    lens = [19, 11]
    out, vmag, smag = kr.relkey_attention(q, k, v, E, lens, H, L, R)
    for bh in range(B * H):
        n = lens[bh // H]
        for i in range(T):
            s = np.array([q[bh, i] @ k[bh, j] + q[bh, i] @ E[min(max(j - i, -L), R) + L] for j in range(n)]) * math.log(2)
            p = np.exp(s - s.max())
            np.testing.assert_allclose(out[bh, i], p @ v[bh, :n] / p.sum(), rtol=1e-12, atol=1e-12)
            assert vmag[bh, i].min() > 0 and smag[bh, i, 0] > 0


def _reference_get_emb():
    path = os.path.join(REF, "indextts", "infer_v2_5.py")
    if not os.path.exists(path):
        pytest.skip("the reference tree is not present")
    tree = ast.parse(open(path, encoding="utf-8").read())
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "IndexTTS2")
    return next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "get_emb")


def test_reference_get_emb_reads_hidden_state_17_and_normalises():
    from indextts_b200.dropin import SEMANTIC_LAYERS
    fn = _reference_get_emb()
    idx = [n.slice.value for n in ast.walk(fn) if isinstance(n, ast.Subscript)
           and isinstance(n.value, ast.Attribute) and n.value.attr == "hidden_states" and isinstance(n.slice, ast.Constant)]
    assert idx == [SEMANTIC_LAYERS]
    norm = [ast.unparse(n) for n in ast.walk(fn) if isinstance(n, ast.BinOp) and isinstance(n.op, ast.Div)]
    assert norm == ["(feat - self.semantic_mean) / self.semantic_std"]
