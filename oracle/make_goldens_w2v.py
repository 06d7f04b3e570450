"""Mint tests/golden/w2v_{small,full}.npz from transformers' Wav2Vec2BertModel with seeded weights, by running the body of
the reference's IndexTTS2.get_emb (indextts/infer_v2_5.py:281-290, read with `ast`) on a stand-in `self`.

    python -m oracle.make_goldens_w2v            (build container: needs transformers and the reference tree)

Each file stores the seed, the model's layer count (the weights are regenerated from both by oracle.w2v_bert.make_weights),
the hidden_states index get_emb reads, input_features, attention_mask and the output.
"""
import ast
import os
import types

import numpy as np
import torch

from oracle import w2v_bert
from oracle.refimport import REF

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def reference_get_emb(layer_index):
    """IndexTTS2.get_emb as written in the reference, with its hidden_states index replaced by layer_index."""
    src = open(os.path.join(REF, "indextts", "infer_v2_5.py"), encoding="utf-8").read()
    cls = next(n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == "IndexTTS2")
    fn = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "get_emb")

    class Index(ast.NodeTransformer):
        def visit_Subscript(self, node):
            self.generic_visit(node)
            if isinstance(node.slice, ast.Constant) and node.slice.value == 17:
                node.slice = ast.Constant(layer_index)
            return node
    fn = ast.fix_missing_locations(Index().visit(fn))
    ns = {"torch": torch}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), "infer_v2_5.py", "exec"), ns)
    return ns["get_emb"]


def hf_model(cfg, model_layers, sd):
    from transformers import Wav2Vec2BertConfig, Wav2Vec2BertModel
    hc = Wav2Vec2BertConfig(hidden_size=cfg["hidden"], num_hidden_layers=model_layers, num_attention_heads=cfg["heads"],
                            intermediate_size=cfg["ffn"], feature_projection_input_dim=cfg["feat_dim"], hidden_act="swish",
                            position_embeddings_type="relative_key", left_max_position_embeddings=cfg["left_max"],
                            right_max_position_embeddings=cfg["right_max"], conv_depthwise_kernel_size=cfg["conv_kernel"],
                            layer_norm_eps=cfg["eps"], add_adapter=False)
    m = Wav2Vec2BertModel(hc).eval()
    missing, _ = m.load_state_dict({k: v for k, v in sd.items() if not k.startswith("semantic_")}, strict=False)
    assert all(k == "masked_spec_embed" for k in missing), missing
    return m


def mint(name, cfg, model_layers, seed, lens, T):
    sd = w2v_bert.make_weights(cfg, seed, n_layers=model_layers)
    g = torch.Generator().manual_seed(seed + 1)
    feats = torch.randn(len(lens), T, cfg["feat_dim"], generator=g)
    mask = (torch.arange(T)[None, :] < torch.tensor(lens)[:, None]).to(torch.int32)
    me = types.SimpleNamespace(semantic_model=hf_model(cfg, model_layers, sd), semantic_mean=sd["semantic_mean"],
                               semantic_std=sd["semantic_std"])
    out = reference_get_emb(cfg["layers"])(me, feats, mask)
    ours = w2v_bert.get_emb(sd, cfg, feats.double(), mask).float()
    print(name, "oracle vs HF max abs", float((ours - out).abs().max()), "output rms", float(out.pow(2).mean().sqrt()))
    np.savez_compressed(os.path.join(OUT, name), seed=seed, model_layers=model_layers, layers=cfg["layers"],
                        hidden=cfg["hidden"], heads=cfg["heads"], ffn=cfg["ffn"], input_features=feats.numpy(),
                        attention_mask=mask.numpy(), out=out.numpy())


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count() or 1)
    mint("w2v_small.npz", w2v_bert.SMALL, 3, 1234, [50, 37], 50)
    mint("w2v_full.npz", w2v_bert.FULL, 17, 4321, [74], 75)
