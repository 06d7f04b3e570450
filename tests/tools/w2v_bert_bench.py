"""Time one get_emb call (the w2v-BERT 2.0 prompt encoder, 17 layers) at T = 750 rows (a 15 s prompt) for two
implementations in the same process, alternating, after a warm-up of each:

  engine   idx_semantic_encode (default path: fp16 GEMM operands, the relative_key wgmma flash attention)
  torch    the fp32 PyTorch path on the same GPU: transformers' Wav2Vec2BertModel when it is importable (as the reference
           runs it), else the plain-torch oracle (oracle/w2v_bert.py)

    python tests/tools/w2v_bert_bench.py OUT_DIR [--reps 20] [--T 750]

Prints ms per call (median over the timed calls), TFLOP/s over the algorithmic FLOP (GEMMs 2 T (4 C F + 7 C^2) and
attention 4 T^2 C per layer), and the card's name, power limit and max SM clock; writes OUT_DIR/w2v_bert_bench.json.
Weights are seeded (oracle.w2v_bert.make_weights); the two outputs are compared as a sanity check."""
import argparse
import importlib.util
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from indextts_b200.engine import Engine  # noqa: E402
from oracle import w2v_bert  # noqa: E402


def flop(cfg, T):
    C, Ff = cfg["hidden"], cfg["ffn"]
    gemm = 2.0 * T * (4 * C * Ff + 7 * C * C) + 2.0 * T * cfg["feat_dim"] * C / cfg["layers"]
    attn = 4.0 * T * T * C
    return cfg["layers"] * (gemm + attn)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, clk = (s.strip() for s in q.split(","))
        return {"name": name, "power_limit": pl, "max_sm_clock": clk}
    except Exception as ex:      # the measurement itself does not depend on it
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unknown ({ex})", "max_sm_clock": "unknown"}


def torch_impl(cfg, sd, dev):
    if importlib.util.find_spec("transformers") is not None:
        from oracle.make_goldens_w2v import hf_model
        m = hf_model(cfg, cfg["layers"], sd).to(dev)
        mean, std = sd["semantic_mean"].to(dev), sd["semantic_std"].to(dev)

        def run(x, mask):
            with torch.no_grad():
                hs = m(input_features=x, attention_mask=mask, output_hidden_states=True).hidden_states[cfg["layers"]]
                return (hs - mean) / std
        return "transformers fp32", run
    sdd = {k: v.to(dev) for k, v in sd.items()}

    def run(x, mask):
        with torch.no_grad():
            return w2v_bert.get_emb(sdd, cfg, x, mask)
    return "oracle fp32", run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--T", type=int, default=750)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU and has no CPU fallback")
    os.makedirs(a.out_dir, exist_ok=True)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = w2v_bert.FULL
    sd = w2v_bert.make_weights(cfg, 2024)
    dev = torch.device("cuda", 0)
    T = a.T
    x = torch.randn(1, T, cfg["feat_dim"], generator=torch.Generator().manual_seed(1)).to(dev)
    mask = torch.ones(1, T, dtype=torch.int32, device=dev)
    mask[0, -1] = 0
    eng = Engine(0)
    eng.load_state_dict("semantic.", sd)
    eng.semantic_init(cfg)
    tname, trun = torch_impl(cfg, sd, dev)
    impls = {"engine": lambda: eng.get_emb(x, mask), "torch": lambda: trun(x, mask)}
    outs = {k: f() for k, f in impls.items()}               # warm-up (module load, allocator, algorithm choice)
    for f in impls.values():
        for _ in range(2):
            f()
    torch.cuda.synchronize()
    times = {k: [] for k in impls}
    for _ in range(a.reps):
        for k, f in impls.items():                          # alternating: both see the same clock / neighbours
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            f()
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) * 1e3)
    fl = flop(cfg, T)
    diff = float((outs["engine"] - outs["torch"]).abs().max())
    res = {"T": T, "layers": cfg["layers"], "gflop": fl / 1e9, "torch_impl": tname, "card": card(),
           "max_abs_engine_vs_torch": diff}
    for k, v in times.items():
        ms = float(np.median(v))
        res[k] = {"ms_median": ms, "ms_min": float(np.min(v)), "ms_max": float(np.max(v)), "tflops": fl / (ms * 1e-3) / 1e12}
    res["speedup"] = res["torch"]["ms_median"] / res["engine"]["ms_median"]
    print(json.dumps(res, indent=1))
    with open(os.path.join(a.out_dir, "w2v_bert_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
