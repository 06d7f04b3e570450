"""Weight waits of the batch-1 decode kernel from the stamps `tests.tools.gpt_fine` saves (gpt_fine.npy: [CTAs][64],
globaltimer ns in slots 0-31, clock64 in 32-63; middle layer of the last step).  For each weight phase of the layer:
"weights ready" (the phase's mbarrier wait has returned, CTA thread 0) minus the point the phase's input was ready (its
hand-over poll or LayerNorm done), over all CTAs.  The two stamps are ~300 cycles apart when the weights were already
there (a refill call, the xs stores and the stamp itself sit between them).
    python -m tests.tools.gpt_ring_wait STAMPS.npy [MORE.npy ...]"""
import sys

import numpy as np

PHASES = [("QKV", 2, 3, "LN done"), ("O-proj", 11, 12, "o polled"), ("FC", 17, 18, "LN done"), ("PROJ", 22, 23, "f polled")]


def table(f):
    lines = [f"{'phase':8s} {'from':9s} {'cycles med':>10} {'p90':>6} {'max':>6} | {'ns med':>6} {'p90':>6}"]
    for name, a, b, what in PHASES:
        c = f[:, 32 + b] - f[:, 32 + a]
        t = f[:, b] - f[:, a]
        lines.append(f"{name:8s} {what:9s} {np.median(c):10.0f} {np.percentile(c, 90):6.0f} {c.max():6.0f} | "
                     f"{np.median(t):6.0f} {np.percentile(t, 90):6.0f}")
    step = f[:, 26] - f[:, 0]
    lines.append(f"layer (start -> PROJ epilogue done): {np.median(step) / 1000:.2f} us median over CTAs")
    return "\n".join(lines)


def main():
    for path in sys.argv[1:]:
        print(f"== {path}")
        print(table(np.load(path).astype(np.float64)))


if __name__ == "__main__":
    main()
