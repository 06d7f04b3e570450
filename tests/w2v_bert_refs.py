"""Float64 reference of the w2v-BERT encoder's attention kernel (the RELKEY mode of fa_wgmma_kernel) on its exact inputs."""
import math

import numpy as np


def relkey_attention(q, k, v, E, lens, H, left, right):
    """The w2v-BERT encoder's attention (relative_key positions, key-length mask) on the wgmma kernel's exact inputs, float64:
    q (scaled by log2(e) / 8), k, v [B*H][T][64], E [left + right + 1][64] (the fp16 values the kernel reads), lens [B].
    Weights p_ij = 2^(q_i . k_j + q_i . E[clamp(j - i, -left, right) + left]) over the keys j < lens[b].  Returns
    (out, vmag, smag) [B*H][T][64] / [B*H][T][1]: vmag = sum_j p_ij |v_j| / sum_j p_ij, the scale of an error in the
    weights; smag = max_j of sum_d |q_id| (|k_jd| + |E_d|), the scale of the fp32 summation error of a score."""
    q, k, v, E = (np.asarray(x, np.float64) for x in (q, k, v, E))
    BH, T, _ = q.shape
    pos = np.arange(T)
    idx = np.clip(pos[None, :] - pos[:, None], -left, right) + left              # [T(i)][T(j)] row of E
    out, vmag, smag = np.empty_like(q), np.empty_like(q), np.empty((BH, T, 1))
    for i in range(BH):
        n = int(lens[i // H])
        s = (q[i] @ k[i, :n].T + np.take_along_axis(q[i] @ E.T, idx[:, :n], axis=1)) * math.log(2.0)
        p = np.exp(s - s.max(axis=1, keepdims=True))
        l = p.sum(axis=1, keepdims=True)
        out[i] = (p @ v[i, :n]) / l
        vmag[i] = (p @ np.abs(v[i, :n])) / l
        smag[i] = (np.abs(q[i]) @ (np.abs(k[i, :n]).T + np.abs(E).max(axis=0)[:, None])).max(axis=1, keepdims=True)
    return out, vmag, smag
