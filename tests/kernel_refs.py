"""float64 references of the tensor-core kernels' operations, computed on exactly the operands the kernels read.
tests/test_kernel_refs_cpu.py pins each of them against PyTorch / the oracle, so that a failing GPU comparison
points at the kernel and not at its reference."""
import math

import numpy as np
import torch


def ref_conv(A, wk, taps, dil, pad, M):
    """Multi-tap channels-last GEMM (Conv1d with zero padding):
        out[b][m][n] = sum_tap sum_k A[b][m + tap*dil - pad][k] * wk[b][n][tap*K + k].
    A [B or 1][Tin][K]; wk [N][taps*K] (shared) or [B][N][taps*K] (per batch entry).  Returns (out, mag), both
    float64 [B][M][N]; mag = the same sum over |A| |wk|, the scale of any summation error."""
    A = np.asarray(A, np.float64)
    W = np.asarray(wk, np.float64)
    B = max(A.shape[0], W.shape[0] if W.ndim == 3 else 1)
    if W.ndim == 2:
        W = W[None]
    A = np.broadcast_to(A, (B,) + A.shape[1:])
    W = np.broadcast_to(W, (B,) + W.shape[1:])
    Tin, K = A.shape[1], A.shape[2]
    N = W.shape[1]
    W = W.reshape(B, N, taps, K)
    out = np.zeros((B, M, N), np.float64)
    mag = np.zeros((B, M, N), np.float64)
    for t in range(taps):
        rows = np.arange(M) + t * dil - pad
        ok = (rows >= 0) & (rows < Tin)
        a = np.zeros((B, M, K), np.float64)
        a[:, ok] = A[:, rows[ok]]
        wt = W[:, :, t].transpose(0, 2, 1)
        out += a @ wt
        mag += np.abs(a) @ np.abs(wt)
    return out, mag


def act(x, kind):
    """The GEMM epilogue activations (ops.h ACT_*) in float64."""
    x = np.asarray(x, np.float64)
    if kind == 0:
        return x
    if kind == 1:
        return 0.5 * x * (1.0 + np.vectorize(math.erf)(x / math.sqrt(2.0)))
    if kind == 2:
        return x / (1.0 + np.exp(-x))
    if kind == 3:
        return x * np.tanh(np.logaddexp(0.0, x))
    if kind == 4:
        return 0.5 * x * (1.0 + np.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)))
    if kind == 5:
        return np.maximum(x, 0.0)
    raise ValueError(kind)


def flash_attention(q, k, v, base):
    """Full (non-causal) attention of the flash kernels on their exact inputs: q (already scaled), k, v [BH][T][64]
    (the fp16 values the kernel reads).  Weights p_ij = base^(q_i . k_j): base 2 for the wgmma kernel (q carries
    log2 e), e for the mma.sync kernel.  Returns (out, vmag) float64 [BH][T][64]; vmag = sum_j p_ij |v_j| / sum_j p_ij,
    the scale of an error in the weights."""
    q, k, v = (np.asarray(x, np.float64) for x in (q, k, v))
    lb = math.log(base)
    out = np.empty_like(q)
    vmag = np.empty_like(q)
    for i in range(q.shape[0]):
        s = (q[i] @ k[i].T) * lb
        p = np.exp(s - s.max(axis=1, keepdims=True))
        l = p.sum(axis=1, keepdims=True)
        out[i] = (p @ v[i]) / l
        vmag[i] = (p @ np.abs(v[i])) / l
    return out, vmag


def ref_decode_attention(q, K, V, ctx=None, hd=64, keys=None, chunk=64):
    """Attention of GPT decode steps on the decode kernels' exact operands, in float64.  q [N][H*hd]: the query of each
    step as the kernel read it; K, V [T][H*hd]: the cache (bf16 values); ctx [N] (or one int): step i attends to keys
    0 .. ctx[i] - 1.  Instead of ctx, keys [N][T] bool names the rows of K / V that step i attends to (a beam's keys
    spread over several cache slots).  Scores q . k / sqrt(hd) (= / 8), natural-exp softmax over the keys, weighted V,
    per head.  Returns (out, vmag) float64 [N][H*hd]; vmag = sum_j p_j |v_j| / sum_j p_j, the scale of an error in the
    weights."""
    q = np.atleast_2d(np.asarray(q, np.float64))
    N, D = q.shape
    H = D // hd
    if keys is None:
        ctx = np.broadcast_to(np.asarray(ctx, np.int64), (N,))
        keys = np.arange(int(ctx.max()))[None, :] < ctx[:, None]
    keys = np.asarray(keys, bool)
    T = keys.shape[1]
    assert keys.shape[0] == N and keys.any(axis=1).all(), "every step attends to at least one key"
    Kh = np.ascontiguousarray(np.asarray(K, np.float64)[:T].reshape(T, H, hd).transpose(1, 0, 2))     # [H][T][hd]
    Vt = np.ascontiguousarray(np.asarray(V, np.float64)[:T].reshape(T, H, hd).transpose(1, 2, 0))     # [H][hd][T]
    Va = np.abs(Vt)
    out = np.empty((N, H, hd))
    vmag = np.empty((N, H, hd))
    for i0 in range(0, N, chunk):
        i1 = min(N, i0 + chunk)
        qc = q[i0:i1].reshape(i1 - i0, H, hd).transpose(1, 2, 0)                  # [H][hd][n]
        s = np.where(keys[i0:i1].T[None], (Kh @ qc) / math.sqrt(hd), -np.inf)    # [H][T][n]
        p = np.exp(s - s.max(axis=1, keepdims=True))
        l = p.sum(axis=1)[:, None, :]                                             # [H][1][n]
        out[i0:i1] = ((Vt @ p) / l).transpose(2, 0, 1)
        vmag[i0:i1] = ((Va @ p) / l).transpose(2, 0, 1)
    return out.reshape(N, D), vmag.reshape(N, D)


def beam_key_slots(parents, plen, m, row0):
    """Where the keys of every beam row live in the KV cache, from the beams' traced ancestry alone (never from the
    engine's lineage map).  parents [steps][m]: the parent beam (0 .. m-1) that beam_step_kernel chose for each beam
    after each decode step (idx_gpt_beam_trace; a finished utterance records the identity), plen: the utterance's prompt
    length, row0 = u * m: its first row.  Returns slots [steps][m][plen + steps] int32: at decode step k, beam row
    row0 + r attends to key positions j = 0 .. plen + k, and position j lives in cache slot slots[k, r, j] (-1 beyond).

    Row b of gpt_fused_kernel writes its keys into cache slot b (row_seq[b] = b in decode launches), so:
      * prompt positions 0 .. plen - 1 come from slot row0 (the beam driver's prefill tiles run in the first beam's slot);
      * generated position plen + i (i < k) comes from the slot of r's ancestor at step i: a_k = r, a_i = parents[i][a_(i+1)]
        (phase C of beam_step_kernel copies the parent's map, phys_nxt[r][t] = phys_cur[parent][t] for t <= k, and the
        driver starts every row's map at phys[r][0] = r);
      * position plen + k, the one being decoded, comes from r itself (phys_nxt[r][k + 1] = r)."""
    parents = np.asarray(parents, np.int64)
    steps = parents.shape[0]
    assert parents.shape == (steps, m) and ((parents >= 0) & (parents < m)).all()
    slots = np.full((steps, m, plen + steps), -1, np.int32)
    slots[:, :, :plen] = row0
    for k in range(steps):
        a = np.arange(m)                      # a_k = r for every beam r
        slots[k, :, plen + k] = row0 + a
        for i in range(k - 1, -1, -1):
            a = parents[i][a]                 # a_i = parents[i][a_(i+1)]
            slots[k, :, plen + i] = row0 + a
    return slots


def rope_angles(T, hd=64):
    """Rotary angles as the model computes them: fp32 freqs, fp32 t * freq (oracle/s2mel.py:_rope)."""
    freqs = 1.0 / (10000 ** (torch.arange(0, hd, 2)[: hd // 2].float() / hd))
    return torch.outer(torch.arange(T).float(), freqs).double().numpy()      # [T][hd/2], fp32 values


def rope_table(T, hd=64):
    """The (cos, sin) table the RoPE epilogue reads, [T][hd/2][2] fp32: cos / sin of the fp32 angles, rounded once."""
    ang = rope_angles(T, hd)
    return np.stack([np.cos(ang), np.sin(ang)], -1).astype(np.float32)


def rope(x, hd=64):
    """Interleaved-pair rotation of x [..., T, hd] (pairs (2i, 2i+1) by angle t * freq_i) in float64."""
    x = np.asarray(x, np.float64)
    ang = rope_angles(x.shape[-2], hd)
    c, s = np.cos(ang), np.sin(ang)
    a, b = x[..., 0::2], x[..., 1::2]
    out = np.empty_like(x)
    out[..., 0::2] = a * c - b * s
    out[..., 1::2] = b * c + a * s
    return out


def swiglu(a, b):
    """F.silu(a) * b in float64."""
    a = np.asarray(a, np.float64)
    return a / (1.0 + np.exp(-a)) * np.asarray(b, np.float64)


def wn_gate(a, c):
    """WaveNet fused_add_tanh_sigmoid_multiply: tanh(a) * sigmoid(c) (the conditioning g already added), float64."""
    return np.tanh(np.asarray(a, np.float64)) / (1.0 + np.exp(-np.asarray(c, np.float64)))


# ---------------------------------------------------------------- the tail's non-GEMM kernels ----
U = 2.0 ** -24            # unit roundoff of fp32


def pad1d_reflect_rows(T, left, right):
    """Source row of every row of a reflect-padded frame of T rows (encodec.py pad1d mode='reflect'), -1 for a zero row:
    an input of T <= max(left, right) rows is zero-extended to max(left, right) + 1 rows, reflected by F.pad, cropped."""
    Tr = max(T, max(left, right) + 1)
    idx = np.pad(np.arange(Tr), (left, right), mode="reflect")[:T + left + right]
    return np.where(idx < T, idx, -1)


def pad1d_reflect(x, left, right):
    """x [..., T, C] reflect-padded along T as pad1d does, float64."""
    x = np.asarray(x, np.float64)
    src = pad1d_reflect_rows(x.shape[-2], left, right)
    out = np.take(x, np.maximum(src, 0), axis=-2)
    out[..., src < 0, :] = 0.0
    return out


def rownorm(x, T, mode, w=None, b=None, eps=0.0, m0=None, m1=None, mod_stride=0):
    """The row norms of rownorm_kernel on x [rows][C], float64: mode 0 LayerNorm (affine w, b; modulation
    v * (1 + m0[r // T]) + m1[r // T]), mode 1 RMSNorm times w (modulation m0[r // T] * v + m1[r // T]).  m0 / m1 are flat
    [B * mod_stride (+ C)] vectors read at (r // T) * mod_stride.  Returns (out, bound): bound is the worst-case error of
    the kernel's fp32 evaluation: warp sums of C / 32 terms and a 5-level tree (n = C / 32 + 5), rsqrtf (2 ulp), and one
    rounding per later product / sum."""
    x = np.asarray(x, np.float64)
    R, C = x.shape
    n = -(-C // 32) + 5
    bi = np.arange(R) // T
    if mode == 0:
        mean = x.mean(1, keepdims=True)
        dm = (n + 1) * U * np.abs(x).sum(1, keepdims=True) / C          # error of the fp32 mean
    else:
        mean, dm = 0.0, 0.0
    d = x - mean
    q = (d * d).mean(1, keepdims=True)
    rstd = 1.0 / np.sqrt(q + eps)
    v = d * rstd
    # q: n + 2 roundings per term, plus the mean's error through 2|d|; the variance + eps and rsqrtf
    rel_q = (n + 3) * U + 2 * np.abs(d).mean(1, keepdims=True) * dm / np.maximum(q + eps, 1e-300)
    rel_rstd = 0.5 * rel_q + 4 * U
    err = np.abs(v) * (rel_rstd + 2 * U) + dm * rstd
    one = np.ones(C)
    ww = one if w is None else np.asarray(w, np.float64)
    bb = np.zeros(C) if b is None else np.asarray(b, np.float64)
    v = v * ww + bb
    err = err * np.abs(ww) + 2 * U * (np.abs(v) + np.abs(bb))
    if m0 is not None:
        m0, m1 = np.asarray(m0, np.float64), np.asarray(m1, np.float64)
        rows = bi[:, None] * mod_stride + np.arange(C)[None]
        s, t = m0[rows], m1[rows]
        f = 1.0 + s if mode == 0 else s
        vo = v * f + t
        err = err * np.abs(f) + 3 * U * (np.abs(v * f) + np.abs(t)) + (U * np.abs(v * f) if mode == 0 else 0.0)
        v = vo
    return v, err + U * np.abs(v)


def gn_mish(x, w, b, eps):
    """GroupNorm(1 group) over each [T][C] block of x [B][T][C], per-channel affine, then Mish (F.mish), float64.
    Returns (out, y): y = the normalised, affine value Mish is applied to."""
    x = np.asarray(x, np.float64)
    mean = x.mean(axis=(1, 2), keepdims=True)
    var = x.var(axis=(1, 2), keepdims=True)
    y = (x - mean) / np.sqrt(var + eps) * np.asarray(w, np.float64) + np.asarray(b, np.float64)
    return y * np.tanh(np.logaddexp(0.0, y)), y


def dwconv(x, w, b, k):
    """Depthwise Conv1d of x [B][T][C] with w [C][k], zero padding (k - 1) // 2, bias b [C] or None.  Returns (out, mag)
    float64; mag = the same sum over absolute values."""
    x = np.asarray(x, np.float64)
    w = np.asarray(w, np.float64)
    B, T, C = x.shape
    pad = (k - 1) // 2
    out = np.zeros((B, T, C)) + (0.0 if b is None else np.asarray(b, np.float64))
    mag = np.abs(out)
    for j in range(k):
        src = np.arange(T) + j - pad
        ok = (src >= 0) & (src < T)
        out[:, ok] += x[:, src[ok]] * w[:, j]
        mag[:, ok] += np.abs(x[:, src[ok]] * w[:, j])
    return out, mag


def activation1d(x, alpha, beta, taps, logscale):
    """BigVGAN's Activation1d(SnakeBeta) on channels-last x [B][T][C] with the 12 FIR taps, float64 (sine included):
        u[2j] = 2 sum_q x[clamp(j - 3 + q)] f[11 - 2q],  u[2j + 1] = 2 sum_q x[clamp(j - 2 + q)] f[10 - 2q]
        a[m] = u[m] + sin(u[m] ea)^2 / (eb + 1e-9),        y[t] = sum_k a[clamp(2t - 5 + k)] f[k]
    (resample.py UpSample1d / DownSample1d and activations.py SnakeBeta on one line each).  Returns (y, bound): the
    worst-case error of the kernel's fp32 evaluation: 6- and 12-term fma chains (taps within one fp32 rounding of f),
    the argument u * ea, the two-constant reduction and __sinf (2^-21.41 absolute on [-pi, pi])."""
    x = np.asarray(x, np.float64)
    f = np.asarray(taps, np.float64)
    B, T, C = x.shape
    a, bt = np.asarray(alpha, np.float64), np.asarray(beta, np.float64)
    ea, eb = (np.exp(a), np.exp(bt)) if logscale else (a, bt)
    ib = 1.0 / (eb + 1e-9)
    cl = lambda i: np.clip(i, 0, T - 1)                                  # noqa: E731
    j = np.arange(T)
    u = np.zeros((B, 2 * T, C))
    um = np.zeros((B, 2 * T, C))
    for q in range(6):
        u[:, 0::2] += 2 * x[:, cl(j - 3 + q)] * f[11 - 2 * q]
        um[:, 0::2] += 2 * np.abs(x[:, cl(j - 3 + q)] * f[11 - 2 * q])
        u[:, 1::2] += 2 * x[:, cl(j - 2 + q)] * f[10 - 2 * q]
        um[:, 1::2] += 2 * np.abs(x[:, cl(j - 2 + q)] * f[10 - 2 * q])
    arg = u * ea
    s = np.sin(arg)
    act = u + ib * s * s
    du = 9 * U * um                                                      # 6 fmas + the tap rounding
    dsin = 2.0 ** -21.41 + U * (4 * np.abs(arg) + 8) + np.abs(ea) * du   # argument rounding (ea 2 ulp), reduction, __sinf
    dact = du + ib * (2 * np.abs(s) * dsin + 8 * U * s * s) + U * np.abs(act)
    y = np.zeros((B, T, C))
    bound = np.zeros((B, T, C))
    for k in range(12):
        m = np.clip(2 * j - 5 + k, 0, 2 * T - 1)
        y += act[:, m] * f[k]
        bound += dact[:, m] * abs(f[k]) + 15 * U * np.abs(act[:, m] * f[k])
    return y, bound


def conv_post(x, w, bias, use_tanh):
    """BigVGAN conv_post on x [B][T][C]: Conv1d(C -> 1, k 7, pad 3) with w [7][C] (+ bias), then tanh or a clamp to
    [-1, 1], float64.  Returns (y, pre, mag): pre = the conv before the final function, mag = its sum of |terms|."""
    x = np.asarray(x, np.float64)
    w = np.asarray(w, np.float64)
    B, T, C = x.shape
    b0 = 0.0 if bias is None else float(np.asarray(bias).reshape(-1)[0])
    pre = np.full((B, T), b0)
    mag = np.full((B, T), abs(b0))
    for k in range(7):
        src = np.arange(T) + k - 3
        ok = (src >= 0) & (src < T)
        pre[:, ok] += x[:, src[ok]] @ w[k]
        mag[:, ok] += np.abs(x[:, src[ok]]) @ np.abs(w[k])
    y = np.tanh(pre) if use_tanh else np.clip(pre, -1.0, 1.0)
    return y, pre, mag


def cfg_euler(x, vc, vu, dt, rate, zero_rows):
    """One CFG Euler step of flow_matching.py:96-113, float64: x + dt * ((1 + r) vc - r vu), rows with zero_rows set
    to 0.  x, vc, vu [T][C]; zero_rows [T] bool.  Returns (out, mag): mag bounds the terms of the fp32 evaluation."""
    x, vc, vu = (np.asarray(v, np.float64) for v in (x, vc, vu))
    d = (1.0 + rate) * vc - rate * vu
    out = x + dt * d
    mag = np.abs(x) + abs(dt) * ((1.0 + abs(rate)) * np.abs(vc) + abs(rate) * np.abs(vu))
    z = np.asarray(zero_rows, bool)
    out[z] = 0.0
    mag[z] = 0.0
    return out, mag
