"""float64 references of the prompt encoders' kernels (index-tts_b200/csrc/emo.cu, ecapa.cu), computed on exactly the fp32
operands the kernels read.  Each returns (out, bound): bound is the worst-case error of the kernel's own fp32 evaluation,
derived from its summation shape, the documented ulp errors of the CUDA math functions (expf, erff, sinf / cosf 2 ulp;
sqrtf and division correctly rounded; rsqrtf 2 ulp) and, for the tensor-core GEMMs, the tf32 operand rounding.  A k-ulp
function error is a relative error of at most 2k * U (U = 2^-24).  tests/test_cond_refs_cpu.py pins each reference
against PyTorch and the pinned oracles, so that a failing GPU comparison points at the kernel."""
import math

import numpy as np
import torch

U = 2.0 ** -24            # unit roundoff of fp32
TF32 = 2.0 ** -9 + 2.0 ** -20     # a product of two operands each cut to tf32's 10 mantissa bits
TINY = 1e-30              # subnormal leftovers of underflowed exponentials


def _f64(x):
    return np.asarray(x, np.float64)


def tc_gemm(M, N, K):
    """Whether conv_gemm takes the tf32 tensor-core path for an fp32 GEMM of this shape (gemm_tc.cu gemm_tc_supported:
    K a multiple of 4, aligned operands, and M * N * K >= 2^18; below that the SIMT kernel runs)."""
    return K % 4 == 0 and M * N * K >= 1 << 18


def gemm_err(K, tf32):
    """Relative worst case of one fp32-accumulated dot product of K terms, times sum |a||b|: K fma roundings on the SIMT
    kernel; the tf32 cut of both operands plus K + 8 roundings of the accumulation on the tensor cores."""
    return (TF32 + (K + 8) * U) if tf32 else (K + 1) * U


def conv2d_sub2(x, w, b):
    """Conv2d(1 -> C, 3, stride 2) + ReLU of x [T][F] in the [T2][C * Fs] layout of Conv2dSubsampling2's x.transpose(1, 2)
    .view(t, c * f).  w [C][9] (or [C][1][3][3]), b [C].  The kernel starts at the bias and adds 9 fmas."""
    x, w, b = _f64(x), _f64(w).reshape(-1, 9), _f64(b)
    T, F = x.shape
    C = w.shape[0]
    T2, Fs = (T - 3) // 2 + 1, (F - 3) // 2 + 1
    pre = np.zeros((T2, C, Fs)) + b[None, :, None]
    mag = np.zeros((T2, C, Fs)) + np.abs(b)[None, :, None]
    for i in range(3):
        for j in range(3):
            xs = x[i:i + 2 * T2:2, j:j + 2 * Fs:2]                            # [T2][Fs]
            pre += w[None, :, 3 * i + j, None] * xs[:, None, :]
            mag += np.abs(w[None, :, 3 * i + j, None] * xs[:, None, :])
    return np.maximum(pre, 0.0).reshape(T2, C * Fs), (10 * U * mag).reshape(T2, C * Fs)


def pos_table(T, d):
    """RelPositionalEncoding's table (embedding.py:47-53) as the reference builds it, in fp32: div = exp(2i * -(ln 1e4 / d)),
    pe[t][2i] = sin(t * div), pe[t][2i + 1] = cos(t * div).  The reference value is that fp32 table.  The kernel's
    argument t * div differs from it by the rounding of div on both sides (logf 1 ulp, the product, expf 2 ulp in the
    kernel; the scalar, the product and exp in torch) and of t * div, times t; the sines add 2 ulp on each side."""
    i = torch.arange(0, d, 2)
    div = torch.exp(i * -(math.log(10000.0) / d))
    arg = torch.arange(T).unsqueeze(1) * div
    pe = torch.zeros(T, d)
    pe[:, 0::2] = torch.sin(arg)
    pe[:, 1::2] = torch.cos(arg)
    x = np.abs(2.0 * np.arange(d // 2) * math.log(10000.0) / d)                 # |exponent| of div
    rel_div = (4 * x + 4) * U + (2 * x + 4) * U                                  # kernel + torch
    a = np.outer(np.arange(T), np.exp(-x))                                       # t * div
    darg = a * (rel_div + 2 * U)
    darg[:, 0] = 0.0                                                             # div = exp(0) = 1 and t * 1 are exact
    bound = np.repeat(darg, 2, axis=1) + 10 * U
    return pe.double().numpy(), bound


def relpos_attention(qkv, pp, u, v, H, tc_scores, tc_pv):
    """RelPositionMultiHeadedAttention without rel_shift (attention.py:189-312) on the fp32 operands of the op:
    qkv [T][3 * H * dk] (q | k | v), pp = linear_pos(pe) [T][H * dk], pos_bias_u / _v [H * dk].  Per head
    s_ij = ((q_i + u) . k_j + (q_i + v) . p_j) / sqrt(dk), out_i = softmax_j(s_ij) v_j.  Returns (out [T][H * dk], bound).
    The bound follows the kernel chain: A' = [q + u | q + v] rounded once; the score GEMM over 2 dk terms (SIMT, or tf32
    when tc_scores) times fl(1 / sqrtf(dk)); the exact-exp row softmax (subtraction of the row max, expf, 32 lanes of
    ceil(T / 32) terms and a 5-level tree, 1 / sum, the product); the P V GEMM over Tp = T rounded up to 4 terms (SIMT, or
    tf32 when tc_pv).  The row max the kernel subtracts cancels in the normalisation, so a score error ds_j changes weight j
    by a factor exp(+-ds_j); relative weight errors eps_j move the output by at most
    (sum_j w_j |eps_j| |v_j| + mean(eps) sum_j w_j |v_j|) / (1 - mean(eps))."""
    qkv, pp = _f64(qkv), _f64(pp)
    T = qkv.shape[0]
    od = qkv.shape[1] // 3
    dk = od // H
    Tp = (T + 3) & ~3
    heads = lambda m: m.reshape(T, H, dk).transpose(1, 0, 2)                    # noqa: E731  [H][T][dk]
    q, k, vv, p = heads(qkv[:, :od]), heads(qkv[:, od:2 * od]), heads(qkv[:, 2 * od:]), heads(pp)
    a = np.concatenate([q + _f64(u).reshape(H, 1, dk), q + _f64(v).reshape(H, 1, dk)], axis=2)
    bb = np.concatenate([k, p], axis=2)
    c = 1.0 / math.sqrt(dk)
    s = (a @ bb.transpose(0, 2, 1)) * c
    mag = (np.abs(a) @ np.abs(bb).transpose(0, 2, 1)) * c
    ds = mag * (gemm_err(2 * dk, tc_scores) + U) + 3 * U * np.abs(s)          # + the rounding of A'; scale and product
    r = s.max(axis=2, keepdims=True)
    w = np.exp(s - r)
    w /= w.sum(axis=2, keepdims=True)
    eps = np.expm1(ds + U * np.abs(s - r) + 4 * U)
    ebar = (w * eps).sum(axis=2, keepdims=True)
    va = np.abs(vv)
    out = w @ vv
    vmag = w @ va
    werr = ((w * eps) @ va + ebar * vmag) / (1 - ebar)
    theta = (-(-T // 32) + 7) * U                                                # row sum, 1 / sum, the product
    emax = eps.max(axis=2, keepdims=True)
    bound = werr + vmag * (1 + emax) * (1 + theta) / (1 - ebar) * (theta + gemm_err(Tp, tc_pv)) + TINY
    merge = lambda m: m.transpose(1, 0, 2).reshape(T, od)                       # noqa: E731
    return merge(out), merge(bound)


def glu(x):
    """F.glu over the last dim of x [T][2C]: a * sigmoid(b).  Kernel: a * (1 / (1 + expf(-b))): expf 2 ulp and three
    roundings, 8 U relative."""
    x = _f64(x)
    C = x.shape[1] // 2
    y = x[:, :C] / (1.0 + np.exp(-x[:, C:]))
    return y, 8 * U * np.abs(y) + TINY


def geglu(x):
    """The perceiver's GEGLU on x [T][2C] (x | gate): gelu(gate) * x with the erf GELU.  Kernel: ((0.5 g) (1 + erff(g c)))
    a, c = fl(1 / sqrt 2): the argument rounds twice (c and the product), erff 2 ulp, 1 + erf once, two products."""
    x = _f64(x)
    C = x.shape[1] // 2
    a, g = x[:, :C], x[:, C:]
    z = g / math.sqrt(2.0)
    erf = np.vectorize(math.erf)(z)
    y = 0.5 * g * (1.0 + erf) * a
    e1 = 4 * U * np.abs(erf) + 2 / math.sqrt(math.pi) * np.exp(-z * z) * np.abs(z) * 2 * U + U * np.abs(1.0 + erf)
    return y, 0.5 * np.abs(g * a) * e1 * (1 + 4 * U) + 2 * U * np.abs(y) + TINY


def l2norm_scale(x, gamma):
    """PerceiverResampler's RMSNorm per row of x [T][C]: F.normalize(x) * sqrt(C) * gamma.  Kernel: 256 threads of
    ceil(C / 256) squares, a 5-level warp tree and 8 warp sums (n roundings, relative); sqrtf, 1 / max(., 1e-12), and the
    products x * inv * sqrtf(C) * gamma (sqrtf(C) rounded once)."""
    x, gm = _f64(x), _f64(gamma)
    C = x.shape[1]
    nrm = np.sqrt((x * x).sum(axis=1, keepdims=True))
    y = x / np.maximum(nrm, 1e-12) * math.sqrt(C) * gm
    n = -(-C // 256) + 5 + 8 + 1
    return y, (0.5 * n + 7) * U * np.abs(y) + TINY


def _softmax_err(s, ds, R, w):
    """(eps, ebar): relative error bound of every unnormalised weight expf(s_j - max) with score errors ds_j (the max
    cancels in the normalisation), and its w-weighted mean; R = |s_j - max| (the rounding of the subtraction)."""
    eps = np.expm1(ds + U * R + 4 * U)
    return eps, (w * eps).sum(axis=-1, keepdims=True)


def latent_attention(q, kv, H):
    """The perceiver's attention for nl latents: q [nl][H * dh], kv [n][2 * H * dh] (k | v); per head
    softmax_j(q . k_j / sqrt(dh)) v_j.  Kernel (one CTA per head and latent, 128 threads): dh fmas per score times
    rsqrtf(dh) (2 ulp); expf; ceil(n / 128) terms per thread, a 5-level tree and 4 warp sums; the value sum over n fmas
    and one division.  Returns (out [nl][H * dh], bound)."""
    q, kv = _f64(q), _f64(kv)
    nl, inner = q.shape
    n = kv.shape[0]
    dh = inner // H
    k = kv[:, :inner].reshape(n, H, dh).transpose(1, 0, 2)                     # [H][n][dh]
    vv = kv[:, inner:].reshape(n, H, dh).transpose(1, 0, 2)
    qh = q.reshape(nl, H, dh).transpose(1, 0, 2)                               # [H][nl][dh]
    c = 1.0 / math.sqrt(dh)
    s = (qh @ k.transpose(0, 2, 1)) * c                                        # [H][nl][n]
    ds = (np.abs(qh) @ np.abs(k).transpose(0, 2, 1)) * c * (dh + 1) * U + 6 * U * np.abs(s)
    r = s.max(axis=2, keepdims=True)
    w = np.exp(s - r)
    w /= w.sum(axis=2, keepdims=True)
    eps, ebar = _softmax_err(s, ds, np.abs(s - r), w)
    va = np.abs(vv)
    out = w @ vv
    vmag = w @ va
    werr = ((w * eps) @ va + ebar * vmag) / (1 - ebar)
    theta = (-(-n // 128) + 9 + 1) * U + (n + 1) * U                           # denominator, division, numerator
    bound = werr + vmag * (1 + eps.max(axis=2, keepdims=True)) / (1 - ebar) * theta + TINY
    merge = lambda m: m.transpose(1, 0, 2).reshape(nl, inner)                   # noqa: E731
    return merge(out), merge(bound)


def _sqrt_err(var, dvar):
    """Error of sqrtf(max(var~, 1e-12)) against sqrt(max(var, 1e-12)) when |var~ - var| <= dvar."""
    A = np.maximum(var, 1e-12)
    sd = np.sqrt(A)
    return dvar / sd + U * sd


def col_mean_std(x):
    """ECAPA's per-channel statistics over the T rows of x [T][C] (SE mean; the pooling's global mean and std):
    mean, std = sqrt(max(mean (x - mean)^2, 1e-12)).  Kernel: 8 row-strided partial sums of ceil(T / 8) terms each, then
    those 8 in order, then / T (n = ceil(T / 8) + 8 roundings); the variance sums (x - mean~)^2 the same way around the
    kernel's own mean.  Returns (mean, std, bound_mean, bound_std), each [C]."""
    x = _f64(x)
    T = x.shape[0]
    n = -(-T // 8) + 8
    mean = x.mean(axis=0)
    dm = n * U * np.abs(x).sum(axis=0) / T + U * np.abs(mean)
    var = ((x - mean) ** 2).mean(axis=0)
    dvar = (var + dm * dm) * ((n + 4) * U) + dm * dm
    return mean, np.sqrt(np.maximum(var, 1e-12)), dm + TINY, _sqrt_err(var, dvar) + TINY


def asp_pool(logits, x):
    """ECAPA's attentive statistics per channel c: a = softmax over t of logits[t][c]; mean = sum a x,
    std = sqrt(max(sum a (x - mean)^2, 1e-12)).  logits, x [T][C].  Kernel: the column max, expf(l - max), 8 row-strided
    partial sums of the weights, of p x and of p (x - mean~)^2, each reduced in order, then divided by the weight sum.
    Returns (mean, std, bound_mean, bound_std), each [C]."""
    lg, x = _f64(logits), _f64(x)
    T = x.shape[0]
    n = -(-T // 8) + 8
    r = lg.max(axis=0)
    w = np.exp(lg - r)
    w /= w.sum(axis=0)
    eps = np.expm1(U * np.abs(lg - r) + 4 * U)
    ebar = (w * eps).sum(axis=0)
    emax = eps.max(axis=0)
    xa = np.abs(x)
    mean = (w * x).sum(axis=0)
    xmag = (w * xa).sum(axis=0)
    dm = ((w * eps * xa).sum(axis=0) + ebar * xmag) / (1 - ebar) + xmag * (1 + emax) / (1 - ebar) * (2 * n + 3) * U + TINY
    d2 = (x - mean) ** 2
    var = (w * d2).sum(axis=0)
    dvar = ((w * eps * d2).sum(axis=0) + ebar * var) / (1 - ebar) + (var + dm * dm) * (1 + emax) / (1 - ebar) * (2 * n + 8) * U \
        + 2 * dm * dm
    return mean, np.sqrt(np.maximum(var, 1e-12)), dm, _sqrt_err(var, dvar) + TINY
