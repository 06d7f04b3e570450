"""GPU: the wgmma (tf32, TMA + register accumulators) implicit-GEMM back end against the SIMT fp32 back end and a
float64 numpy reference, over the shapes the vocoder / s2mel paths use (multi-tap, dilation, ragged
K and N, ConvTranspose output mapping, fused epilogues).  tf32 keeps 10 mantissa bits: the bound is
|err| <= 2e-3 * (sum_k |a||w|) per output, far looser than what is observed (printed)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def ref_conv(A, wk, taps, dil, pad, M):
    B, Tin, K = A.shape
    N = wk.shape[0]
    out = np.zeros((B, M, N), np.float64)
    mag = np.zeros((B, M, N), np.float64)
    W = wk.reshape(N, taps, K).astype(np.float64)
    for t in range(taps):
        rows = np.arange(M) + t * dil - pad
        ok = (rows >= 0) & (rows < Tin)
        a = np.zeros((B, M, K), np.float64)
        a[:, ok] = A[:, rows[ok]]
        out += a @ W[:, t].T
        mag += np.abs(a) @ np.abs(W[:, t]).T
    return out, mag


CASES = [
    # B, Tin, K, N, taps, dil, pad
    (2, 300, 512, 1536, 1, 1, 0),      # DiT wqkv
    (1, 500, 96, 96, 7, 3, 9),         # BigVGAN resblock conv, dilation 3
    (2, 131, 80, 1536, 7, 1, 3),       # conv_pre: ragged K = 80
    (1, 2000, 48, 48, 11, 5, 25),      # small channels, K = 1.5 chunks
    (1, 4096, 24, 24, 3, 1, 1),        # last stage: K = 24 < one chunk, BN = 32
    (2, 257, 1536, 512, 1, 1, 0),      # FFN w2: long K
    (1, 129, 592, 512, 1, 1, 0),       # skip_linear: K = 592
]


@pytest.mark.parametrize("B,Tin,K,N,taps,dil,pad", CASES)
def test_tc_matches_simt_and_fp64(engine, B, Tin, K, N, taps, dil, pad):
    rng = np.random.default_rng(B * 1000 + Tin + K + N)
    A = rng.standard_normal((B, Tin, K)).astype(np.float32)
    wk = (rng.standard_normal((N, taps * K)) / np.sqrt(taps * K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32) * 0.1
    ref, mag = ref_conv(A, wk, taps, dil, pad, Tin)
    ref = ref + bias
    simt = engine.debug_conv_gemm(A, wk, taps, dil, pad, bias=bias, backend=1).reshape(B, Tin, N)
    tc = engine.debug_conv_gemm(A, wk, taps, dil, pad, bias=bias, backend=2).reshape(B, Tin, N)
    assert np.abs(simt - ref).max() <= 1e-4 * max(1.0, np.abs(ref).max())
    err = np.abs(tc - ref)
    print(f"tc max err {err.max():.2e} (ref max {np.abs(ref).max():.2f}, bound {2e-3 * mag.max():.2e}); "
          f"rel rms {np.sqrt((err ** 2).mean()) / np.sqrt((ref ** 2).mean()):.2e}")
    assert np.all(err <= 2e-3 * mag + 1e-5)
    # fp16 operands (wgmma .f16, the tail path): same 10-bit mantissa, same bound; needs K % 8 == 0
    if K % 8 == 0:
        h = engine.debug_conv_gemm(A, wk, taps, dil, pad, bias=bias, backend=3).reshape(B, Tin, N)
        errh = np.abs(h - ref)
        print(f"fp16-operand tc max err {errh.max():.2e}; rel rms {np.sqrt((errh ** 2).mean()) / np.sqrt((ref ** 2).mean()):.2e}")
        assert np.all(errh <= 2e-3 * mag + 1e-5)


def test_tc_epilogues_and_transposed_mapping(engine):
    """ConvTranspose1d(k=2u, stride u) as a 2-tap GEMM with N = u*Co written through
    (out_off = -pad*Co, ldo = u*Co, out_valid = T*u*Co); plus act/res/accum/scale epilogue."""
    rng = np.random.default_rng(5)
    T, Ci, Co, u = 77, 64, 32, 4
    x = rng.standard_normal((1, T, Ci)).astype(np.float32)
    w = (rng.standard_normal((Ci, Co, 2 * u)) / np.sqrt(2 * Ci)).astype(np.float32)   # torch layout [in,out,k]
    bias = rng.standard_normal(Co).astype(np.float32) * 0.1
    pad = (2 * u - u) // 2
    # reference ConvTranspose1d
    full = np.zeros((T * u + 2 * u, Co), np.float64)
    for m in range(T):
        for k in range(2 * u):
            full[m * u + k] += x[0, m].astype(np.float64) @ w[:, :, k].astype(np.float64)
    ref = full[pad:pad + T * u] + bias
    wk = np.zeros((u * Co, 2 * Ci), np.float32)
    for r in range(u):
        wk[r * Co:(r + 1) * Co, :Ci] = w[:, :, r].T
        wk[r * Co:(r + 1) * Co, Ci:] = w[:, :, r + u].T
    for backend in (1, 2):
        out = engine.debug_conv_gemm(x, wk, taps=2, dil=-1, pad=0, M=T + 1, bias=bias, biasN=Co, out_off=-pad * Co,
                                     ldo=u * Co, out_valid=T * u * Co, backend=backend).reshape(T * u, Co)
        tol = 1e-4 if backend == 1 else 5e-3
        assert np.abs(out - ref).max() <= tol, (backend, np.abs(out - ref).max())
    # fused epilogue: out = scale * (gelu(acc + bias) + res + out_old)
    A = rng.standard_normal((2, 200, 128)).astype(np.float32)
    wk = (rng.standard_normal((96, 128)) / np.sqrt(128)).astype(np.float32)
    b2 = rng.standard_normal(96).astype(np.float32) * 0.1
    res = rng.standard_normal((2, 200, 96)).astype(np.float32)
    old = rng.standard_normal((2, 200, 96)).astype(np.float32)
    acc = A.astype(np.float64) @ wk.T.astype(np.float64) + b2
    from math import erf
    gelu = 0.5 * acc * (1 + np.vectorize(erf)(acc / np.sqrt(2)))
    ref = 0.5 * (gelu + res + old)
    for backend in (1, 2):
        out = engine.debug_conv_gemm(A, wk, bias=b2, act=1, res=res, accum=True, scale=0.5, out_init=old,
                                     backend=backend).reshape(2, 200, 96)
        tol = 1e-4 if backend == 1 else 5e-3
        assert np.abs(out - ref).max() <= tol, (backend, np.abs(out - ref).max())
