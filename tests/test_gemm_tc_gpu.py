"""GPU: the wgmma (tf32, TMA + register accumulators) implicit-GEMM back end against the SIMT fp32 back end and a
float64 numpy reference, over the shapes the vocoder / s2mel paths use (multi-tap, dilation, ragged
K and N, ConvTranspose output mapping, fused epilogues).  tf32 keeps 10 mantissa bits: the bound is
|err| <= 2e-3 * (sum_k |a||w|) per output, far looser than what is observed (printed).

Below that, every tile width (32 / 64 / 128, forced) x operand format (tf32 / fp16) on ragged shapes, the automatic tile
choice at the benchmarked DiT size, and every epilogue mode of the kernel (activations, column / row scales, broadcast A,
per-batch weights, operand row pitches, in-place residual), with fp16-exact operands and a summation-only bound.  The
library's diagnostic entry surrounds every output with sentinel guard bands and fails on a write outside the output."""
import numpy as np
import pytest

from tests.kernel_refs import act as ref_act
from tests.kernel_refs import ref_conv

pytestmark = pytest.mark.gpu


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
        h = engine.debug_conv_gemm(A, wk, taps, dil, pad, bias=bias, backend=2, operands=1).reshape(B, Tin, N)
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


# ---------------------------------------------------------------------------------------------------------------------
# Every tile width and operand format, forced, on ragged shapes.  Two input families:
#   random fp32 -> tf32 / fp16 rounding of the operands, bound 2e-3 * sum |a||w| as above;
#   fp16-exact operands (values rounded to fp16 on the host: exact in tf32 and fp16, so every product is exact and only
#   the fp32 summation rounds) -> bound (taps*K + 8) * 2^-24 * sum |a||w|: the worst case of n fp32 additions plus the
#   epilogue's few operations.  One dropped / duplicated 8-wide K step is ~20x that at K = 1536.
U = 2.0 ** -24


def fp16_exact(x):
    return np.asarray(x, np.float32).astype(np.float16).astype(np.float32)


def operands(rng, B, Tin, K, N, taps, exact):
    A = rng.standard_normal((B, Tin, K)).astype(np.float32)
    wk = (rng.standard_normal((N, taps * K)) / np.sqrt(taps * K)).astype(np.float32)
    bias = (rng.standard_normal(N) * 0.1).astype(np.float32)
    if exact:
        A, wk = fp16_exact(A), fp16_exact(wk)
    return A, wk, bias


def check(name, got, ref, bound):
    err = np.abs(got - ref)
    worst = (err / bound).max()
    print(f"{name}: max err {err.max():.2e}, max err / bound {worst:.3f}")
    assert np.all(err <= bound), (name, err.max(), float(worst))


RAGGED = [
    # B, Tin, K, N, taps, dil, pad
    (2, 300, 200, 200, 1, 1, 0),       # M % 128, N % 128 / 64 / 32, K % 32 / 64 all != 0
    (1, 257, 72, 100, 5, 2, 4),        # multi-tap, dilation 2, padding 4, K = 72
    (1, 130, 1536, 96, 1, 1, 0),       # long K: 48 (tf32) / 24 (fp16) stages, the ring wraps many times
    (1, 70, 24, 40, 1, 1, 0),          # one stage of work (n_iters == 1, ring clamped to 2 stages)
]


@pytest.mark.parametrize("tile_n", [32, 64, 128])
@pytest.mark.parametrize("ops", [0, 1], ids=["tf32", "fp16"])
@pytest.mark.parametrize("B,Tin,K,N,taps,dil,pad", RAGGED)
def test_tile_widths_forced(engine, tile_n, ops, B, Tin, K, N, taps, dil, pad):
    for exact in (False, True):
        rng = np.random.default_rng(B + Tin + K + N + taps)
        A, wk, bias = operands(rng, B, Tin, K, N, taps, exact)
        ref, mag = ref_conv(A, wk, taps, dil, pad, Tin)
        ref = ref + bias
        out = engine.debug_conv_gemm(A, wk, taps, dil, pad, bias=bias, backend=2, operands=ops, tile_n=tile_n,
                                     pad_cols=8)
        if exact:
            bound = (taps * K + 8) * U * (mag + np.abs(bias)) + 1e-30
        else:
            bound = 2e-3 * mag + 1e-5
        check(f"BN={tile_n} {'fp16' if ops else 'tf32'} {'fp16-exact' if exact else 'random'}", out, ref, bound)


@pytest.mark.parametrize("ops", [0, 1], ids=["tf32", "fp16"])
def test_auto_tile_at_dit_wqkv(engine, ops):
    """The DiT wqkv at the benchmarked size (B = 2, T = 1741, K = 512, N = 1536): 336 tiles of 128 columns, more than
    an H100 has SMs, so the automatic choice is the 128-wide tile."""
    B, T, K, N = 2, 1741, 512, 1536
    rng = np.random.default_rng(17)
    A, wk, bias = operands(rng, B, T, K, N, 1, True)
    ref, mag = ref_conv(A, wk, 1, 1, 0, T)
    out = engine.debug_conv_gemm(A, wk, bias=bias, backend=2, operands=ops).reshape(B, T, N)
    check(f"auto tile {'fp16' if ops else 'tf32'}", out, ref + bias, (K + 8) * U * (mag + np.abs(bias)))


# epilogue modes of the tensor-core kernel: name -> debug_conv_gemm arguments (fp16-exact operands)
MODES = {
    "gelu_erf": dict(act=1), "silu": dict(act=2), "mish": dict(act=3), "gelu_tanh": dict(act=4), "relu": dict(act=5),
    "colscale": dict(colscale=True), "rowscale": dict(rowscale=True),
    "a_bcast": dict(a_bcast=True), "w_batched": dict(w_batched=True),
    "lda_ldw": dict(lda=24, ldw=40),
    "res_inplace_interior": dict(res_is_out=True, M=256),
    "res_inplace_edge": dict(res_is_out=True, M=250, act=1),
    "res_accum_scale": dict(res=True, accum=True, scale=0.75),
}


@pytest.mark.parametrize("tile_n", [32, 64, 128])
@pytest.mark.parametrize("ops", [0, 1], ids=["tf32", "fp16"])
@pytest.mark.parametrize("mode", list(MODES))
def test_epilogue_modes(engine, mode, ops, tile_n):
    o = MODES[mode]
    B, Tin, K, N, taps, dil, pad = 2, 260, 96, 160, 3, 1, 1
    M = o.get("M", Tin)
    rng = np.random.default_rng(len(mode) * 7 + ops)
    A = fp16_exact(rng.standard_normal((1 if o.get("a_bcast") else B, Tin, K)))
    wshape = (B, N, taps * K) if o.get("w_batched") else (N, taps * K)
    wk = fp16_exact(rng.standard_normal(wshape) / np.sqrt(taps * K))
    bias = (rng.standard_normal(N) * 0.1).astype(np.float32)
    cs = (rng.uniform(0.5, 2.0, N).astype(np.float32) if o.get("colscale") else None)
    rs = (rng.uniform(0.0, 2.0, (B, M)).astype(np.float32) if o.get("rowscale") else None)
    init = rng.standard_normal((B, M, N)).astype(np.float32)
    res = rng.standard_normal((B, M, N)).astype(np.float32) if o.get("res") else None
    scale = o.get("scale", 1.0)
    kw = dict(bias=bias, act=o.get("act", 0), colscale=cs, rowscale=rs, M=M, scale=scale, B=B,
              a_bcast=o.get("a_bcast", False), w_batched=o.get("w_batched", False), res=res,
              res_is_out=o.get("res_is_out", False), accum=o.get("accum", False))
    A_dev, wk_dev, K_arg = A, wk, None
    if "lda" in o:      # operands stored with a wider row pitch: the extra columns are garbage the GEMM must skip
        A_dev = np.concatenate([A, rng.standard_normal(A.shape[:2] + (o["lda"],)).astype(np.float32)], -1)
        wk_dev = np.concatenate([wk, rng.standard_normal(wk.shape[:-1] + (o["ldw"],)).astype(np.float32)], -1)
        K_arg = K
    ref_pre, mag = ref_conv(A, wk, taps, dil, pad, M)
    pre = ref_pre + bias
    post = ref_act(pre, kw["act"])
    mult = np.ones_like(post)
    if cs is not None:
        mult = mult * cs
    if rs is not None:
        mult = mult * rs[:, :, None]
    ref = post * mult
    extra = np.zeros_like(ref)
    if res is not None:
        extra += res
    if kw["res_is_out"] or kw["accum"]:
        extra += init
    ref = (ref + extra) * scale
    # summation bound through the activation (slope <= 1.2), fast-intrinsic error of the activation, epilogue roundings
    bound = ((1.2 * (taps * K + 8) * U * (mag + np.abs(bias)) + (2e-6 if kw["act"] else 0) * np.abs(post)) * np.abs(mult)
             + 8 * U * np.abs(extra)) * abs(scale) + 1e-30
    out = engine.debug_conv_gemm(A_dev, wk_dev, taps, dil, pad, K=K_arg, backend=2, operands=ops, tile_n=tile_n,
                                 out_init=init, **kw).reshape(B, M, N)
    check(f"{mode} BN={tile_n} {'fp16' if ops else 'tf32'}", out, ref, bound)
