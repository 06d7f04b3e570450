"""GPU: the fused pair epilogues of the wgmma GEMM (fp16 operands, fp16 results) against float64 references, at every
tile width: EPI_ROPE (RoPE on q and k, the flash-attention q scale, head split to Qr | Kr | Vb), EPI_SWIGLU (silu(w1 x) *
w3 x) and EPI_WNGATE (the WaveNet gate).  The SwiGLU / gate weights go in as the plain [w1; w3] / [a; c] matrices and are
packed by the library exactly as the model packs them.

Operands are fp16-exact (rounded to fp16 on the host), so the products are exact and the GEMM itself only adds fp32
summation error; what is left is the fp16 rounding of the result (2^-11 relative) and the fast intrinsics.  Bound per
element: 2^-10 |ref| + the summation bound (K + 8) 2^-24 sum|a||w| carried through the epilogue's slope + 2^-24."""
import math

import numpy as np
import pytest

from tests import kernel_refs as kr

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TILES = [32, 64, 128]


def fp16_exact(x):
    return np.asarray(x, np.float32).astype(np.float16).astype(np.float32)


def check(name, got, ref, bound):
    got = np.asarray(got, np.float64)
    assert np.all(np.isfinite(got)), name
    err = np.abs(got - ref)
    worst = (err / bound).max()
    print(f"{name}: max err {err.max():.2e} (max |ref| {np.abs(ref).max():.2f}), max err / bound {worst:.3f}")
    assert np.all(err <= bound), (name, err.max(), float(worst))


def q_scale():
    """FLASH_Q_SCALE (ops.h): what EPI_ROPE multiplies q by for the wgmma flash attention."""
    return float(np.float32(0.125 * math.log2(math.e)))


_rope_cache = {}


def rope_case(B, H, T):
    key = (B, H, T)
    if key not in _rope_cache:
        rng = np.random.default_rng(B * 100 + H * 10 + T)
        K, N = 256, 3 * H * 64
        A = fp16_exact(rng.standard_normal((B, T, K)))
        wk = fp16_exact(rng.standard_normal((N, K)) / np.sqrt(K))
        bias = (rng.standard_normal(N) * 0.1).astype(np.float32)
        acc, mag = kr.ref_conv(A, wk, 1, 1, 0, T)
        acc, mag = acc + bias, mag + np.abs(bias)

        def heads(x, i):      # [B][T][3*H*64] -> section i as [B*H][T][64]
            return x[..., i * H * 64:(i + 1) * H * 64].reshape(B, T, H, 64).transpose(0, 2, 1, 3).reshape(B * H, T, 64)
        sc = q_scale()
        ref = np.stack([kr.rope(heads(acc, 0)) * sc, kr.rope(heads(acc, 1)), heads(acc, 2)])
        # a rotation mixes the two elements of a pair: their summation bounds add
        m = [heads(mag, i) for i in range(3)]
        pair = lambda x: np.repeat(x[..., 0::2] + x[..., 1::2], 2, axis=-1)
        accb = np.stack([pair(m[0]) * sc, pair(m[1]), m[2]]) * (K + 8) * U
        _rope_cache[key] = (A, wk, bias, ref, accb)
    return _rope_cache[key]


@pytest.mark.parametrize("tile_n", TILES)
@pytest.mark.parametrize("T", [1, 61, 129, 1741])
@pytest.mark.parametrize("B,H", [(1, 2), (2, 2), (1, 8), (2, 8)])
def test_rope_epilogue(engine, B, H, T, tile_n):
    A, wk, bias, ref, accb = rope_case(B, H, T)
    # scale 0: the entry uses FLASH_Q_SCALE, as the DiT does
    out = engine.debug_conv_gemm(A, wk, bias=bias, operands=1, tile_n=tile_n, epi=3, heads=H, aux=kr.rope_table(T),
                                 scale=0.0)
    check(f"rope B={B} H={H} T={T} BN={tile_n}", out, ref, 2.0 ** -10 * np.abs(ref) + accb + U)


@pytest.mark.parametrize("tile_n", TILES)
@pytest.mark.parametrize("inter", [64, 1536])
def test_swiglu_epilogue(engine, inter, tile_n):
    B, T, K = 2, 300, 512
    rng = np.random.default_rng(inter)
    A = fp16_exact(rng.standard_normal((B, T, K)))
    w13 = fp16_exact(rng.standard_normal((2 * inter, K)) / np.sqrt(K))      # [w1; w3]
    acc, mag = kr.ref_conv(A, w13, 1, 1, 0, T)
    a, b = acc[..., :inter], acc[..., inter:]
    ea, eb = ((K + 8) * U * mag[..., :inter], (K + 8) * U * mag[..., inter:])
    ref = kr.swiglu(a, b)
    silu = kr.swiglu(a, np.ones_like(a))
    bound = 2.0 ** -10 * np.abs(ref) + 1.1 * np.abs(b) * ea + np.abs(silu) * eb + 2e-6 * np.abs(ref) + U
    out = engine.debug_conv_gemm(A, w13, operands=1, tile_n=tile_n, epi=1)
    check(f"swiglu inter={inter} BN={tile_n}", out, ref, bound)


@pytest.mark.parametrize("tile_n", TILES)
@pytest.mark.parametrize("shared_g", [True, False], ids=["g_shared", "g_per_batch"])
@pytest.mark.parametrize("WH", [128, 512])
def test_wavenet_gate_epilogue(engine, WH, shared_g, tile_n):
    """The 5-tap in_layer on reflect-padded rows (Tin = T + 4, M = T, no further padding), bias packed with the
    weight, conditioning g shared by the batch (aux_stride 0, as the DiT uses it) or per batch entry."""
    B, T, taps = 2, 203, 5
    rng = np.random.default_rng(WH + shared_g)
    x = rng.standard_normal((B, T, WH))
    A = fp16_exact(np.concatenate([x[:, 2:0:-1], x, x[:, -2:-4:-1]], axis=1))           # F.pad(..., (2, 2), "reflect")
    w = fp16_exact(rng.standard_normal((2 * WH, taps * WH)) / np.sqrt(taps * WH))     # [a; c]
    bias = (rng.standard_normal(2 * WH) * 0.1).astype(np.float32)
    stride = 0 if shared_g else 3 * WH
    g = (rng.standard_normal((1 if shared_g else B, max(stride, 2 * WH))) * 0.5).astype(np.float32)
    acc, mag = kr.ref_conv(A, w, taps, 1, 0, T)
    gb = np.broadcast_to(g[:, None, :2 * WH], (B, 1, 2 * WH))
    acc = acc + bias + gb
    ref = kr.wn_gate(acc[..., :WH], acc[..., WH:])
    e = (taps * WH + 8) * U * (mag + np.abs(bias))
    bound = 2.0 ** -10 * np.abs(ref) + e[..., :WH] + 0.25 * e[..., WH:] + 2e-6 + U
    out = engine.debug_conv_gemm(A, w, taps, 1, 0, M=T, bias=bias, operands=1, tile_n=tile_n, epi=2, aux=g,
                                 aux_stride=stride)
    check(f"wn gate WH={WH} {'shared' if shared_g else 'per-batch'} g BN={tile_n}", out, ref, bound)
