"""GPU: the wgmma flash attention on fp16 q / k / v against a float64 reference computed on the same fp16 values
(tests/kernel_refs.py), fp32 and fp16 outputs, through both kernel values of idx_debug_flash_attention that select it
(0, the one the DiT uses, and 2).

Query rows come in five kinds (row index mod 5), so every tile meets each of them:
  0  plain random scores;
  1  one key dominates, and it is the last key: the running max jumps in the last key tile (the O rescale);
  2  large-magnitude scores (up to ~150: only a max-subtracted softmax stays finite);
  3  every real score strongly negative, so the zero-filled keys beyond T (score 0) would win if they were not masked;
  4  near-uniform scores.
T crosses the 128-key tiles and, from T = 257 on, wraps the kernel's 2-stage K/V ring; T = 1741 is the benchmarked size.

Bound per row and dimension: 1e-3 * sum_j p_ij |v_j| / sum_j p_ij (about twice the fp16 rounding of P, the dominant
term), plus the worst-case fp32 summation error of the scores where they are large, plus 2^-11 |ref| for the fp16 output."""
import math

import numpy as np
import pytest

from tests import kernel_refs as kr

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
KERNELS = {"default": 0, "wgmma": 2}


def make_qkv(B, H, T, seed):
    rng = np.random.default_rng(seed)
    BH = B * H
    u = rng.standard_normal((BH, 1, 64))                     # a direction every key shares
    k = rng.standard_normal((BH, T, 64)) + u
    v = rng.standard_normal((BH, T, 64)) + 1.0               # mean 1: an unmasked zero key would pull the output down
    q = rng.standard_normal((BH, T, 64)) * 0.4
    kind = np.arange(T) % 5
    klast = k[:, -1:, :]
    q[:, kind == 1] = 40.0 * klast / (klast ** 2).sum(-1, keepdims=True)     # score 40 with the last key
    q[:, kind == 2] *= 16.0
    q[:, kind == 3] = -0.5 * u + 0.05 * rng.standard_normal(q[:, kind == 3].shape)
    q[:, kind == 4] *= 2e-3
    return tuple(x.astype(np.float16) for x in (q, k, v))


_cache = {}


def reference(B, H, T, base):
    key = (B, H, T, base)
    if key not in _cache:
        q, k, v = make_qkv(B, H, T, seed=T * 31 + B * 7 + H)
        ref, vmag = kr.flash_attention(q, k, v, base)
        # worst-case fp32 summation error of a row's scores (64 exact products), in the exponent
        qa, ka = np.abs(q.astype(np.float64)), np.abs(k.astype(np.float64))
        smag = np.stack([(qa[i] @ ka[i].T).max(axis=1) for i in range(B * H)])[..., None]
        bound = vmag * (1e-3 + 2 * math.log(base) * 64 * U * smag)
        to_out = lambda x: x.reshape(B, H, T, 64).transpose(0, 2, 1, 3).reshape(B, T, H * 64)
        _cache[key] = (q, k, v, to_out(ref), to_out(bound))
    return _cache[key]


@pytest.mark.parametrize("kernel", list(KERNELS))
@pytest.mark.parametrize("B,H", [(1, 1), (1, 3), (2, 8)])
@pytest.mark.parametrize("T", [1, 7, 64, 65, 127, 128, 129, 256, 257, 385, 1741])
def test_flash_attention(engine, T, B, H, kernel):
    q, k, v, ref, bound = reference(B, H, T, 2.0)
    out, out16 = engine.debug_flash_attention(q, k, v, B, H, kernel=KERNELS[kernel])
    for name, got, bd in (("out", out, bound), ("out16", out16.astype(np.float32), bound + 2.0 ** -11 * np.abs(ref))):
        assert np.all(np.isfinite(got)), name
        err = np.abs(got - ref)
        worst = (err / bd).max()
        print(f"{kernel} T={T} B={B} H={H} {name}: max err {err.max():.2e}, max err / bound {worst:.3f}")
        assert np.all(err <= bd), (name, float(err.max()), float(worst))


@pytest.mark.parametrize("kernel", [1, 3, -1])
def test_unknown_kernel_is_refused(engine, kernel):
    q, k, v, _, _ = reference(1, 1, 7, 2.0)
    with pytest.raises(RuntimeError, match=r"failed \(2\)"):
        engine.debug_flash_attention(q, k, v, 1, 1, kernel=kernel)
