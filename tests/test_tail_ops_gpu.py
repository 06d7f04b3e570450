"""GPU: the tail's non-GEMM kernels (row norms, GroupNorm + Mish, depthwise conv, nearest interpolation, reflect padding
and the packed-segment layout kernels, the CFG Euler updates, the RoPE table, BigVGAN's fused Snake and conv_post)
against float64 references, each through the host function the model calls (Engine.debug_tail_op).  Row-indexed inputs
sit between NaN rows, so a read outside a sequence shows up as NaN; every output sits between sentinel guard bands.

Layout kernels copy values, so they must equal the reference rounded once, bit for bit.  Arithmetic kernels are held to
the worst-case error of their fp32 evaluation (tests/kernel_refs.py derives each bound from the operation: summation
(n + c) 2^-24 sum|terms|, the documented errors of rsqrtf / __sinf / expf / tanhf / log1pf, and one rounding per product);
an fp16 output must be the fp16 rounding of the fp32 one."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from indextts_b200.synth import BIGVGAN_V2_22K, CODEC_CFG, S2MEL_CFG, kaiser_sinc_filter1d, small_s2mel_cfg
from tests import kernel_refs as kr

pytestmark = pytest.mark.gpu

U = kr.U
SHORT = [1, 2, 3, 4, 5, 127, 128, 129]
DIT_C = S2MEL_CFG["wn_hidden"]                    # the WaveNet / FinalLayer width
SMALL_C = small_s2mel_cfg()["wn_hidden"]
CODEC_C = CODEC_CFG["vocos_dim"]
BIGVGAN_LAST_C = BIGVGAN_V2_22K["upsample_initial_channel"] >> len(BIGVGAN_V2_22K["upsample_rates"])


def check(name, got, ref, bound):
    got = np.asarray(got, np.float64)
    assert np.all(np.isfinite(got)), name
    err = np.abs(got - ref)
    worst = float((err / bound).max())
    print(f"{name}: max err {err.max():.2e} (max |ref| {np.abs(ref).max():.2f}), max err / bound {worst:.3f}")
    assert np.all(err <= bound), (name, float(err.max()), worst)


def exact(name, got, want):
    """Bitwise equality (NaN-free)."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (name, got.shape, want.shape)
    assert not np.isnan(got.astype(np.float32)).any(), f"{name}: NaN (a read outside the input rows)"
    bad = got.view(np.uint16 if got.dtype == np.float16 else np.uint32) != want.view(np.uint16 if want.dtype == np.float16 else np.uint32)
    assert not bad.any(), f"{name}: {int(bad.sum())} elements differ, first at {np.argwhere(bad)[0].tolist()}"


# ------------------------------------------------------------------------------------------------ layout ----
@pytest.mark.parametrize("C", [DIT_C, SMALL_C, 33, 20])
def test_reflect_pad_rows(engine, C):
    rng = np.random.default_rng(C)
    for T in SHORT:
        for left, right in ((2, 2), (3, 1)):
            x = rng.standard_normal((2, T, C)).astype(np.float32)
            want = kr.pad1d_reflect(x, left, right).astype(np.float32)
            y, y16 = engine.debug_tail_op("reflect_pad_rows", x, left=left, right=right, out=True, out16=True)
            exact(f"reflect_pad_rows T={T} C={C} pad=({left},{right})", y, want)
            exact("  fp16", y16, want.astype(np.float16))
            _, only16 = engine.debug_tail_op("reflect_pad_rows", x, left=left, right=right, out=False, out16=True)
            exact("  fp16 only", only16, want.astype(np.float16))


def seg_ref(x, off, left, right):
    return np.concatenate([kr.pad1d_reflect(x[:, off[u]:off[u + 1]], left, right) for u in range(len(off) - 1)], axis=1)


SEG_TABLES = [SHORT, [1, 129, 2, 1], [5, 1], [1], [2], [128, 1, 3, 1, 2], [1, 2], [2, 1]]


@pytest.mark.parametrize("C", [DIT_C, SMALL_C, 64])
def test_reflect_pad_segments_and_compact(engine, C):
    rng = np.random.default_rng(C + 1)
    for lens in SEG_TABLES:
        off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
        x = rng.standard_normal((2, int(off[-1]), C)).astype(np.float32)
        _, y16 = engine.debug_tail_op("reflect_pad_segments", x, seg_off=off, left=2, right=2, out=False, out16=True)
        exact(f"reflect_pad_segments {lens} C={C}", y16, seg_ref(x, off, 2, 2).astype(np.float16))
        # compact: rows of the gapped GEMM output (total + (n - 1) * gap) back to the packed rows
        gap = 4
        Mg = int(off[-1]) + (len(lens) - 1) * gap
        g16 = rng.standard_normal((2, Mg, C)).astype(np.float16)
        src = np.concatenate([np.arange(off[u], off[u + 1]) + u * gap for u in range(len(lens))])
        _, c16 = engine.debug_tail_op("compact_segments16", x16=g16, seg_off=off, gap=gap, out=False, out16=True)
        exact(f"compact_segments16 {lens} C={C}", c16, g16[:, src])


def test_layout_beyond_65535_rows(engine):
    """A packed solve longer than gridDim.y allows: the rows loop past 65535."""
    rng = np.random.default_rng(5)
    C = 64
    lens = [1, 40000, 2, 30000, 1]
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    x = rng.standard_normal((2, int(off[-1]), C)).astype(np.float32)
    _, y16 = engine.debug_tail_op("reflect_pad_segments", x, seg_off=off, left=2, right=2, out=False, out16=True)
    exact("reflect_pad_segments 70004 rows", y16, seg_ref(x, off, 2, 2).astype(np.float16))
    Mg = int(off[-1]) + (len(lens) - 1) * 4
    g16 = rng.standard_normal((2, Mg, C)).astype(np.float16)
    src = np.concatenate([np.arange(off[u], off[u + 1]) + u * 4 for u in range(len(lens))])
    _, c16 = engine.debug_tail_op("compact_segments16", x16=g16, seg_off=off, gap=4, out=False, out16=True)
    exact("compact_segments16 70004 rows", c16, g16[:, src])
    xs = x[:1]
    y, _ = engine.debug_tail_op("reflect_pad_rows", xs, left=2, right=2)
    exact("reflect_pad_rows 70004 rows", y, kr.pad1d_reflect(xs, 2, 2).astype(np.float32))
    y, _ = engine.debug_tail_op("nearest_interp", xs, n2=70100)
    want = F.interpolate(torch.from_numpy(xs).transpose(1, 2), size=70100, mode="nearest").transpose(1, 2).numpy()
    exact("nearest_interp 70004 -> 70100 rows", y, want)
    w = rng.standard_normal((C, 7)).astype(np.float32)
    y, _ = engine.debug_tail_op("dwconv1d", xs, w=w, n2=7)
    ref, mag = kr.dwconv(xs, w, None, 7)
    check("dwconv1d 70004 rows", y, ref, 9 * U * mag + 1e-30)


def test_nearest_interp_every_length(engine):
    rng = np.random.default_rng(6)
    for Tin in range(1, 401):
        C = 20 if Tin % 50 else DIT_C
        x = rng.standard_normal((1, Tin, C)).astype(np.float32)
        for Tout in sorted({int(1.72 * Tin), 2 * Tin, Tin - 1, 1} - {0}):
            y, _ = engine.debug_tail_op("nearest_interp", x, n2=Tout)
            want = F.interpolate(torch.from_numpy(x).transpose(1, 2), size=Tout, mode="nearest").transpose(1, 2).numpy()
            exact(f"nearest_interp {Tin} -> {Tout}", y, want)


# ------------------------------------------------------------------------------------------- arithmetic ----
@pytest.mark.parametrize("C", [CODEC_C, 33])
def test_dwconv_short_sequences(engine, C):
    rng = np.random.default_rng(C + 2)
    k = 7
    w, b = rng.standard_normal((C, k)).astype(np.float32), rng.standard_normal(C).astype(np.float32)
    for T in (1, 2, 3, 6, 50):
        x = rng.standard_normal((1, T, C)).astype(np.float32)
        y, _ = engine.debug_tail_op("dwconv1d", x, w=w, b=b, n2=k)
        ref, mag = kr.dwconv(x, w, b, k)
        check(f"dwconv1d T={T} C={C}", y, ref, (k + 2) * U * mag)


def rownorm_case(engine, name, x, B, T, mode, w=None, b=None, eps=1e-6, m0=None, m1=None, mod_stride=0):
    op = "layernorm" if mode == 0 else "rmsnorm_adaln"
    C = x.shape[-1]
    kw = dict(B=B, T=T, C=C, w=w, b=b, eps=eps, m0=m0, m1=m1, mod_stride=mod_stride)
    y, y16 = engine.debug_tail_op(op, x, out=True, out16=True, **kw)
    ref, bound = kr.rownorm(x.reshape(B * T, C), T, mode, w, b, np.float32(eps), m0, m1, mod_stride)
    check(name, y.reshape(B * T, C), ref, bound)
    exact(f"{name} fp16", y16, y.astype(np.float16))
    _, only16 = engine.debug_tail_op(op, x, out=False, out16=True, **kw)
    exact(f"{name} fp16 only", only16, y.astype(np.float16))


@pytest.mark.parametrize("C", [CODEC_C, DIT_C, SMALL_C, 33, 20])
def test_row_norms(engine, C):
    rng = np.random.default_rng(C + 3)
    f32 = lambda a: np.asarray(a, np.float32)            # noqa: E731
    B, T = 2, 13                                         # 26 rows: not a multiple of the 8 rows of a CTA
    x = f32(rng.standard_normal((B, T, C)) * 2 + 0.5)
    w, b = f32(rng.standard_normal(C)), f32(rng.standard_normal(C))
    rownorm_case(engine, f"layernorm affine C={C}", x, B, T, 0, w, b)
    # FinalLayer: no affine, one (shift, scale) row for the whole batch
    stride = 2 * C
    mod = f32(rng.standard_normal(stride) * 0.5)
    rownorm_case(engine, f"layernorm modulated C={C}", x, B, T, 0, m0=mod[C:], m1=mod[:C], mod_stride=0)
    # DiT adaLN: RMSNorm, then a per-batch modulation read at a stride (the rows of every layer's modulation)
    stride = 3 * C
    mw, mb = f32(rng.standard_normal(B * stride)), f32(rng.standard_normal(B * stride))
    rownorm_case(engine, f"rmsnorm_adaln C={C}", x, B, T, 1, w, eps=1e-5, m0=mw, m1=mb, mod_stride=stride)
    # |mean| >> std: a one-pass variance cancels here, the two-pass one does not
    xm = f32(1000.0 + rng.standard_normal((1, 37, C)))
    rownorm_case(engine, f"layernorm |mean| >> std C={C}", xm, 1, 37, 0, w, b)


def test_groupnorm_mish(engine):
    """The length regulator's GroupNorm(1) + Mish: n_per = T * C far above 296 blocks of 256, values past Mish's 20."""
    rng = np.random.default_rng(7)
    T, C = 700, 512
    x = (rng.standard_normal((1, T, C)) * 3 + 1).astype(np.float32)
    w = (rng.standard_normal(C) * 4).astype(np.float32)
    b = rng.standard_normal(C).astype(np.float32)
    b[:64] += 30.0
    y, _ = engine.debug_tail_op("groupnorm1_mish", x, w=w, b=b, eps=1e-5)
    ref, v = kr.gn_mish(x, w, b, np.float32(1e-5))
    assert v.max() > 20 and T * C > 296 * 256
    mean, rstd = x.astype(np.float64).mean(), 1 / math.sqrt(x.astype(np.float64).var() + 1e-5)
    # v = (x - fp32 mean) * rstd * w + b: 4 roundings on the product, one on the mean, one on + b
    dv = 5 * U * np.abs((x - mean) * rstd * w) + U * abs(mean) * rstd * np.abs(w) + 2 * U * np.abs(v)
    sp = np.logaddexp(0.0, v)
    t = np.tanh(sp)
    # Mish' <= 1.1; softplus through expf (2 ulp) / log1pf (1 ulp) or the v > 20 cut (e^-20), tanhf (2 ulp), the product
    bound = 1.1 * dv + np.abs(v) * ((1 - t * t) * (2.0 ** -22 + 2.0 ** -23 * sp + math.exp(-20)) + 2.0 ** -22 * t) + 2 * U * np.abs(ref)
    check("groupnorm1_mish", y, ref, bound)


ACT_C = [5, 24, 33, 48, 96, 1536]


def lanes_t(C):
    return 256 // min(C, 32)


@pytest.mark.parametrize("C", ACT_C)
def test_activation1d(engine, C):
    rng = np.random.default_rng(C + 4)
    taps = kaiser_sinc_filter1d(0.25, 0.3, 12).reshape(-1).numpy().astype(np.float32)
    Ts = [1, 2, 3, 6, 7, 31, 32, 33, lanes_t(C) * 32 - 1, lanes_t(C) * 32 + 1]
    if C == BIGVGAN_LAST_C:
        Ts.append(880 * 256)
    alpha = (rng.standard_normal(C) * 0.5).astype(np.float32)
    beta = (rng.standard_normal(C) * 0.5).astype(np.float32)
    for T in Ts:
        B = 2 if T < 100 else 1
        logscale = 0 if T == 7 else 1
        a, bt = (np.abs(alpha) + 0.2, np.abs(beta) + 0.2) if not logscale else (alpha, beta)
        x = (rng.standard_normal((B, T, C)) * 2).astype(np.float32)
        kw = dict(w=a, b=bt, logscale=logscale)
        y, y16 = engine.debug_tail_op("snake_act", x, out=True, out16=True, **kw)
        ref, bound = kr.activation1d(x, a, bt, taps, logscale)
        check(f"activation1d C={C} T={T} logscale={logscale}", y, ref, bound)
        exact("  fp16", y16, y.astype(np.float16))
        y32, _ = engine.debug_tail_op("snake_act", x, out=True, out16=False, **kw)
        _, only16 = engine.debug_tail_op("snake_act", x, out=False, out16=True, **kw)
        exact("  fp16 only", only16, y32.astype(np.float16))


@pytest.mark.parametrize("C", [BIGVGAN_LAST_C, 33])
def test_conv_post(engine, C):
    rng = np.random.default_rng(C + 5)
    w = (rng.standard_normal((7, C)) * 0.3).astype(np.float32)
    bias = rng.standard_normal(1).astype(np.float32)
    for T in list(range(1, 9)) + [1000]:
        x = rng.standard_normal((2, T, C)).astype(np.float32)
        for use_tanh, bb in ((0, None), (1, bias)):
            y, _ = engine.debug_tail_op("conv_post", x, w=w, b=bb, use_tanh=use_tanh)
            ref, pre, mag = kr.conv_post(x, w, bb, use_tanh)
            bound = (7 * C + 2) * U * mag + (2.0 ** -22 * np.abs(ref) if use_tanh else 0.0) + 1e-30
            check(f"conv_post C={C} T={T} {'tanh' if use_tanh else 'clamp'}", y, ref, bound)


def euler_bound(mag, ref):
    return 5 * U * mag + U * np.abs(ref) + 1e-30


def test_cfg_euler(engine):
    rng = np.random.default_rng(8)
    T, C = 301, 80
    x, vc, vu = (rng.standard_normal((T, C)).astype(np.float32) for _ in range(3))
    dt, rate = np.float32(1 / 25), np.float32(0.7)
    for P in (0, 17, T):
        y, _ = engine.debug_tail_op("cfg_euler", x, x2=vc, x3=vu, dt=dt, rate=rate, P=P)
        ref, mag = kr.cfg_euler(x, vc, vu, dt, rate, np.arange(T) < P)
        check(f"cfg_euler P={P}", y[0], ref, euler_bound(mag, ref))
        assert np.all(y[0, :P] == 0)
    # packed: each segment zeroes its own prompt rows, P_u = 0 and P_u = T_u among them
    lens, Ps = [40, 1, 100, 2, 158], [0, 1, 30, 2, 0]
    zero = np.concatenate([np.arange(n) < p for n, p in zip(lens, Ps)])
    y, _ = engine.debug_tail_op("cfg_euler_rows", x, x2=vc, x3=vu, dt=dt, rate=rate, zero_rows=zero)
    ref, mag = kr.cfg_euler(x, vc, vu, dt, rate, zero)
    check("cfg_euler_rows", y[0], ref, euler_bound(mag, ref))
    assert np.all(y[0, zero] == 0) and np.all(y[0, ~zero] != 0)


def test_rope_table_per_segment(engine):
    lens = [1, 2, 129, 64, 300]
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    T = int(off[-1])
    for seg in (None, off):
        y, _ = engine.debug_tail_op("rope_table", B=1, T=T, C=1, n2=64, seg_off=seg)
        pos = np.arange(T) if seg is None else np.concatenate([np.arange(n) for n in lens])
        ang = kr.rope_angles(T)[pos]                       # fp32 angles of each row's position
        ref = np.stack([np.cos(ang), np.sin(ang)], -1)
        # both angles are fp32(t * fp32(freq)): freq within 3 ulp on either side (powf, division), one rounding each product;
        # cosf / sinf 2 ulp
        bound = 16 * U * np.abs(ang)[..., None] + 2.0 ** -22 + 1e-30
        check(f"rope_table {'per segment' if seg is not None else 'one table'}", y, ref, bound)
