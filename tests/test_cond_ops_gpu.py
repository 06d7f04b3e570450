"""GPU: the prompt encoders' kernels (emo.cu: the emotion conformer and perceiver, which also run the v1 / v1.5 prompt
encoder; ecapa.cu: ECAPA's statistics) one at a time through Engine.debug_cond_op, against the float64 references of
tests/cond_refs.py on the exact fp32 operands.  Every element must satisfy err <= bound, where bound is the worst case of the
kernel's own fp32 evaluation; each case prints max err / bound.  Row-indexed inputs are staged between NaN rows and the
output between sentinel guard bands, so a read or write outside them fails too.

The shapes are derived from the two emotion configs: the relative-position attention runs at T2 on both sides of the
point where each of its GEMMs leaves the SIMT kernel for tf32 wgmma, forced onto each path and on the one the model takes."""
import numpy as np
import pytest

from indextts_b200.synth import EMO_CFG, small_emo_cfg
from tests import cond_refs as cr

pytestmark = pytest.mark.gpu

V1_P_DIM = 1280                   # the v1 perceiver works at model_dim (gpt/model.py:360)
CONFIGS = {"full": EMO_CFG, "small": small_emo_cfg()}


def check(name, got, ref, bound):
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    assert np.all(np.isfinite(got)), f"{name}: non-finite output"
    err = np.abs(got.astype(np.float64) - ref)
    ratio = float((err / bound).max())
    print(f"{name}: max err {err.max():.2e}, max err / bound {ratio:.3f}")
    assert ratio <= 1.0, (name, float(err.max()), ratio)
    return ratio


def _tp(t):
    return (t + 3) & ~3


def switch_points(c):
    """First T2 at which the score GEMM (T2 x T2 x 2dk) and the P V GEMM (T2 x dk x Tp) take the tensor cores."""
    dk = c["odim"] // c["heads"]
    s = next(t for t in range(1, 4096) if cr.tc_gemm(t, t, 2 * dk))
    p = next(t for t in range(1, 4096) if cr.tc_gemm(t, dk, _tp(t)))
    return s, p


def relpos_cases():
    out = []
    for name, c in CONFIGS.items():
        s, p = switch_points(c)
        for t in sorted({1, 2, 63, 64, 65, 128, 129, 374, 511, s - 1, s, p - 1, p}):
            out.append(pytest.param(name, t, id=f"{name}-T2={t}"))
    return out


def test_switch_points_of_the_full_config():
    assert switch_points(EMO_CFG) == (32, 45)


@pytest.mark.parametrize("cfg,T2", relpos_cases())
def test_relpos_attention(engine, cfg, T2):
    c = CONFIGS[cfg]
    H, od = c["heads"], c["odim"]
    dk = od // H
    rng = np.random.default_rng(T2 * 7 + H)
    qkv = rng.standard_normal((T2, 3 * od)).astype(np.float32)
    pp = rng.standard_normal((T2, od)).astype(np.float32)
    u, v = (0.5 * rng.standard_normal(od)).astype(np.float32), (0.5 * rng.standard_normal(od)).astype(np.float32)
    auto = (cr.tc_gemm(T2, T2, 2 * dk), cr.tc_gemm(T2, dk, _tp(T2)))
    for backend, tc in ((1, (False, False)), (2, (True, True)), (0, auto)):
        ref, bound = cr.relpos_attention(qkv, pp, u, v, H, *tc)
        got = engine.debug_cond_op("relpos_attention", qkv, pp, u, v, heads=H, backend=backend)
        path = {1: "SIMT", 2: "tensor core", 0: f"auto (scores {'tc' if tc[0] else 'SIMT'}, PV {'tc' if tc[1] else 'SIMT'})"}
        check(f"relpos_attention {cfg} T2={T2} {path[backend]}", got, ref, bound)


@pytest.mark.parametrize("T,F,C", [(3, 1024, 512), (4, 1024, 512), (5, 1024, 16), (62, 1024, 16), (751, 1024, 8),
                                   (3, 100, 512), (6, 100, 512), (61, 100, 512), (1406, 100, 32)])
def test_conv2d_sub2(engine, T, F, C):
    rng = np.random.default_rng(T + F + C)
    x = rng.standard_normal((T, F)).astype(np.float32)
    w = (rng.standard_normal((C, 9)) / 3).astype(np.float32)
    b = (0.1 * rng.standard_normal(C)).astype(np.float32)
    ref, bound = cr.conv2d_sub2(x, w, b)
    got = engine.debug_cond_op("conv2d_sub2", x, w=w, b=b, n2=C)
    check(f"conv2d_sub2 T={T} F={F} C={C}", got, ref, bound)


@pytest.mark.parametrize("T,d", [(1, 512), (29, 32), (374, 512), (702, 512), (1024, 512)])
def test_pos_table(engine, T, d):
    ref, bound = cr.pos_table(T, d)
    got = engine.debug_cond_op("pos_table", T=T, C=d)
    check(f"pos_table T={T} d={d}", got, ref, bound)


@pytest.mark.parametrize("T,C", [(1, 512), (29, 512), (374, 512), (37, 33)])
def test_glu(engine, T, C):
    rng = np.random.default_rng(T * 3 + C)
    x = (rng.standard_normal((T, 2 * C)) * 3).astype(np.float32)
    x[0, C:] = np.linspace(-100, 100, C)                 # saturated gates
    ref, bound = cr.glu(x)
    check(f"glu T={T} C={C}", engine.debug_cond_op("glu", x), ref, bound)


@pytest.mark.parametrize("rows,pd", [(1, EMO_CFG["p_dim"]), (32, V1_P_DIM), (2, 64)])
def test_geglu_and_l2norm_scale(engine, rows, pd):
    di = int(pd * 2 * 2 / 3)                              # the perceiver's FF inner width at ff_mult 2
    rng = np.random.default_rng(rows + pd)
    x = (rng.standard_normal((rows, 2 * di)) * 2).astype(np.float32)
    n = min(di, 200)
    x[0, di:di + n] = np.linspace(-12, 12, n)            # the gate through the erf tails
    ref, bound = cr.geglu(x)
    check(f"geglu rows={rows} N={di}", engine.debug_cond_op("geglu", x), ref, bound)
    lat = (rng.standard_normal((rows, pd)) * 5).astype(np.float32)
    gamma = (1 + 0.1 * rng.standard_normal(pd)).astype(np.float32)
    ref, bound = cr.l2norm_scale(lat, gamma)
    check(f"l2norm_scale rows={rows} d={pd}", engine.debug_cond_op("l2norm_scale", lat, w=gamma), ref, bound)


LATENT = [(nl, n, H) for nl, H in ((1, 4), (32, 8)) for n in (2, 33, 129, 376, 703, 3000) if n > nl]


@pytest.mark.parametrize("nl,n,H", LATENT)
@pytest.mark.parametrize("kind", ["random", "one key dominates"])
def test_latent_attention(engine, nl, n, H, kind):
    dh = 64
    inner = H * dh
    rng = np.random.default_rng(nl * 1000 + n)
    q = rng.standard_normal((nl, inner)).astype(np.float32)
    kv = rng.standard_normal((n, 2 * inner)).astype(np.float32)
    if kind != "random":                                  # key n // 2 scores ~40 above the others in every head
        kv[n // 2, :inner] = q[0] * (40 * 8 / np.maximum(1e-3, (q[0] ** 2).reshape(H, dh).sum(1))).repeat(dh)
    ref, bound = cr.latent_attention(q, kv, H)
    got = engine.debug_cond_op("latent_attention", q, kv, n2=n, heads=H)
    check(f"latent_attention nl={nl} n={n} heads={H} ({kind})", got, ref, bound)


@pytest.mark.parametrize("T", [5, 6, 7, 8, 9, 33, 1406])
@pytest.mark.parametrize("C", [512, 1536, 333])
def test_ecapa_statistics(engine, T, C):
    rng = np.random.default_rng(T * 10 + C)
    x = (rng.standard_normal((T, C)) * 2 + 3).astype(np.float32)      # a mean well away from 0: the variance cancels
    x[:, 0] = 1.25                                                    # a constant channel: std at the 1e-12 clamp
    lg = (rng.standard_normal((T, C)) * 4).astype(np.float32)
    mean, std, bm, bs = cr.col_mean_std(x)
    got = engine.debug_cond_op("col_mean_std", x, n2=0)
    check(f"col_mean_std (mean only) T={T} C={C}", got, mean, bm)
    got = engine.debug_cond_op("col_mean_std", x, n2=1)
    check(f"col_mean_std T={T} C={C}", got, np.concatenate([mean, std]), np.concatenate([bm, bs]))
    mean, std, bm, bs = cr.asp_pool(lg, x)
    got = engine.debug_cond_op("asp_pool", x, lg)
    check(f"asp_pool T={T} C={C}", got, np.concatenate([mean, std]), np.concatenate([bm, bs]))
