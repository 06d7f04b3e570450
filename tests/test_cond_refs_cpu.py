"""CPU: the float64 references of the prompt encoders' kernels (tests/cond_refs.py) against PyTorch and the pinned oracles
(oracle/emo.py, pinned against the reference's ConformerEncoder / PerceiverResampler; oracle/v1.py, pinned against its
ECAPA_TDNN), at small shapes.  Each bound must also be positive and below the size of what it bounds."""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import emo, v1
from tests import cond_refs as cr


def test_conv2d_sub2_matches_conv2d():
    rng = np.random.default_rng(0)
    for T, Fb in ((3, 3), (8, 100), (9, 41)):
        x = rng.standard_normal((T, Fb))
        w = rng.standard_normal((5, 1, 3, 3))
        b = rng.standard_normal(5)
        y = F.relu(F.conv2d(torch.from_numpy(x)[None, None], torch.from_numpy(w), torch.from_numpy(b), stride=2))
        _, C, T2, Fs = y.shape
        want = y.transpose(1, 2).reshape(T2, C * Fs).numpy()          # Conv2dSubsampling2's layout (subsampling.py:181-185)
        got, bound = cr.conv2d_sub2(x, w, b)
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)
        assert got.shape == (T2, C * Fs) and np.all(bound > 0) and np.all(bound < 1e-5 * (1 + np.abs(got)))


def test_pos_table_is_the_oracle_table_and_bounds_its_rounding():
    for T, d in ((1, 2), (64, 32), (1024, 512)):
        got, bound = cr.pos_table(T, d)
        np.testing.assert_array_equal(got, emo.pos_table(T, d).double().numpy())
        # the fp32 table against the same formula in float64: within the reference's share of the bound
        t = np.arange(T)[:, None]
        arg = t * np.exp(np.arange(0, d, 2) * -(math.log(10000.0) / d))
        exact = np.empty((T, d))
        exact[:, 0::2], exact[:, 1::2] = np.sin(arg), np.cos(arg)
        assert np.all(np.abs(got - exact) <= bound)
        assert bound.max() < 1e-3 * max(1, T / 1000)
    pe = emo.pos_table(7, 4, dtype=torch.float64)
    assert pe.dtype == torch.float64 and torch.equal(pe, emo.pos_table(7, 4).double())


def test_relpos_attention_matches_the_oracle():
    rng = np.random.default_rng(2)
    for T, H, dk in ((1, 2, 16), (7, 2, 16), (29, 4, 8)):
        od = H * dk
        qkv = rng.standard_normal((T, 3 * od))
        pp = rng.standard_normal((T, od))
        u, v = rng.standard_normal(od), rng.standard_normal(od)
        q, k, vv = (torch.from_numpy(qkv[:, i * od:(i + 1) * od]) for i in range(3))
        want = emo.rel_attention(q, k, vv, torch.from_numpy(pp), torch.from_numpy(u).view(H, dk),
                                 torch.from_numpy(v).view(H, dk), H).numpy()
        for tc in ((False, False), (True, False), (True, True)):
            got, bound = cr.relpos_attention(qkv, pp, u, v, H, *tc)
            np.testing.assert_allclose(got, want, rtol=1e-10, atol=1e-12)
            assert np.all(bound > 0)
        # the tf32 bound is the loose one, and both stay far below the values they bound
        b_simt = cr.relpos_attention(qkv, pp, u, v, H, False, False)[1]
        b_tc = cr.relpos_attention(qkv, pp, u, v, H, True, True)[1]
        assert np.all(b_tc > b_simt) and b_tc.max() < 0.2 * np.abs(vv.numpy()).max()


def test_tc_switch_points():
    """conv_gemm's automatic choice (gemm_tc.cu gemm_tc_supported) at the full emotion config: the score GEMM (T2 x T2 x 256)
    moves to the tensor cores at T2 = 32, P V (T2 x 128 x Tp) at T2 = 45."""
    tp = lambda t: (t + 3) & ~3                                                # noqa: E731
    assert not cr.tc_gemm(31, 31, 256) and cr.tc_gemm(32, 32, 256)
    assert not cr.tc_gemm(44, 128, tp(44)) and cr.tc_gemm(45, 128, tp(45))


def test_glu_and_geglu_match_torch():
    rng = np.random.default_rng(3)
    x = np.concatenate([rng.standard_normal((5, 40)) * 4, np.linspace(-30, 30, 200).reshape(5, 40)], axis=1)
    y, bound = cr.glu(x)
    np.testing.assert_allclose(y, F.glu(torch.from_numpy(x), dim=-1).numpy(), rtol=1e-12, atol=1e-300)
    assert np.all(bound <= 1e-6 * np.abs(y) + 1e-29)
    y, bound = cr.geglu(x)
    a, g = torch.from_numpy(x).chunk(2, -1)
    np.testing.assert_allclose(y, (F.gelu(g) * a).numpy(), rtol=1e-12, atol=1e-14)
    assert np.all(bound > 0) and np.all(bound <= 1e-5 * (np.abs(x[:, :40]) * np.abs(x[:, 40:]) + 1))


def test_l2norm_scale_matches_the_perceiver_norm():
    rng = np.random.default_rng(4)
    for C in (64, 1024, 1280):
        x = rng.standard_normal((3, C)) * 3
        gamma = 1 + 0.1 * rng.standard_normal(C)
        y, bound = cr.l2norm_scale(x, gamma)
        want = (F.normalize(torch.from_numpy(x), dim=-1) * C ** 0.5 * torch.from_numpy(gamma)).numpy()
        np.testing.assert_allclose(y, want, rtol=1e-12, atol=1e-14)
        assert np.all(bound <= 1e-5 * np.abs(y) + 1e-29)


def test_latent_attention_matches_the_oracle():
    rng = np.random.default_rng(5)
    for nl, n, H, dh in ((1, 2, 2, 64), (32, 300, 8, 64), (3, 17, 4, 16)):
        q = rng.standard_normal((nl, H * dh))
        kv = rng.standard_normal((n, 2 * H * dh))
        got, bound = cr.latent_attention(q, kv, H)
        want = emo.latent_attention(torch.from_numpy(q), torch.from_numpy(kv), H).numpy()
        np.testing.assert_allclose(got, want, rtol=1e-10, atol=1e-12)
        assert np.all(bound > 0) and bound.max() < 1e-3 * np.abs(kv).max()


def test_ecapa_statistics_match_the_oracle_pooling():
    rng = np.random.default_rng(6)
    for T, C in ((5, 3), (9, 40), (203, 33)):
        x = rng.standard_normal((T, C)) * 2 + 0.5
        lg = rng.standard_normal((T, C)) * 3
        xt = torch.from_numpy(x.T)[None]                                        # [1, C, T] as ECAPA holds it
        m, s = v1.weighted_stats(xt, torch.full((1, 1, T), 1.0 / T, dtype=torch.float64))
        mean, std, bm, bs = cr.col_mean_std(x)
        np.testing.assert_allclose(mean, m[0].numpy(), rtol=1e-12, atol=1e-13)
        np.testing.assert_allclose(std, s[0].numpy(), rtol=1e-12, atol=1e-13)
        assert np.all(bm > 0) and np.all(bs > 0) and bm.max() < 1e-5 and bs.max() < 1e-5
        m, s = v1.weighted_stats(xt, F.softmax(torch.from_numpy(lg.T)[None], dim=2))
        mean, std, bm, bs = cr.asp_pool(lg, x)
        np.testing.assert_allclose(mean, m[0].numpy(), rtol=1e-12, atol=1e-13)
        np.testing.assert_allclose(std, s[0].numpy(), rtol=1e-12, atol=1e-13)
        assert np.all(bm > 0) and np.all(bs > 0) and bm.max() < 1e-4 and bs.max() < 1e-4
    # a constant column: std is sqrt(1e-12), the clamp of the reference
    mean, std, _, _ = cr.col_mean_std(np.ones((6, 2)))
    np.testing.assert_allclose(std, 1e-6)
