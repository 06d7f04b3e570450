"""CPU: the float64 kernel references of tests/kernel_refs.py against PyTorch and the oracle, at small shapes."""
import math
import os

import numpy as np
import torch
import torch.nn.functional as F

from oracle.s2mel import _rope
from tests import kernel_refs as kr


def test_ref_conv_matches_conv1d():
    rng = np.random.default_rng(0)
    B, Tin, K, N, taps, dil, pad = 2, 23, 5, 7, 3, 2, 3
    A = rng.standard_normal((B, Tin, K))
    w = rng.standard_normal((N, K, taps))                       # torch Conv1d weight [out][in][k]
    wk = w.transpose(0, 2, 1).reshape(N, taps * K)              # K-major [N][taps*K]
    M = Tin + 2 * pad - dil * (taps - 1)
    want = F.conv1d(torch.from_numpy(A).transpose(1, 2), torch.from_numpy(w), padding=pad, dilation=dil)
    got, mag = kr.ref_conv(A, wk, taps, dil, pad, M)
    np.testing.assert_allclose(got, want.transpose(1, 2).numpy(), rtol=1e-12, atol=1e-12)
    assert np.all(mag >= np.abs(got))
    # per-batch weights and a broadcast A
    wb = rng.standard_normal((B, N, taps * K))
    got_b, _ = kr.ref_conv(A[:1], wb, taps, dil, pad, M)
    for b in range(B):
        np.testing.assert_allclose(got_b[b], kr.ref_conv(A[:1], wb[b], taps, dil, pad, M)[0][0], rtol=1e-12, atol=1e-12)


def test_activations():
    x = np.linspace(-9, 9, 301)
    t = torch.from_numpy(x)
    np.testing.assert_allclose(kr.act(x, 1), F.gelu(t).numpy(), rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(kr.act(x, 2), F.silu(t).numpy(), rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(kr.act(x, 3), F.mish(t).numpy(), rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(kr.act(x, 4), F.gelu(t, approximate="tanh").numpy(), rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(kr.act(x, 5), F.relu(t).numpy(), rtol=0, atol=0)


def test_flash_reference_matches_sdpa():
    rng = np.random.default_rng(1)
    BH, T = 3, 37
    q, k, v = (rng.standard_normal((BH, T, 64)).astype(np.float16) for _ in range(3))
    qt, kt, vt = (torch.from_numpy(x.astype(np.float64)) for x in (q, k, v))
    for base in (math.e, 2.0):
        got, vmag = kr.flash_attention(q, k, v, base)
        want = F.scaled_dot_product_attention(qt, kt, vt, scale=math.log(base))
        np.testing.assert_allclose(got, want.numpy(), rtol=1e-10, atol=1e-12)
        assert np.all(vmag >= np.abs(got) - 1e-12)


def test_decode_attention_reference_matches_sdpa():
    rng = np.random.default_rng(4)
    H, T = 3, 90
    q = rng.standard_normal((5, H * 64)).astype(np.float32) * 2
    K, V = (rng.standard_normal((T, H * 64)).astype(np.float32) for _ in range(2))
    ctx = np.array([1, 2, 33, 64, T])
    got, vmag = kr.ref_decode_attention(q, K, V, ctx)
    for i, n in enumerate(ctx):
        qt = torch.from_numpy(q[i].astype(np.float64)).view(H, 1, 64)
        kt, vt = (torch.from_numpy(x[:n].astype(np.float64)).view(n, H, 64).transpose(0, 1) for x in (K, V))
        want = F.scaled_dot_product_attention(qt, kt, vt).reshape(-1).numpy()       # default scale 1/sqrt(64)
        np.testing.assert_allclose(got[i], want, rtol=1e-10, atol=1e-12)
    assert np.all(vmag >= np.abs(got) - 1e-12)
    # one key: the output is that key's value row; keys at or beyond ctx never contribute (one query, ctx as an int)
    np.testing.assert_allclose(got[0], V[0], rtol=1e-12, atol=0)
    K2, V2 = K.copy(), V.copy()
    K2[64:], V2[64:] = 1e3, 1e3
    np.testing.assert_allclose(kr.ref_decode_attention(q[3], K2, V2, 64)[0][0], got[3], rtol=1e-13, atol=1e-15)


def test_decode_attention_reference_key_sets():
    """keys= (a step's keys spread over the rows of K / V) equals the same keys gathered into a contiguous cache."""
    rng = np.random.default_rng(6)
    H, T, N = 2, 70, 9
    q = rng.standard_normal((N, H * 64)) * 2
    K, V = rng.standard_normal((T, H * 64)), rng.standard_normal((T, H * 64))
    keys = rng.random((N, T)) < 0.3
    keys[:, 5] = True
    got, vmag = kr.ref_decode_attention(q, K, V, keys=keys, chunk=4)
    for i in range(N):
        idx = np.flatnonzero(keys[i])
        want, wmag = kr.ref_decode_attention(q[i], K[idx], V[idx], len(idx))
        np.testing.assert_allclose(got[i], want[0], rtol=1e-12, atol=1e-13)
        np.testing.assert_allclose(vmag[i], wmag[0], rtol=1e-12, atol=1e-13)


def test_beam_key_slots_follow_hf_cache_reordering():
    """beam_key_slots against HF's own bookkeeping: every beam keeps a private cache row, appends the key it computes at
    each step, and the whole cache is reordered by the chosen parents after the step (`cache = cache[beam_idx]`).  The
    keys are unique tags of the (cache slot, position) the engine writes them to; the helper's slots must name the
    same tags at every (step, beam, position), including the identity reorders after an utterance is done."""
    rng = np.random.default_rng(7)
    for m, u, plen, steps, done_at in ((2, 0, 1, 12, None), (3, 1, 5, 40, 25), (4, 1, 3, 60, 7), (4, 0, 2, 30, 0)):
        row0 = u * m
        parents = rng.integers(0, m, (steps, m))
        parents[steps // 3] = 0                         # every beam from one parent
        parents[steps // 2] = np.arange(m)[::-1]        # a permutation
        if done_at is not None:
            parents[done_at:] = np.arange(m)            # finished utterance: identity reorder
        tag = lambda slot, pos: slot * 100000 + pos     # noqa: E731
        cache = [[tag(row0, j) for j in range(plen)] for _ in range(m)]    # HF replicates the prompt into every beam
        slots = kr.beam_key_slots(parents, plen, m, row0)
        assert slots.shape == (steps, m, plen + steps)
        for k in range(steps):
            for r in range(m):
                cache[r].append(tag(row0 + r, plen + k))                   # the key beam r computes at step k
                got = [tag(int(slots[k, r, j]), j) for j in range(plen + k + 1)]
                assert got == cache[r], (m, k, r)
                assert (slots[k, r, plen + k + 1:] == -1).all()
            cache = [list(cache[int(b)]) for b in parents[k]]              # cache = cache[beam_idx]


def test_rope_matches_oracle():
    rng = np.random.default_rng(2)
    B, T, H = 2, 300, 3
    x = rng.standard_normal((B, T, H, 64)).astype(np.float32)
    want = _rope(torch.from_numpy(x), 64).numpy()                      # fp32, [B][T][H][64]
    got = kr.rope(x.transpose(0, 2, 1, 3)).transpose(0, 2, 1, 3)
    # same angles; the oracle rotates in fp32
    assert np.abs(got - want).max() <= 4e-6 * np.abs(x).max()
    tab = kr.rope_table(T)
    ang = kr.rope_angles(T)
    assert tab.shape == (T, 32, 2) and tab.dtype == np.float32
    np.testing.assert_array_equal(tab[..., 0], np.cos(ang).astype(np.float32))
    np.testing.assert_array_equal(tab[..., 1], np.sin(ang).astype(np.float32))
    # the angle of pair i at position t really is fp32(t * fp32(freq_i)): the rotation of position 1 by pair 0 is 1 rad
    assert ang[1, 0] == 1.0 and ang[0].max() == 0.0


def test_pair_epilogue_references():
    rng = np.random.default_rng(3)
    a, b = rng.standard_normal((2, 50, 40)) * 4
    np.testing.assert_allclose(kr.swiglu(a, b), (F.silu(torch.from_numpy(a)) * torch.from_numpy(b)).numpy(), rtol=1e-12, atol=1e-14)
    ta, tc = torch.from_numpy(a), torch.from_numpy(b)
    np.testing.assert_allclose(kr.wn_gate(a, b), (torch.tanh(ta) * torch.sigmoid(tc)).numpy(), rtol=1e-12, atol=1e-14)


def test_pad1d_reflect_matches_reference_golden():
    """pad1d_reflect against the reference's SConv1d (encodec.py pad1d) at 1, 2 and 3 frames, and against F.pad beyond."""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "s2mel_short.npz"))
    w, b = torch.from_numpy(g["sconv_weight"]).double(), torch.from_numpy(g["sconv_bias"]).double()
    for T in (1, 2, 3):
        x = g[f"sconv_x{T}"][0].T                                        # [T][C]
        xp = torch.from_numpy(kr.pad1d_reflect(x, 2, 2)).T[None]
        np.testing.assert_allclose(F.conv1d(xp, w, b).numpy(), g[f"sconv_y{T}"], rtol=1e-5, atol=1e-5)
    assert kr.pad1d_reflect_rows(2, 2, 2).tolist() == [-1, 1, 0, 1, -1, 1]
    assert kr.pad1d_reflect_rows(1, 2, 2).tolist() == [-1, -1, 0, -1, -1]
    for T in (3, 4, 9):
        x = np.random.default_rng(T).standard_normal((T, 3))
        want = F.pad(torch.from_numpy(x).T[None], (2, 2), mode="reflect")[0].T.numpy()
        np.testing.assert_array_equal(kr.pad1d_reflect(x, 2, 2), want)


def test_row_norm_references():
    rng = np.random.default_rng(8)
    B, T, C = 2, 5, 48
    x = rng.standard_normal((B * T, C)) * 3 + 1
    w, b = rng.standard_normal(C), rng.standard_normal(C)
    m0, m1 = rng.standard_normal(B * C), rng.standard_normal(B * C)
    xt = torch.from_numpy(x)
    got, bound = kr.rownorm(x, T, 0, w, b, 1e-6)
    np.testing.assert_allclose(got, F.layer_norm(xt, (C,), torch.from_numpy(w), torch.from_numpy(b), 1e-6).numpy(), atol=1e-12)
    assert np.all(bound > 0)
    ln = F.layer_norm(xt, (C,), None, None, 1e-6).view(B, T, C)
    sc, sh = torch.from_numpy(m0).view(B, 1, C), torch.from_numpy(m1).view(B, 1, C)
    got, _ = kr.rownorm(x, T, 0, None, None, 1e-6, m0, m1, C)
    np.testing.assert_allclose(got, (ln * (1 + sc) + sh).view(B * T, C).numpy(), atol=1e-12)
    got, _ = kr.rownorm(x, T, 0, None, None, 1e-6, m0[:C], m1[:C], 0)           # one modulation row for every batch entry
    np.testing.assert_allclose(got, (ln * (1 + sc[:1]) + sh[:1]).view(B * T, C).numpy(), atol=1e-12)
    rms = xt * torch.rsqrt(xt.pow(2).mean(-1, keepdim=True) + 1e-5) * torch.from_numpy(w)     # gpt_fast RMSNorm
    got, _ = kr.rownorm(x, T, 1, w, None, 1e-5, m0, m1, C)
    np.testing.assert_allclose(got, (sc * rms.view(B, T, C) + sh).view(B * T, C).numpy(), atol=1e-12)


def test_groupnorm_mish_and_dwconv_references():
    rng = np.random.default_rng(9)
    B, T, C, k = 2, 11, 6, 7
    x = rng.standard_normal((B, T, C)) * 4
    w, b = rng.standard_normal(C), rng.standard_normal(C)
    want = F.mish(F.group_norm(torch.from_numpy(x).transpose(1, 2), 1, torch.from_numpy(w), torch.from_numpy(b), 1e-5))
    np.testing.assert_allclose(kr.gn_mish(x, w, b, 1e-5)[0], want.transpose(1, 2).numpy(), atol=1e-12)
    wd, bd = rng.standard_normal((C, k)), rng.standard_normal(C)
    for TT in (1, 2, 3, 11):
        xs = x[:, :TT]
        want = F.conv1d(torch.from_numpy(xs).transpose(1, 2), torch.from_numpy(wd)[:, None], torch.from_numpy(bd),
                        padding=(k - 1) // 2, groups=C).transpose(1, 2).numpy()
        got, mag = kr.dwconv(xs, wd, bd, k)
        np.testing.assert_allclose(got, want, atol=1e-12)
        assert np.all(mag >= np.abs(got) - 1e-12)


def test_activation1d_matches_oracle():
    from indextts_b200.synth import kaiser_sinc_filter1d
    from oracle.bigvgan import activation1d
    rng = np.random.default_rng(10)
    filt = kaiser_sinc_filter1d(0.25, 0.3, 12).double()
    for T, logscale in ((1, True), (2, False), (7, True), (40, True)):
        B, C = 2, 5
        x = rng.standard_normal((B, T, C)) * 2
        alpha, beta = rng.standard_normal(C) * 0.5, rng.standard_normal(C) * 0.5
        if not logscale:
            alpha, beta = np.abs(alpha) + 0.2, np.abs(beta) + 0.2
        got, bound = kr.activation1d(x, alpha, beta, filt.reshape(-1).numpy(), logscale)
        want = activation1d(torch.from_numpy(x).transpose(1, 2), torch.from_numpy(alpha), torch.from_numpy(beta),
                            filt.view(1, 1, -1), logscale).transpose(1, 2).numpy()
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)
        assert np.all(bound > 0)


def test_conv_post_and_cfg_euler_references():
    rng = np.random.default_rng(11)
    B, T, C = 2, 9, 5
    x = rng.standard_normal((B, T, C))
    w, bias = rng.standard_normal((7, C)), rng.standard_normal(1)
    pre = F.conv1d(torch.from_numpy(x).transpose(1, 2), torch.from_numpy(w.T.copy())[None], torch.from_numpy(bias), padding=3)
    for use_tanh in (0, 1):
        got, p, mag = kr.conv_post(x, w, bias, use_tanh)
        np.testing.assert_allclose(p, pre[:, 0].numpy(), atol=1e-12)
        np.testing.assert_allclose(got, (torch.tanh(pre) if use_tanh else pre.clamp(-1, 1))[:, 0].numpy(), atol=1e-12)
        assert np.all(mag >= np.abs(p) - 1e-12)
    # flow_matching.py:96-113: dphi = (1 + r) * cond - r * uncond ; x = x + dt * dphi ; x[:, :, :P] = 0
    xs, vc, vu = rng.standard_normal((3, 10, 4))
    zero = np.arange(10) < 3
    got, _ = kr.cfg_euler(xs, vc, vu, 0.125, 0.7, zero)
    want = xs + 0.125 * ((1 + 0.7) * vc - 0.7 * vu)
    want[:3] = 0
    np.testing.assert_allclose(got, want, atol=1e-14)
