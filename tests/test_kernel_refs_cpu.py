"""CPU: the float64 kernel references of tests/kernel_refs.py against PyTorch and the oracle, at small shapes."""
import math

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
