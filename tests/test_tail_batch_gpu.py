"""GPU: idx_codes_to_wav_batch (one packed CFM solve for several utterances of different lengths) against each utterance's
own idx_codes_to_wav call, and the varlen wgmma flash attention it runs on against a float64 reference.

Every GEMM of the solve sums each output element over K in an order that does not depend on M, the norms and pointwise
kernels work per row, and the varlen attention sees a segment's keys in the same 128-key tiles as a solo solve, so the
packed result is expected to equal the solo one bit for bit; the bounds below allow a little more and each test prints
whether the results were bitwise equal.  Utterances are at least 32 frames long: below about 2^18 / (N K) rows the solo
call runs its three fp32 input GEMMs (merge of x, cond projection, merge constant) on the SIMT kernel instead of tf32
tensor cores, and the packed solve, having more rows, does not."""
import ctypes
import os

import numpy as np
import pytest
import torch

from indextts_b200 import synth
from indextts_b200.engine import VocodeRequest, fold_weight_norm
from oracle.make_goldens_tail_full import make_inputs
from tests.test_flash_attention_gpu import reference

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden", "tail_full_cfg2.npz")


def _load(engine, full):
    if full:
        c, cc, h = dict(synth.S2MEL_CFG), dict(synth.CODEC_CFG), dict(synth.BIGVGAN_V2_22K)
        ws, wc, wb = synth.make_s2mel_weights(c, seed=1234), synth.make_codec_weights(cc, seed=4321), synth.make_bigvgan_weights(h, seed=1234)
    else:
        c, cc, h = synth.small_s2mel_cfg(), synth.small_codec_cfg(), synth.small_config()
        ws, wc, wb = synth.make_s2mel_weights(c, 1234), synth.make_codec_weights(cc, 4321), synth.make_bigvgan_weights(h, 1)
    engine.load_state_dict("s2mel.", {k: v for k, v in fold_weight_norm(ws).items() if v.is_floating_point()})
    engine.load_state_dict("codec.", fold_weight_norm(wc))
    engine.load_state_dict("bigvgan.", wb)
    engine.s2mel_init(c)
    engine.codec_init(cc)
    engine.bigvgan_init(h)
    return c, cc


def _utterance(seed, P, n_codes, F, codebook, content_dim, style_dim=192):
    g = torch.Generator().manual_seed(seed)
    return dict(codes=torch.randint(0, codebook, (n_codes,), generator=g).numpy().astype(np.int32),
                prompt_condition=torch.randn(P, content_dim, generator=g).numpy(),
                ref_mel=(torch.randn(80, P, generator=g) * 1.5 - 4.0).numpy(),
                style=torch.randn(style_dim, generator=g).numpy(),
                z=torch.randn(80, P + F, generator=g).numpy(), F=F)


# (P, n_codes, F): T = P + F of 129, 46 (one generated frame), 128, 137 (no prompt), 81
SMALL = [(61, 20, 68), (45, 1, 1), (60, 20, 68), (0, 40, 137), (40, 12, 41)]


def _small_set(n, cc, c):
    return [_utterance(100 + i, P, nc, F, cc["codebook_size"], c["content_dim"]) for i, (P, nc, F) in enumerate(SMALL[:n])]


def _compare(engine, utts, tag):
    kw = dict(want_wav=True, want_pcm16=True, want_mel=True)
    batch = engine.codes_to_wav_batch(utts, 25, 0.7, **kw)
    for i, (u, b) in enumerate(zip(utts, batch)):
        solo = engine.codes_to_wav(u["codes"], u["prompt_condition"], u["ref_mel"], u["style"], u["z"], u["F"], 25, 0.7, **kw)
        same = all(np.array_equal(np.asarray(solo[k]), np.asarray(b[k])) for k in ("mel", "wav", "pcm16"))
        dmel = float(np.abs(b["mel"] - solo["mel"]).max())
        dwav = float(np.sqrt(((b["wav"] - solo["wav"]) ** 2).mean()))
        print(f"[{tag}] utterance {i} (P={u['ref_mel'].shape[1]}, F={u['F']}): bitwise equal to its solo call: {same}; "
              f"max |dmel| {dmel:.3e}, wav rms diff {dwav:.3e}")
        assert np.isfinite(b["mel"]).all() and np.isfinite(b["wav"]).all()
        assert dmel <= 1e-5 * float(np.abs(solo["mel"]).max()), (i, dmel)
        assert dwav <= 1e-6, (i, dwav)
        assert np.array_equal(b["pcm16"], solo["pcm16"]), i
    return batch


@pytest.mark.parametrize("order", ["given", "reversed"])
@pytest.mark.parametrize("n", [1, 2, 3, 5])
def test_small_batch_equals_solo_calls(engine, n, order):
    c, cc = _load(engine, full=False)
    utts = _small_set(n, cc, c)
    if order == "reversed":
        utts = utts[::-1]
    _compare(engine, utts, f"small n={n} {order}")
    ms = engine.s2mel_last_ms()
    assert ms["cfm_ms"] > 0 and engine.bigvgan_last_ms() > 0


def test_small_batch_on_device_buffers(engine):
    c, cc = _load(engine, full=False)
    utts = _small_set(3, cc, c)
    host = engine.codes_to_wav_batch(utts, 25, 0.7, want_wav=True, want_pcm16=True)
    dev = [{k: (torch.from_numpy(np.ascontiguousarray(v)).cuda() if isinstance(v, np.ndarray) else v) for k, v in u.items()}
           for u in utts]
    out = engine.codes_to_wav_batch(dev, 25, 0.7, want_wav=True, want_pcm16=True)
    for h, d in zip(host, out):
        assert d["wav"].is_cuda and d["pcm16"].is_cuda
        assert np.array_equal(h["wav"], d["wav"].cpu().numpy()) and np.array_equal(h["pcm16"], d["pcm16"].cpu().numpy())


def test_full_geometry_batch_with_the_golden_utterance(engine):
    c, cc = _load(engine, full=True)
    codes, pc, ref_mel, style, z, F = make_inputs()
    gold = dict(codes=codes[0].numpy().astype(np.int32), prompt_condition=pc[0].numpy(), ref_mel=ref_mel[0].numpy(),
                style=style[0].numpy(), z=z[0].numpy(), F=F)
    others = [_utterance(7000 + i, P, nc, int(2 * nc * 1.72), cc["codebook_size"], c["content_dim"])
              for i, (P, nc) in enumerate([(300, 128), (500, 200), (100, 60)])]
    utts = [others[0], gold, others[1], others[2]]
    batch = _compare(engine, utts, "full geometry")
    g = np.load(GOLD)
    wav = np.clip(batch[1]["wav"], -1.0, 1.0)
    err = float(np.sqrt(((wav - g["wav"]) ** 2).mean()))
    rms = float(np.sqrt((g["wav"] ** 2).mean()))
    print(f"[full geometry] golden config-2 utterance from the packed solve vs fp32 oracle: wav rms error {err:.3e} "
          f"(relative {err / rms:.3e}); stage ms {engine.s2mel_last_ms()}, bigvgan {engine.bigvgan_last_ms():.2f}")
    assert err <= 1e-3 and err / rms <= 1e-2


@pytest.mark.parametrize("option,value", [("tail_f16", 0), ("gemm_backend", 1)])
def test_other_modes_run_the_solo_path(engine, option, value):
    c, cc = _load(engine, full=False)
    utts = _small_set(3, cc, c)
    kw = dict(want_wav=True, want_pcm16=True, want_mel=True)
    engine.set_option(option, value)
    try:
        batch = engine.codes_to_wav_batch(utts, 25, 0.7, **kw)
        for u, b in zip(utts, batch):
            solo = engine.codes_to_wav(u["codes"], u["prompt_condition"], u["ref_mel"], u["style"], u["z"], u["F"], 25, 0.7, **kw)
            for k in ("mel", "wav", "pcm16"):
                assert np.array_equal(solo[k], b[k]), k
    finally:
        engine.set_option("gemm_backend", 0)
        engine.set_option("tail_f16", 1)


def test_errors_write_nothing(engine):
    c, cc = _load(engine, full=False)
    with pytest.raises(RuntimeError, match=r"failed \(2\)"):
        engine.codes_to_wav_batch([], 25, 0.7)
    assert engine.lib.idx_codes_to_wav_batch(engine.h, None, 3, 25, 0.7) == 2
    utts = _small_set(3, cc, c)
    utts[2]["F"] = 0
    reqs = (VocodeRequest * 3)()
    keep, outs = [], []
    for i, u in enumerate(utts):
        r, res, k = engine._vocode_request(u["codes"], u["prompt_condition"], u["ref_mel"], u["style"], u["z"], u["F"],
                                           True, True, True)
        for a in res.values():
            a[...] = 7
        reqs[i] = r
        keep.append(k)
        outs.append(res)
    rc = engine.lib.idx_codes_to_wav_batch(engine.h, reqs, 3, 25, 0.7)
    msg = engine.lib.idx_last_error(engine.h).decode()
    print("F = 0 at index 2:", rc, msg)
    assert rc == 2 and "request 2" in msg and "bad request" in msg
    for res in outs:
        for a in res.values():
            assert np.all(a == 7)


def test_codebook_error_writes_nothing(engine):
    """A code outside the codebook fails idx_codes_to_wav after the whole tail has run, before any output is written."""
    c, cc = _load(engine, full=False)
    u = _small_set(1, cc, c)[0]
    u["codes"][5] = cc["codebook_size"] + 7
    r, res, keep = engine._vocode_request(u["codes"], u["prompt_condition"], u["ref_mel"], u["style"], u["z"], u["F"],
                                          True, True, True)
    for a in res.values():
        a[...] = 7
    rc = engine.lib.idx_codes_to_wav(engine.h, ctypes.byref(r), 25, 0.7)
    msg = engine.lib.idx_last_error(engine.h).decode()
    print("code outside the codebook at position 5:", rc, msg)
    assert rc == 2 and "outside the codebook" in msg and "request" not in msg
    for a in res.values():
        assert np.all(a == 7)
    u["codes"][5] = 3      # the engine stays usable afterwards
    out = engine.codes_to_wav(u["codes"], u["prompt_condition"], u["ref_mel"], u["style"], u["z"], u["F"], 25, 0.7)
    assert np.isfinite(out["wav"]).all()


# ------------------------------------------------------------------------------------- varlen flash attention --
SEGMENTS = [1, 7, 64, 65, 127, 128, 129, 257, 1741]


def _packed(B, H, order):
    """q, k, v [BH][sum T][64] of the segments (each the adversarial rows of test_flash_attention_gpu.py at its own length),
    packed in `order`, with the float64 reference and bound [B][sum T][H*64] and the segment offsets."""
    parts = [reference(B, H, SEGMENTS[i], 2.0) for i in order]
    q, k, v = (np.concatenate([p[j] for p in parts], axis=1) for j in range(3))
    ref, bound = (np.concatenate([p[j] for p in parts], axis=1) for j in (3, 4))
    off = np.concatenate([[0], np.cumsum([SEGMENTS[i] for i in order])]).astype(np.int32)
    return q, k, v, ref, bound, off


@pytest.mark.parametrize("B,H", [(1, 1), (2, 8)])
def test_varlen_flash_attention_against_fp64(engine, B, H):
    order = np.random.default_rng(5).permutation(len(SEGMENTS))
    q, k, v, ref, bound, off = _packed(B, H, order)
    out, out16 = engine.debug_flash_attention_varlen(q, k, v, B, H, off)
    for name, got, bd in (("out", out, bound), ("out16", out16.astype(np.float32), bound + 2.0 ** -11 * np.abs(ref))):
        assert np.all(np.isfinite(got)), name
        err = np.abs(got - ref)
        print(f"varlen B={B} H={H} {name}: max err {err.max():.2e}, max err / bound {(err / bd).max():.3f}")
        assert np.all(err <= bd), (name, float(err.max()))


@pytest.mark.parametrize("B,H", [(1, 1), (2, 8)])
def test_varlen_flash_attention_does_not_leak(engine, B, H):
    """Keys and values of every other segment made large and aligned with one segment's queries: that segment's output
    must not move by a bit."""
    order = np.random.default_rng(6).permutation(len(SEGMENTS))
    q, k, v, _, _, off = _packed(B, H, order)
    base, base16 = engine.debug_flash_attention_varlen(q, k, v, B, H, off)
    for u in range(len(order)):
        a, b = int(off[u]), int(off[u + 1])
        qd = q[:, a:b].astype(np.float32).mean(axis=1, keepdims=True)
        qd = qd / np.maximum(np.linalg.norm(qd, axis=-1, keepdims=True), 1e-6)
        k2, v2 = k.copy(), v.copy()
        k2[:, :a], k2[:, b:] = (40.0 * qd).astype(np.float16), (40.0 * qd).astype(np.float16)
        v2[:, :a], v2[:, b:] = 1000.0, 1000.0
        out, out16 = engine.debug_flash_attention_varlen(q, k2, v2, B, H, off)
        assert np.array_equal(out[:, a:b], base[:, a:b]), (u, float(np.abs(out[:, a:b] - base[:, a:b]).max()))
        assert np.array_equal(out16[:, a:b], base16[:, a:b]), u


# ------------------------------------------------------------------------------ short utterances, long batches --
def test_one_and_two_frame_utterances_against_the_oracle_tail(engine):
    """P = 0 and F = 1 or 2: the WaveNet's reflect padding zero-extends such a sequence (encodec.py pad1d) before it
    reflects.  idx_codes_to_wav (strict fp32 back end) against the oracle chain of tests/test_zz_tail_wiring.py."""
    from oracle.bigvgan import bigvgan_forward
    from oracle.s2mel import cfm_inference, codec_decode, length_regulate
    from oracle.s2mel import fold_weight_norm as oracle_fold
    c, cc = _load(engine, full=False)
    h = synth.small_config()
    wsf, wcf = oracle_fold(synth.make_s2mel_weights(c, 1234)), oracle_fold(synth.make_codec_weights(cc, 4321))
    wb = synth.make_bigvgan_weights(h, 1)
    for F in (1, 2):
        u = _utterance(300 + F, 0, 1, F, cc["codebook_size"], c["content_dim"])
        cond = length_regulate(wsf, codec_decode(wcf, torch.from_numpy(u["codes"]).long()[None]), F)
        mel_ref = cfm_inference(wsf, c, cond, torch.LongTensor([F]), torch.zeros(1, 80, 0),
                                torch.from_numpy(u["style"])[None], torch.from_numpy(u["z"])[None], 25, 0.7)
        wav_ref = bigvgan_forward(h, wb, mel_ref.float()).reshape(-1).numpy()
        engine.set_option("gemm_backend", 1)
        try:
            res = engine.codes_to_wav(u["codes"], u["prompt_condition"], u["ref_mel"], u["style"], u["z"], F, 25, 0.7,
                                      want_wav=True, want_mel=True)
        finally:
            engine.set_option("gemm_backend", 0)
        dmel = float(np.abs(res["mel"] - mel_ref[0].numpy()).max())
        dwav = float(np.abs(res["wav"] - wav_ref).max())
        print(f"P=0 F={F}: max |dmel| vs oracle {dmel:.2e} (max |mel| {float(mel_ref.abs().max()):.2f}), max |dwav| {dwav:.2e}")
        assert np.isfinite(res["mel"]).all() and dmel < 1e-3 and dwav < 1e-3


def test_short_utterances_in_a_packed_batch_do_not_see_their_neighbours(engine):
    """A 1-frame and a 2-frame utterance between long ones: new codes and noise for the neighbours, same lengths, and the
    short utterances' mel does not move by a bit (a reflect read past a 1- or 2-frame segment lands in its neighbour)."""
    c, cc = _load(engine, full=False)
    long_ = [(40, 20, 68), (0, 40, 137), (30, 12, 41)]
    short = [_utterance(400, 0, 1, 1, cc["codebook_size"], c["content_dim"]),
             _utterance(401, 0, 1, 2, cc["codebook_size"], c["content_dim"])]
    kw = dict(want_wav=True, want_pcm16=True, want_mel=True)
    mels = []
    for seed in (500, 600):
        nb = [_utterance(seed + i, P, nc, F, cc["codebook_size"], c["content_dim"]) for i, (P, nc, F) in enumerate(long_)]
        batch = engine.codes_to_wav_batch([nb[0], short[0], nb[1], short[1], nb[2]], 25, 0.7, **kw)
        mels.append((batch[1]["mel"], batch[3]["mel"], batch[0]["mel"]))
    assert not np.array_equal(mels[0][2], mels[1][2])            # the neighbours did change
    for i, F in ((0, 1), (1, 2)):
        a, b = mels[0][i], mels[1][i]
        assert a.shape == (80, F) and np.isfinite(a).all()
        assert np.array_equal(a, b), (F, float(np.abs(a - b).max()))
        solo = engine.codes_to_wav(*(short[i][k] for k in ("codes", "prompt_condition", "ref_mel", "style", "z", "F")), 25, 0.7,
                                   want_mel=True)["mel"]
        # below 32 frames the solo call runs its fp32 input GEMMs on the SIMT kernel, the packed solve on tf32 (module doc)
        print(f"{F}-frame utterance: bitwise unchanged by its neighbours; max |packed - solo| {float(np.abs(a - solo).max()):.2e}")
        assert np.abs(a - solo).max() < 2e-2


def test_batch_longer_than_65535_packed_frames(engine):
    """One packed solve over more than 65 535 frames (the grid-y limit of a one-block-per-row launch): its first and last
    utterances equal their solo calls."""
    c, cc = _load(engine, full=False)
    spec = [(20, 30, 500)] + [(0, 40, 16500)] * 4 + [(10, 25, 300)]
    utts = [_utterance(700 + i, P, nc, F, cc["codebook_size"], c["content_dim"]) for i, (P, nc, F) in enumerate(spec)]
    assert sum(P + F for P, _, F in spec) > 65535
    kw = dict(want_wav=True, want_pcm16=True, want_mel=True)
    batch = engine.codes_to_wav_batch(utts, 25, 0.7, **kw)
    for i in (1, 2, 3, 4):
        assert np.isfinite(batch[i]["mel"]).all()
    for i in (0, len(utts) - 1):
        u, b = utts[i], batch[i]
        solo = engine.codes_to_wav(u["codes"], u["prompt_condition"], u["ref_mel"], u["style"], u["z"], u["F"], 25, 0.7, **kw)
        dmel = float(np.abs(b["mel"] - solo["mel"]).max())
        dwav = float(np.sqrt(((b["wav"] - solo["wav"]) ** 2).mean()))
        same = all(np.array_equal(np.asarray(solo[k]), np.asarray(b[k])) for k in ("mel", "wav", "pcm16"))
        print(f"[{sum(P + F for P, _, F in spec)} packed frames] utterance {i}: bitwise equal to its solo call: {same}; "
              f"max |dmel| {dmel:.3e}, wav rms diff {dwav:.3e}")
        assert dmel <= 1e-5 * float(np.abs(solo["mel"]).max()) and dwav <= 1e-6
        assert np.array_equal(b["pcm16"], solo["pcm16"])
