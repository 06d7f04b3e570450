"""GPU: the IndexTTS-1.5 chain (SURVEY section 8 row a13) at its real geometry, against float64 oracles run on the GPU.

* Vocoder (`idx_v1_vocode`) at synth.v1_5_config(): ECAPA speaker embedding, then the latent-conditioned BigVGAN
  (1280 -> 1536 channels, six upsamples, x1024) with the speaker embedding folded into the biases of conv_pre and of
  every upsample.  Latent lengths 1 .. 600 (614 400 samples), reference mels of 5 .. 1406 frames, on the default fp16-operand
  path, on tf32 (tail_f16 0) and on the strict fp32 back end.  Also: bitwise reruns, a live speaker path at every stage,
  and time locality with the receptive field derived from the config.
* Latent pass (`idx_gpt_latents_v1`) at 24 x 1280 on the strict and on the fused bf16 engine, over rows
  32 + text + 2 + codes + 2 across the 8-row prefill tiles, up to the end of the KV cache; one row more is refused.
* The no-cache position rule (`mel_pos_mode = 1`, infer.py:99-101: every step re-embeds its mel positions as 0..k).  On
  weights W it is the KV-cached rule (`mel_pos_mode = 0`) on W' = W with mel_pos_embedding shifted (W'[k + 1] = W[k] for
  k >= 1), so every decode path must return bitwise the same codes and logits for (mode 1, W) and (mode 0, W').
  The strict path decodes 128 free-running tokens at 24 layers against the fp32 oracle on W'.
The weights are seeded and synthetic; the configs are [ASSUMED] from the published IndexTTS-1.5 config (synth.py)."""
import os

import numpy as np
import pytest
import torch

from indextts_b200 import synth
from indextts_b200.engine import _ptr
from indextts_b200.synth import V1_COND_CFG
from oracle import v1
from oracle.gpt import GptOracle
from oracle.validate_gpt_vs_hf import small_case
from tests.test_gpt_picks_gpu import PATHS, _env

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden", "v1_vocoder_full.npz")
MODES = {"f16": (0, 1), "tf32": (0, 0), "strict": (1, 1)}        # name: (gemm_backend, tail_f16)
RMS_TC, MAX_TC, MAX_STRICT = 1e-3, 2e-2, 2e-4                  # BigVGAN north-star bound (test_bigvgan_gpu.py); strict


def _gpu64(w):
    return {k: v.double().cuda() for k, v in w.items()}


def _in_mode(engine, mode, fn):
    backend, f16 = MODES[mode]
    engine.set_option("gemm_backend", backend)
    engine.set_option("tail_f16", f16)
    try:
        return fn()
    finally:
        engine.set_option("gemm_backend", 0)
        engine.set_option("tail_f16", 1)


# ------------------------------------------------------------------------------------------------------ vocoder --
@pytest.fixture(scope="module")
def v15_vocoder(engine):
    h = synth.v1_5_config()
    w = synth.make_bigvgan_v1_weights(h, seed=int(np.load(GOLD)["seed"]), post_gain=synth.V1_5_POST_GAIN)
    engine.load_state_dict("bigvgan_v1.", {k: v for k, v in w.items() if v.is_floating_point()})
    engine.v1_vocoder_init(h)
    return h, _gpu64(w)


def _reference(h, wd, latent, mel_ref):
    return v1.bigvgan_v1_forward(h, wd, torch.as_tensor(latent)[None].double().cuda(),
                                 torch.as_tensor(mel_ref)[None].double().cuda())[0, 0].cpu().numpy()


def _inputs(T, Tm, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(T, 1280, generator=g).numpy(), (torch.randn(Tm, 100, generator=g) * 1.5 - 4.0).numpy())


def _errors(got, ref):
    d = got.astype(np.float64) - ref
    return float(np.sqrt((d ** 2).mean())), float(np.abs(d).max())


def first_touched(h, t0, taps=12):
    """First output sample that latents t0.. can reach: each op's left reach in its own sample rate.  conv_pre and
    conv_post (k = 7, padding 3) reach 3 back; ConvTranspose1d(u, k, padding (k - u) // 2) maps input t to outputs from
    t * u - (k - u) // 2; a conv (ks, dilation d, "same") reaches d * (ks - 1) // 2; Activation1d (x2 up, SnakeBeta, x2
    down, both `taps`-tap filters) reaches taps // 2; the resblocks of a stage run in parallel (the longest counts)."""
    A = taps // 2
    a = t0 - 3
    for u, k in zip(h["upsample_rates"], h["upsample_kernel_sizes"]):
        a = a * u - (k - u) // 2
        a -= max(sum(2 * A + d * (ks - 1) // 2 + (ks - 1) // 2 for d in dil)
                 for ks, dil in zip(h["resblock_kernel_sizes"], h["resblock_dilation_sizes"]))
    return a - A - 3


def test_v1_5_vocoder_vs_reference_golden(engine, v15_vocoder):
    """The golden minted from the reference's own v1 BigVGAN at this geometry (4 latents, 61-frame mel)."""
    g = np.load(GOLD)
    for mode in MODES:
        wav = _in_mode(engine, mode, lambda: engine.v1_vocode(g["latent"][0], g["mel_ref"][0]))
        rms, mx = _errors(wav, g["wav"][0, 0])
        print(f"v1.5 vocoder vs reference golden [{mode}]: rms {rms:.2e}, max {mx:.2e}")
        assert wav.shape == (4096,)
        assert mx <= MAX_STRICT if mode == "strict" else (rms <= RMS_TC and mx <= MAX_TC)


@pytest.mark.parametrize("T,Tm", [(1, 5), (2, 61), (3, 1406), (37, 5), (150, 61), (600, 1406)])
def test_v1_5_vocoder_full_geometry(engine, v15_vocoder, T, Tm):
    h, wd = v15_vocoder
    latent, mel = _inputs(T, Tm, 1000 * T + Tm)
    ref = _reference(h, wd, latent, mel)
    assert ref.shape == (T * 1024,)
    for mode in MODES:
        wav = _in_mode(engine, mode, lambda: engine.v1_vocode(latent, mel))
        rms, mx = _errors(wav, ref)
        print(f"v1.5 vocoder T={T} ({T * 1024} samples) Tm={Tm} [{mode}]: rms {rms:.2e}, max {mx:.2e} "
              f"(ref rms {np.sqrt((ref ** 2).mean()):.3f})")
        assert wav.shape == (T * 1024,) and np.all(np.abs(wav) <= 1.0)
        if mode == "strict":
            assert mx <= MAX_STRICT
        else:
            assert rms <= RMS_TC and mx <= MAX_TC
        again = _in_mode(engine, mode, lambda: engine.v1_vocode(latent, mel))
        assert np.array_equal(again.view(np.uint32), wav.view(np.uint32)), mode


def test_v1_5_speaker_path_live_at_every_stage(engine, v15_vocoder):
    """Dropping the speaker term at any one stage (cond_layer after conv_pre, conds[i] after ups[i]) moves the float64
    reference far beyond the tensor-core bound, so the accuracy tests above see a missed fold at any stage; and the engine's
    own output follows a swapped reference mel by as much."""
    h, wd = v15_vocoder
    latent, mel = _inputs(37, 61, 77)
    ref = _reference(h, wd, latent, mel)
    for name in ["cond_layer"] + [f"conds.{i}" for i in range(len(h["upsample_rates"]))]:
        w2 = dict(wd, **{name + ".weight": torch.zeros_like(wd[name + ".weight"]),
                         name + ".bias": torch.zeros_like(wd[name + ".bias"])})
        rms, _ = _errors(_reference(h, w2, latent, mel), ref)
        print(f"speaker term {name} dropped: reference moves by rms {rms:.2e}")
        assert rms > 10 * RMS_TC, name
    mel2 = np.ascontiguousarray(mel[::-1] * 0.5)
    for mode in MODES:
        a = _in_mode(engine, mode, lambda: engine.v1_vocode(latent, mel))
        b = _in_mode(engine, mode, lambda: engine.v1_vocode(latent, mel2))
        rms, _ = _errors(a, b.astype(np.float64))
        print(f"[{mode}] swapped reference mel: output moves by rms {rms:.2e}")
        assert rms > 50 * RMS_TC


def test_v1_5_vocoder_time_locality(engine, v15_vocoder):
    """Changing the last two latents leaves every sample before their receptive field bitwise unchanged."""
    h, wd = v15_vocoder
    T = 150
    latent, mel = _inputs(T, 61, 5)
    lat2 = latent.copy()
    lat2[T - 2:] += 1.0
    a0 = first_touched(h, T - 2, taps=wd["activation_post.upsample.filter"].shape[-1])
    assert 0 < a0 < (T - 2) * 1024
    d_ref = np.nonzero(_reference(h, wd, latent, mel) != _reference(h, wd, lat2, mel))[0]
    assert d_ref.size and d_ref[0] >= a0
    for mode in MODES:
        a = _in_mode(engine, mode, lambda: engine.v1_vocode(latent, mel))
        b = _in_mode(engine, mode, lambda: engine.v1_vocode(lat2, mel))
        d = np.nonzero(a.view(np.uint32) != b.view(np.uint32))[0]
        print(f"[{mode}] last 2 of {T} latents changed: first changed sample {d[0]} (float64 reference {d_ref[0]}, "
              f"receptive-field bound {a0})")
        assert d.size and d[0] >= a0


# --------------------------------------------------------------------------------------------- GPT, full size --
MAX_PROMPT = 425        # KV cache rows = max_prompt + max_mel_positions + 8 = 1041 = the longest latent pass below


@pytest.fixture(scope="module")
def v15_gpt():
    cfg = synth.gpt_config(max_mel_tokens=605, max_text_tokens=402)
    w = synth.make_gpt_v1_weights(cfg, V1_COND_CFG, seed=1500)
    return cfg, w


def _shifted(w):
    """W' = W with mel_pos_embedding moved one row on from position 1: W'[k + 1] = W[k] (k >= 1), W'[0] = W[0]."""
    t = w["mel_pos_embedding.emb.weight"]
    s = t.clone()
    s[2:] = t[1:-1]
    return s


def _init(engine, cfg, bf16, max_prompt, max_batch=1, env=None):
    with _env(env or {}):
        engine.gpt_init(cfg["layers"], cfg["model_dim"], cfg["heads"], cfg["number_mel_codes"], cfg["start_mel_token"],
                        cfg["stop_mel_token"], cfg["max_mel_positions"], max_prompt=max_prompt, max_batch=max_batch,
                        weights_bf16=bf16)


def _set_pos(engine, table):
    engine.load_weight("gpt.mel_pos_embedding.emb.weight", table)


@pytest.fixture(scope="module")
def v15_loaded(engine, v15_gpt):
    """Full-size v1 weights in the engine and real conds from its v1_get_conditioning on a random 200-frame mel."""
    cfg, w = v15_gpt
    engine.load_state_dict("gpt.", w)
    _init(engine, cfg, False, MAX_PROMPT)
    engine.v1_cond_init(V1_COND_CFG, 32)
    mel = torch.randn(200, 100, generator=torch.Generator().manual_seed(15)).numpy() * 1.5 - 4.0
    conds = engine.v1_get_conditioning(mel)
    assert conds.shape == (32, 1280) and np.all(np.isfinite(conds))
    return cfg, w, conds


LAT_CASES = [(nt, nc) for nt in (1, 30, 400) for nc in (1, 7, 8, 9, 300, 605)]


@pytest.fixture(scope="module")
def latent_refs(v15_loaded):
    cfg, w, conds = v15_loaded
    gw = _gpu64({k: v for k, v in w.items() if not k.startswith(("conditioning_encoder.", "perceiver_encoder."))})
    orc = GptOracle(cfg, gw, bf16=False)
    g = torch.Generator().manual_seed(16)
    out = {}
    for nt, nc in LAT_CASES:
        text = torch.randint(2, cfg["number_text_tokens"], (nt,), generator=g).numpy().astype(np.int32)
        codes = torch.randint(0, 8192, (nc,), generator=g).numpy().astype(np.int32)
        ref = v1.latents_v1(orc, torch.from_numpy(conds).double().cuda(), text, codes).cpu().numpy()
        out[(nt, nc)] = (text, codes, ref)
    del gw, orc
    torch.cuda.empty_cache()
    return out


@pytest.mark.parametrize("bf16", [False, True], ids=["strict", "bf16"])
def test_v1_5_latent_pass_full_depth(engine, v15_loaded, latent_refs, bf16):
    cfg, w, conds = v15_loaded
    _init(engine, cfg, bf16, MAX_PROMPT)
    worst = 0.0
    for (nt, nc), (text, codes, ref) in latent_refs.items():
        lat = engine.gpt_latents_v1(conds, text, codes)
        R = 32 + nt + 2 + nc + 2
        assert lat.shape == ref.shape == (nc, 1280) and np.all(np.isfinite(lat))
        if bf16:
            err = float(np.sqrt(((lat - ref) ** 2).mean()) / ref.std())
            print(f"v1 latents bf16 n_text={nt} n_codes={nc} (R={R}): relative rms {err:.4f}")
            assert err <= 0.05
        else:
            err = float(np.abs(lat - ref).max())
            print(f"v1 latents strict n_text={nt} n_codes={nc} (R={R}): max abs {err:.2e} (ref std {ref.std():.2f})")
            assert err <= 1e-3
        worst = max(worst, err)
    print(f"{'bf16 relative rms' if bf16 else 'strict max abs'}: worst {worst:.3g}")
    # one row past the KV cache (R = 32 + 401 + 2 + 605 + 2 = 1042 > 1041 rows) is refused before anything is written
    text = np.full(401, 5, np.int32)
    codes = np.zeros(605, np.int32)
    out = np.full((605, 1280), np.nan, np.float32)
    n0 = engine.launches
    rc = engine.lib.idx_gpt_latents_v1(engine.h, _ptr(conds), 32, _ptr(text), 401, _ptr(codes), 605, _ptr(out))
    assert rc != 0 and b"KV cache" in engine.lib.idx_last_error(engine.h)
    assert engine.launches == n0 and np.all(np.isnan(out))        # (400, 605) above fills the cache to its last row


def _v1_prompt(w, conds, n_text, seed):
    text = torch.randint(2, 100, (n_text,), generator=torch.Generator().manual_seed(seed))
    return v1.prepare_inputs_v1(w, torch.as_tensor(conds), text).numpy()


def test_v1_5_no_cache_decode_strict_full_depth(engine, v15_loaded):
    """Production path: strict fp32, 24 layers, a v1 prompt (32 conds + 30 text ids), 128 free-running greedy tokens
    with mel_pos_mode = 1, against the fp32 oracle's KV-cached decode on W'.  That W' is the same function as the
    reference's decode without a cache is pinned once, over 16 steps."""
    cfg, w, conds = v15_loaded
    prompt = _v1_prompt(w, conds, 30, 30)
    assert prompt.shape == (64, 1280)
    gw = {k: v.cuda() for k, v in w.items() if not k.startswith(("conditioning_encoder.", "perceiver_encoder."))}
    gs = dict(gw, **{"mel_pos_embedding.emb.weight": _shifted(w).cuda()})
    c_nc, l_nc = v1.generate_v1(GptOracle(cfg, gw, bf16=False), prompt, 16, 10.0, kv_cache=False)
    c_sh, l_sh = GptOracle(cfg, gs, bf16=False).generate(prompt, 16, 10.0)
    e0 = float(np.abs(l_nc - l_sh).max())
    print(f"no-cache decode on W vs KV-cached decode on W' (fp32, 16 steps): max logit diff {e0:.2e}")
    assert c_nc.tolist() == c_sh.tolist() and e0 <= 1e-4
    n = 128
    o_codes, o_logits = GptOracle(cfg, gs, bf16=False).generate(prompt, n, 10.0, n)
    del gw, gs
    torch.cuda.empty_cache()
    _init(engine, cfg, False, MAX_PROMPT)
    (codes,), (logits,) = engine.gpt_generate([prompt], n, 10.0, forbid_stop_before=n, return_logits=True, mel_pos_mode=1)
    err = float(np.abs(logits - o_logits).max())
    print(f"strict 24 x 1280, mel_pos_mode 1, {n} tokens: {int((codes == o_codes).sum())}/{n} equal, max logit err {err:.2e}")
    assert codes.tolist() == o_codes.tolist() and err <= 5e-4


def _generate(engine, prompts, n, mode, beams=1, sampled=False):
    kw = dict(forbid_stop_before=n, return_logits=True, mel_pos_mode=mode, num_beams=beams)
    if sampled:
        kw.update(do_sample=True, top_k=30, top_p=0.8, temperature=0.8, seed=123)
    codes, logits = engine.gpt_generate(prompts, n, 10.0, **kw)
    return [c.copy() for c in codes], [lg.copy() for lg in logits]


def _bitwise_equal(a, b):
    (ca, la), (cb, lb) = a, b
    return (all(np.array_equal(x, y) for x, y in zip(ca, cb)) and
            all(x.shape == y.shape and np.array_equal(x.view(np.uint32), y.view(np.uint32)) for x, y in zip(la, lb)))


def _check_pos_rule(engine, cfg, w, prompts, n, bf16, max_prompt, max_batch, env, beams, label):
    """(mode 1, W) == (mode 0, W') bitwise, greedy and sampled; and (mode 0, W) differs (the mode reaches the kernel)."""
    for sampled in (False, True):
        _set_pos(engine, w["mel_pos_embedding.emb.weight"])
        _init(engine, cfg, bf16, max_prompt, max_batch, env)
        plain = _generate(engine, prompts, n, 1, beams, sampled)
        cached = _generate(engine, prompts, n, 0, beams, sampled)
        _set_pos(engine, _shifted(w))
        _init(engine, cfg, bf16, max_prompt, max_batch, env)
        shifted = _generate(engine, prompts, n, 0, beams, sampled)
        same = _bitwise_equal(plain, shifted)
        print(f"{label} {'sampled' if sampled else 'greedy'}: mel_pos_mode 1 on W vs mode 0 on W' bitwise equal: {same}; "
              f"{sum(len(c) for c in plain[0])} codes")
        assert same, label
        assert not _bitwise_equal(plain, cached), label
    _set_pos(engine, w["mel_pos_embedding.emb.weight"])


SMALL_PATHS = {name: PATHS[name] for name in ("decode1", "decode8_3", "fused_1", "fused_bt8", "strict_1")}


@pytest.fixture(scope="module")
def small_v1(engine):
    cfg = small_case()[0]
    w = synth.make_gpt_v1_weights(cfg, synth.small_v1_cond_cfg(cfg["model_dim"]), seed=321)
    w = {k: v for k, v in w.items() if not k.startswith(("conditioning_encoder.", "perceiver_encoder."))}
    g = torch.Generator().manual_seed(3)
    prompts = [_v1_prompt(w, torch.randn(32, cfg["model_dim"], generator=g) * 0.5, 5 + 4 * i, 40 + i) for i in range(3)]
    return cfg, w, prompts


@pytest.mark.parametrize("path", list(SMALL_PATHS) + ["beam_3"])
def test_no_cache_position_rule_every_path_small(engine, small_v1, path):
    cfg, w, prompts = small_v1
    engine.load_state_dict("gpt.", w)
    if path == "beam_3":
        _check_pos_rule(engine, cfg, w, prompts[:2], 40, True, 128, 8, {}, 3, "beam search, 3 beams")
        return
    nreq, max_batch, bf16, env = SMALL_PATHS[path]
    _check_pos_rule(engine, cfg, w, prompts[:nreq], 40, bf16, 128, max_batch, env, 1, path)


@pytest.mark.parametrize("path", ["decode1", "decode8_3"])
def test_no_cache_position_rule_full_depth(engine, v15_loaded, path):
    cfg, w, conds = v15_loaded
    engine.load_state_dict("gpt.", w)                               # the small-geometry tests above replaced them
    nreq, max_batch, _, env = PATHS[path]
    prompts = [_v1_prompt(w, conds * (1 + 0.1 * i), 30 + 3 * i, 60 + i) for i in range(nreq)]
    _check_pos_rule(engine, cfg, w, prompts, 64, True, MAX_PROMPT, max_batch, env, 1, f"{path} 24 x 1280")


def test_mel_pos_table_end_both_modes(engine, small_v1):
    """idx_gpt_generate takes max_new_tokens + 2 <= max_mel_positions (SURVEY A.3).  At that last length both modes run to
    the end and match the fp32 oracle (mode 0 on W, mode 1 as mode 0 on W'), whose tables hold exactly max_mel_positions
    rows; one step more is refused before any launch."""
    cfg, w, prompts = small_v1
    last = cfg["max_mel_positions"] - 2
    engine.load_state_dict("gpt.", w)
    ws = dict(w, **{"mel_pos_embedding.emb.weight": _shifted(w)})
    for bf16 in (False, True):
        _init(engine, cfg, bf16, 128)
        for mode, ow in ((0, w), (1, ws)):
            (codes,), (logits,) = engine.gpt_generate(prompts[:1], last, 10.0, forbid_stop_before=last, return_logits=True,
                                                      mel_pos_mode=mode)
            assert len(codes) == last and np.all(np.isfinite(logits))
            if not bf16:
                o_codes, o_logits = GptOracle(cfg, ow, bf16=False).generate(prompts[0], last, 10.0, last)
                err = float(np.abs(logits - o_logits).max())
                print(f"strict, mel_pos_mode {mode}, {last} = max_mel_positions - 2 tokens: max logit err {err:.2e}")
                assert codes.tolist() == o_codes.tolist() and err <= 5e-4
            before = engine.gpt_last_timing()
            with pytest.raises(RuntimeError, match="max_new_tokens"):
                engine.gpt_generate(prompts[:1], last + 1, 10.0, mel_pos_mode=mode)
            assert engine.gpt_last_timing() == before


def test_mel_pos_mode_refused_before_launch(engine, small_v1):
    cfg, w, prompts = small_v1
    engine.load_state_dict("gpt.", w)
    for bf16 in (True, False):
        _init(engine, cfg, bf16, 128)
        engine.gpt_generate(prompts[:1], 4, 10.0, mel_pos_mode=1)
        before = engine.gpt_last_timing()
        for mode in (-1, 2, 7):
            with pytest.raises(RuntimeError, match="mel_pos_mode"):
                engine.gpt_generate(prompts[:1], 4, 10.0, mel_pos_mode=mode)
            assert engine.gpt_last_timing() == before, mode
