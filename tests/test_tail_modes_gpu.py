"""GPU: the precision switches of the environment are read once, when an engine is created, as that engine's initial
options.  IDX_NO_TC=1 starts it at gemm_backend 1 and IDX_TAIL_F16=0 at tail_f16 0, so a small-geometry codes_to_wav
(mel, wav, pcm16) on such an engine is bitwise equal to the shared engine's with the option set by idx_set_option."""
import numpy as np
import pytest

from indextts_b200.engine import Engine
from tests.test_tail_batch_gpu import _load, _small_set

pytestmark = pytest.mark.gpu

MODES = [("IDX_NO_TC", "1", "gemm_backend", 1, 0), ("IDX_TAIL_F16", "0", "tail_f16", 0, 1)]


@pytest.fixture(params=MODES, ids=[m[0] for m in MODES])
def env_engine(request, lib_built, monkeypatch):
    """An engine created with one switch in the environment (removed again right after idx_create), and its mode."""
    var, value, option, on, off = request.param
    monkeypatch.setenv(var, value)
    e = Engine(0)
    monkeypatch.delenv(var)
    yield e, option, on, off
    e.close()


def test_environment_sets_the_initial_mode(engine, env_engine):
    e, option, on, off = env_engine
    c, cc = _load(engine, full=False)
    _load(e, full=False)
    u = _small_set(1, cc, c)[0]
    args = (u["codes"], u["prompt_condition"], u["ref_mel"], u["style"], u["z"], u["F"], 25, 0.7)
    kw = dict(want_wav=True, want_pcm16=True, want_mel=True)
    got = e.codes_to_wav(*args, **kw)
    engine.set_option(option, on)
    try:
        want = engine.codes_to_wav(*args, **kw)
    finally:
        engine.set_option(option, off)
    default = engine.codes_to_wav(*args, **kw)
    for k in ("mel", "wav", "pcm16"):
        assert np.array_equal(got[k], want[k]), k
    assert not np.array_equal(got["mel"], default["mel"])      # the mode did change the arithmetic
