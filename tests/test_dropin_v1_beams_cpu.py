"""CPU: `attach_v1` sizes the strict fp32 GPT for the reference's default beam search (`infer.py` passes num_beams=3 to
`inference_speech`; the strict path needs one sequence slot per beam, so max_batch must be at least 3)."""
import types

from tests.test_dropin_cpu import RecordingEngine, StandIn, _golden, _gpt


def test_attach_v1_leaves_room_for_the_default_beams():
    from indextts_b200.dropin import attach_v1

    g = _golden("dropin_modules.json")
    tts = types.SimpleNamespace(gpt=_gpt(g["gpt_v1"]),
                                bigvgan=StandIn(g["bigvgan_v1"]["state_dict"], h=g["bigvgan_v1"]["attrs"]["h"]))

    class Rec(RecordingEngine):
        def v1_cond_init(self, c, n):
            pass

        def v1_vocoder_init(self, hh):
            pass

    eng = Rec()
    attach_v1(tts, engine=eng)
    _, kw = eng.calls["gpt_init"]
    assert kw["weights_bf16"] is False and kw["max_batch"] >= 3
