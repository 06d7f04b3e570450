"""The entry-point classes keep the reference's constructor / .infer() signatures (SURVEY §8b).  The reference's signatures
are stored in tests/golden/reference_signatures.json (oracle/make_goldens_signatures.py reads them from the reference
source with ast).  Building a live reference IndexTTS2 additionally needs checkpoints and the w2v-BERT / CAMPPlus /
BigVGAN downloads of infer_v2_5.py:170-260, which do not exist offline — that is what blocks an end-to-end `.infer()`
test here, not anything in this package."""
import inspect
import json
import os

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_signatures.json")


def _params(fn, drop=()):
    return [(n, p.default) for n, p in inspect.signature(fn).parameters.items() if n not in drop]


def _reference(cls_name):
    with open(GOLDEN) as f:
        return json.load(f)[cls_name]


def test_indextts2_signatures_match_the_reference():
    ref = _reference("IndexTTS2")
    from indextts_b200.infer_v2_5 import IndexTTS2
    for name, drop in (("__init__", ("engine_device",)), ("infer", ())):
        ref_args = ref[name]["args"]
        mine = [n for n, _ in _params(getattr(IndexTTS2, name), drop)]
        assert mine == ref_args, (name, mine, ref_args)
        ref_defaults = ref[name]["defaults"]
        my_defaults = [d for n, d in _params(getattr(IndexTTS2, name), drop) if d is not inspect.Parameter.empty]
        assert my_defaults == ref_defaults, (name, my_defaults, ref_defaults)


def test_indextts_v1_signatures_match_the_reference():
    ref = _reference("IndexTTS")
    from indextts_b200.infer import IndexTTS
    for name, drop in (("__init__", ("engine_device",)), ("infer", ())):
        ref_args = ref[name]["args"]
        mine = [n for n, _ in _params(getattr(IndexTTS, name), drop)]
        assert mine == ref_args, (name, mine, ref_args)
