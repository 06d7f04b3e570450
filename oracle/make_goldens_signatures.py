"""Record the public signatures and seam call sites of the reference's entry points as tests/golden/reference_signatures.json.

    IDX_REFERENCE=<reference checkout> python -m oracle.make_goldens_signatures

Read with `ast` from indextts/infer_v2_5.py (class IndexTTS2) and indextts/infer.py (class IndexTTS): the argument names
and literal defaults of `__init__` / `infer`, and every call `infer_v2_5.py` / `infer.py` makes at the compute seams the
drop-in rebinds (positional count, keyword names).  tests/test_entrypoints_cpu.py and tests/test_dropin_cpu.py compare
the package against this file."""
import ast
import json
import os

from oracle.refimport import REF

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "reference_signatures.json")

SEAMS_V2_5 = {"self.gpt.merge_emovec": "merge_emovec", "self.gpt.inference_speech": "inference_speech",
              "self.semantic_codec.decode": "codec_decode", "self.s2mel.models['length_regulator']": "length_regulator",
              "self.s2mel.models['cfm'].inference": "cfm_inference", "self.bigvgan": "bigvgan"}
SEAMS_V1 = {"self.gpt.inference_speech": "inference_speech", "self.gpt": "gpt_forward", "self.bigvgan": "bigvgan"}


def _tree(rel):
    return ast.parse(open(os.path.join(REF, "indextts", rel)).read())


def _signatures(tree, cls_name):
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == cls_name)
    fns = {f.name: f for f in cls.body if isinstance(f, ast.FunctionDef)}
    out = {}
    for name in ("__init__", "infer"):
        a = fns[name].args
        out[name] = {"args": [x.arg for x in a.args] + ([a.kwarg.arg] if a.kwarg else []),
                     "defaults": [ast.literal_eval(d) for d in a.defaults]}
    return out


def _call_sites(tree, seams):
    found = {}
    for node in ast.walk(tree):
        if isinstance(node, ast.Call):
            name = ast.unparse(node.func)
            if name in seams:
                kws = [k.arg for k in node.keywords if k.arg is not None]
                star = any(k.arg is None for k in node.keywords)
                found.setdefault(seams[name], []).append([len(node.args), kws, star])
    return found


def main():
    v25, v1 = _tree("infer_v2_5.py"), _tree("infer.py")
    d = {"IndexTTS2": _signatures(v25, "IndexTTS2"), "IndexTTS": _signatures(v1, "IndexTTS"),
         "call_sites_v2_5": _call_sites(v25, SEAMS_V2_5), "call_sites_v1": _call_sites(v1, SEAMS_V1)}
    with open(OUT, "w") as f:
        json.dump(d, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", OUT)


if __name__ == "__main__":
    main()
