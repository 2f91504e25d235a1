"""Record how the reference's driver scripts use the drop-in modules, as tests/golden/reference_script_surface.json.

    python -m oracle.gen_script_surface REFERENCE_DIR

For every script: the attributes it reads on ``outil`` / ``model`` / ``tgm``, the positional count and keyword names of each
``CoarseAlign(...)`` call, the attributes read on the names bound to a CoarseAlign instance, and the names it imports from
``coarseAlignFeatMatch``.  tests/test_dropin_scripts.py checks this package's mirrors against the stored record."""
import ast
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "reference_script_surface.json")
SCRIPTS = ["quick_start/align2images.py", "evaluation/evalHpatch/evaluation.py", "evaluation/evalCorr/evaluation.py",
           "evaluation/evalKITTI/evaluation.py", "evaluation/evalYFCC/evaluation.py", "evaluation/evalHpatch/getResults.py",
           "evaluation/evalCorr/getResults.py", "evaluation/evalKITTI/getResults.py"]


def surface(tree):
    mod_attrs, ctor_calls, inst_attrs, inst_names, imports = set(), [], {}, set(), set()
    for node in ast.walk(tree):
        if isinstance(node, ast.Assign) and isinstance(node.value, ast.Call) and isinstance(node.value.func, ast.Name) \
                and node.value.func.id == "CoarseAlign":
            ctor_calls.append({"nargs": len(node.value.args), "keywords": sorted(k.arg for k in node.value.keywords if k.arg)})
            for t in node.targets:
                if isinstance(t, ast.Name):
                    inst_names.add(t.id)
        if isinstance(node, ast.ImportFrom) and node.module == "coarseAlignFeatMatch":
            imports.update(al.name for al in node.names)
    for node in ast.walk(tree):
        if isinstance(node, ast.Attribute) and isinstance(node.value, ast.Name):
            if node.value.id in ("outil", "model", "tgm"):
                mod_attrs.add((node.value.id, node.attr))
            if node.value.id in inst_names:
                inst_attrs.setdefault(node.value.id, set()).add(node.attr)
    return {"mod_attrs": sorted(mod_attrs), "ctor_calls": ctor_calls, "inst_attrs": {k: sorted(v) for k, v in sorted(inst_attrs.items())},
            "imports": sorted(imports)}


def main(ref):
    out = {s: surface(ast.parse(open(os.path.join(ref, s)).read())) for s in SCRIPTS}
    with open(OUT, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", OUT)


if __name__ == "__main__":
    if len(sys.argv) != 2:
        raise SystemExit("usage: python -m oracle.gen_script_surface REFERENCE_DIR")
    main(sys.argv[1])
