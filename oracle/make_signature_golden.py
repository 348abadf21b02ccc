"""Extracts the reference pipeline's public signatures with `ast` (no import of the reference needed) and writes
tests/golden/pipeline_signature.json. Needs a checkout of the original project (IDM_VTON_REFERENCE)."""
import ast
import json
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(os.environ.get("IDM_VTON_REFERENCE", ""), "src", "tryon_pipeline.py")


def signature(fn):
    a = fn.args
    names = [x.arg for x in a.args]
    defaults = [None] * (len(names) - len(a.defaults)) + [ast.unparse(d) for d in a.defaults]
    return {"args": names, "defaults": defaults, "kwarg": a.kwarg.arg if a.kwarg else None,
            "has_default": [False] * (len(names) - len(a.defaults)) + [True] * len(a.defaults)}


def extract(path, cls, methods):
    tree = ast.parse(open(path).read())
    for node in tree.body:
        if isinstance(node, ast.ClassDef) and node.name == cls:
            return {f.name: signature(f) for f in node.body if isinstance(f, ast.FunctionDef) and f.name in methods}
    raise RuntimeError(cls)


if __name__ == "__main__":
    out = extract(SRC, "StableDiffusionXLInpaintPipeline", ("__init__", "encode_prompt", "__call__", "check_inputs"))
    with open(os.path.join(ROOT, "tests", "golden", "pipeline_signature.json"), "w") as f:
        json.dump({"source": "src/tryon_pipeline.py:387-401,511-526,763-780,1254-1301", "signatures": out}, f, indent=1)
    print({k: len(v["args"]) for k, v in out.items()})
