#!/usr/bin/env python
"""Write tests/golden/ref_signatures_contrib.json: the parameter lists of the reference's per-pixel contributor queries
(rasterize_num_contributing_gaussians, rasterize_contributing_gaussian_ids, rasterize_top_contributing_gaussian_ids and
their _sparse forms, gsplat/cuda/_wrapper.py), parsed with ast from a gsplat source checkout.

    python tests/golden/make_golden_contrib.py GSPLAT_CHECKOUT      (the directory that holds gsplat/)

tests/golden/make_ref_contrib_golden.py records the reference ops' outputs (ref_contrib.npz) on a GPU.
"""
import ast
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
NAMES = tuple(
    f"rasterize_{n}{s}"
    for n in ("num_contributing_gaussians", "contributing_gaussian_ids", "top_contributing_gaussian_ids")
    for s in ("", "_sparse")
)


def main():
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    path = os.path.join(sys.argv[1], "gsplat", "cuda", "_wrapper.py")
    out = {}
    for node in ast.walk(ast.parse(open(path).read())):
        if isinstance(node, ast.FunctionDef) and node.name in NAMES:
            a = node.args
            out[node.name] = {"params": [x.arg for x in a.posonlyargs + a.args + a.kwonlyargs], "n_defaults": len(a.defaults)}
    assert sorted(out) == sorted(NAMES), f"found {sorted(out)} in {path}"
    with open(os.path.join(HERE, "ref_signatures_contrib.json"), "w") as f:
        json.dump({"params": out}, f, indent=1)
    print("wrote ref_signatures_contrib.json")


if __name__ == "__main__":
    main()
