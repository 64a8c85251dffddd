"""Times rasterize_to_indices_in_range and rasterize_to_indices_in_range_2dgs on bench.py's scene (the garden crop tiled
3 x 3, 1M Gaussians, one 1920x1080 view, seed 42), with one rasterize_to_pixels forward on the same 3DGS intersections
for scale.

    python tools/indices_bench.py [--steps 20] [--warmup 5]

Each call is timed with CUDA events after `warmup` untimed calls; an index call includes its host read of the pair
total between the count and the emit pass.  Projection and tile intersection run once, outside the timed calls.
Prints one JSON line with the median and minimum times, the pair counts, and the device name and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)

import gsplat_b200 as gs  # noqa: E402
from tests import scene  # noqa: E402

W, H, SCENE_GRID = 1920, 1080, 3
TW, TH = (W + 15) // 16, (H + 15) // 16


def device_info() -> dict:
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        info["nvidia_smi"] = out.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["nvidia_smi"] = f"unavailable: {e}"
    return info


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return round(statistics.median(ts), 3), round(min(ts), 3)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("indices_bench needs a GPU")
    dev = "cuda:0"
    sc = scene.make_scene(scene_grid=SCENE_GRID, sh_degree=0)
    Ks = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)[:1]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    vm = t(sc["viewmats"][:1])
    opac = t(sc["opacities"])[None].contiguous()
    colors = t(sc["colors"])[None].contiguous()
    ones = torch.ones((1, H, W), device=dev)
    rec = {"image": f"{W}x{H}", "n_gaussians": int(sc["means"].shape[0]), "steps": args.steps}
    with torch.no_grad():
        radii, m2, depths, conics, _ = gs.fully_fused_projection(t(sc["means"]), None, t(sc["quats"]), t(sc["scales"]), vm, t(Ks), W, H)
        _, ids, fl = gs.isect_tiles(m2, radii, depths, 16, TW, TH, conics=conics, opacities=opac)
        off = gs.isect_offset_encode(ids, 1, TW, TH)
        rec["isects_3dgs"] = int(fl.shape[0])
        rec["pairs_3dgs"] = int(gs.rasterize_to_indices_in_range(0, 2**30, ones, m2, conics, opac, W, H, 16, off, fl)[0].shape[0])
        rec["indices_3dgs_ms"], rec["indices_3dgs_min_ms"] = timed(
            lambda: gs.rasterize_to_indices_in_range(0, 2**30, ones, m2, conics, opac, W, H, 16, off, fl), args.steps, args.warmup)
        rec["raster_fwd_3dgs_ms"], rec["raster_fwd_3dgs_min_ms"] = timed(
            lambda: gs.rasterize_to_pixels(m2, conics, colors, opac, W, H, 16, off, fl), args.steps, args.warmup)

        radii2, m22, depths2, rt, _ = gs.fully_fused_projection_2dgs(t(sc["means"]), t(sc["quats"]), t(sc["scales"]), vm, t(Ks), W, H)
        _, ids2, fl2 = gs.isect_tiles(m22, radii2, depths2, 16, TW, TH)
        off2 = gs.isect_offset_encode(ids2, 1, TW, TH)
        rec["isects_2dgs"] = int(fl2.shape[0])
        rec["pairs_2dgs"] = int(gs.rasterize_to_indices_in_range_2dgs(0, 2**30, ones, m22, rt, opac, W, H, 16, off2, fl2)[0].shape[0])
        rec["indices_2dgs_ms"], rec["indices_2dgs_min_ms"] = timed(
            lambda: gs.rasterize_to_indices_in_range_2dgs(0, 2**30, ones, m22, rt, opac, W, H, 16, off2, fl2), args.steps, args.warmup)
    rec.update(device_info())
    print(json.dumps(rec), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
