"""Time rasterization_2dgs forward + backward on the 1080p bench scene, next to rasterization() on the same scene, in
one process (the bench scene of bench.py: the 3 x 3 tiled garden crop, ~1M Gaussians, one 1920 x 1080 view, SH degree 3,
dense rows).  Prints the card's name and power limit with the numbers, as one JSON line.

    python tools/bench_2dgs.py [--steps 20] [--warmup 5] [--out results/bench_2dgs.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import gsplat_b200  # noqa: E402
from tests import scene  # noqa: E402

W_IMG, H_IMG, SH_DEGREE, SCENE_GRID = 1920, 1080, 3, 3


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"{torch.cuda.get_device_name(0)} (power limit unknown: {e})"


def _time(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(steps):
        step()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_2dgs needs a GPU"
    dev = "cuda"
    sc = scene.make_scene(scene_grid=SCENE_GRID, sh_degree=SH_DEGREE)
    Ks = torch.tensor(scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W_IMG, H_IMG)[:1], device=dev)
    vm = torch.tensor(sc["viewmats"][:1], device=dev)
    p = {k: torch.tensor(sc[k], device=dev).requires_grad_(True) for k in ("means", "quats", "scales", "opacities", "sh")}
    target = torch.rand(1, H_IMG, W_IMG, 3, device=dev, generator=torch.Generator(device=dev).manual_seed(0))

    def step_3dgs():
        rc, ra, _ = gsplat_b200.rasterization(
            p["means"], p["quats"], p["scales"], p["opacities"], p["sh"], vm, Ks, W_IMG, H_IMG, sh_degree=SH_DEGREE, packed=False
        )
        (rc - target).abs().mean().backward()

    def step_2dgs():
        rc, ra, rn, sn, rd, rm, _ = gsplat_b200.rasterization_2dgs(
            p["means"], p["quats"], p["scales"], p["opacities"], p["sh"], vm, Ks, W_IMG, H_IMG, sh_degree=SH_DEGREE,
            render_mode="RGB+ED", distloss=True,
        )
        ((rc[..., :3] - target).abs().mean() + 0.01 * rd.mean() + 0.01 * (1 - (rn * sn).sum(-1)).mean()).backward()

    out = {"card": _card(), "n_gaussians": int(p["means"].shape[0]), "image": f"{W_IMG}x{H_IMG}", "sh_degree": SH_DEGREE,
           "steps": a.steps, "warmup": a.warmup}
    # alternate the two so that both see the same state of a shared machine
    ms3, ms2 = [], []
    for _ in range(3):
        ms3.append(_time(step_3dgs, a.steps, a.warmup))
        ms2.append(_time(step_2dgs, a.steps, a.warmup))
    out["rasterization_ms_fwd_bwd"] = [round(x, 3) for x in ms3]
    out["rasterization_2dgs_ms_fwd_bwd"] = [round(x, 3) for x in ms2]
    out["note"] = "2DGS step: RGB+ED, distloss, depth-normal consistency term; 3DGS step: RGB L1"
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
