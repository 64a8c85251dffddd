#!/usr/bin/env python
"""Where the HOST spends its time issuing one bench.py-style train step (cProfile over the Python side of
rasterization() + fused L1 + backward).  The step is GPU-bound only while the host can issue it faster than the GPU
executes it; this prints the host's issue time per step next to the device time, and the top functions.

    python tools/host_profile.py --steps 300 > out/host_profile.txt
"""
import argparse
import cProfile
import io
import os
import pstats
import sys
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import gsplat_b200  # noqa: E402
from tests import scene  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=300)
ap.add_argument("--grid", type=int, default=3)
args = ap.parse_args()
dev = "cuda:0"
W, H = 1920, 1080
sc = scene.make_scene(scene_grid=args.grid, sh_degree=3)
Ks = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)
P = {k: torch.from_numpy(sc[k]).to(dev).requires_grad_(True) for k in ("means", "quats", "scales", "opacities", "sh")}
vm, K = torch.from_numpy(sc["viewmats"][:1]).to(dev), torch.from_numpy(Ks[:1]).to(dev)
target = torch.rand((1, H, W, 3), device=dev)


def step():
    for p in P.values():
        p.grad = None
    rc, ra, meta = gsplat_b200.rasterization(P["means"], P["quats"], P["scales"], P["opacities"], P["sh"], vm, K, W, H, sh_degree=3, packed=False)
    gsplat_b200.l1_loss(rc, target).backward()


for _ in range(20):
    step()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
t0 = time.perf_counter()
for _ in range(args.steps):
    step()
t1 = time.perf_counter()
e1.record()
torch.cuda.synchronize()
print(f"device {e0.elapsed_time(e1) / args.steps:.3f} ms/step, host issue {(t1 - t0) * 1e3 / args.steps:.3f} ms/step (includes waiting for the totals)")
pr = cProfile.Profile()
pr.enable()
for _ in range(args.steps):
    step()
pr.disable()
torch.cuda.synchronize()
out = io.StringIO()
st = pstats.Stats(pr, stream=out)
st.sort_stats("tottime").print_stats(35)
print(out.getvalue())
out = io.StringIO()
pstats.Stats(pr, stream=out).sort_stats("cumtime").print_stats(30)
print(out.getvalue())
