#!/usr/bin/env python
"""One bench.py-style train step of the BASELINE workload, for use under ncu:

  ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file out/launches.csv \
      python tools/profile_step.py --steps 2 --warmup 2
  ncu --set full --clock-control none --import-source on -k regex:raster_bwd -s 2 -c 1 -o out/prof_bwd \
      python tools/profile_step.py --steps 1 --warmup 2

Numbers printed by a run under ncu are never bench values.  Also prints a CUDA-event breakdown per stage
(forward stages are timed by calling the operators one by one, outside autograd)."""
import argparse
import os
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import gsplat_b200  # noqa: E402
from gsplat_b200 import ops  # noqa: E402
from tests import scene  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=2)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--grid", type=int, default=3)
ap.add_argument("--breakdown", action="store_true")
ap.add_argument("--packed", action="store_true")
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
    rc, ra, meta = gsplat_b200.rasterization(P["means"], P["quats"], P["scales"], P["opacities"], P["sh"], vm, K, W, H, sh_degree=3, packed=args.packed)
    (rc - target).abs().mean().backward()
    return meta


for _ in range(args.warmup):
    meta = step()
torch.cuda.synchronize()
torch.cuda.cudart().cudaProfilerStart()
for _ in range(args.steps):
    meta = step()
torch.cuda.synchronize()
torch.cuda.cudart().cudaProfilerStop()
print("n_isects", meta["flatten_ids"].numel(), "visible", int((meta["radii"] > 0).all(-1).sum()))
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(10):
    step()
e1.record()
torch.cuda.synchronize()
print(f"STEP ms (packed={args.packed}): {e0.elapsed_time(e1) / 10:.3f}")

if args.breakdown:
    def t(fn, reps=20):
        fn(); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            r = fn()
        e1.record(); torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps, r

    with torch.no_grad():
        ms_p, pr = t(lambda: ops.fused_project_sh(P["means"], P["quats"], P["scales"], P["opacities"], P["sh"], vm, K, W, H, 3))
        radii, m2, dep, con, col, _ = pr
        op = P["opacities"][None].contiguous()
        tw, th = 120, 68
        ms_i, ir = t(lambda: ops.isect_tiles(m2, radii, dep, 16, tw, th, conics=con, opacities=op))
        ms_in, _ = t(lambda: ops.isect_tiles(m2, radii, dep, 16, tw, th, conics=con, opacities=op, sort=False))
        tpg, ids, fl = ir
        ms_o, off = t(lambda: ops.isect_offset_encode(ids, 1, tw, th))
        ms_r, _ = t(lambda: ops.rasterize_to_pixels(m2, con, col, op, W, H, 16, off, fl))
    m2g, cong, colg, opg = (x.detach().clone().requires_grad_(True) for x in (m2, con, col, op))
    rc, ra = ops.rasterize_to_pixels(m2g, cong, colg, opg, W, H, 16, off, fl)
    v = torch.randn_like(rc)
    ms_rb, g = t(lambda: torch.autograd.grad((rc,), (m2g, cong, colg, opg), (v,), retain_graph=True))
    L = gsplat_b200._cabi.lib()
    from gsplat_b200._cabi import ptr, stream
    outs = [torch.empty_like(P[k]) for k in ("means", "quats", "scales", "sh")]
    N = P["means"].shape[0]
    vd = torch.zeros_like(dep)
    def pb():
        return L.gsb200_project_sh_bwd(1, N, 16, 3, ptr(P["means"]), ptr(P["quats"]), ptr(P["scales"]), ptr(P["sh"]), ptr(vm), ptr(K), W, H, 0.3,
                                      ptr(radii), ptr(con), None, ptr(col), g[0].data_ptr(), g[0].stride(-2), ptr(vd), 1, g[1].data_ptr(), g[1].stride(-2),
                                      g[2].data_ptr(), g[2].stride(-2), None, ptr(outs[0]), ptr(outs[1]), ptr(outs[2]), ptr(outs[3]), None, stream())
    ms_pb, _ = t(pb)
    ms_step, _ = t(step, 10)
    print("note: each stage below is timed by calling its operator back to back outside autograd (wide-key isect_tiles, per-intersection "
          "pack, no row records, host sync included): the stages do not add up to the step and are not what rasterization() runs since "
          "round 2 -- use an ncu launch list of the real step for its shares")
    print(f"BREAKDOWN ms: project_sh_fwd {ms_p:.3f} | isect(order+count+scan+sync+emit+sort) {ms_i:.3f} (unsorted {ms_in:.3f}) | offsets {ms_o:.3f} | "
          f"raster_fwd(pack+raster) {ms_r:.3f} | raster_bwd(+memset) {ms_rb:.3f} | project_sh_bwd {ms_pb:.3f} | full step {ms_step:.3f}")
