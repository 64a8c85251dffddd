#!/usr/bin/env python
"""Times one 3DGUT step (fully_fused_projection_with_ut + isect_tiles + isect_offset_encode + rasterize_to_pixels_eval3d
forward and backward) next to the EWA step (fully_fused_projection + the same lists + rasterize_to_pixels forward and
backward) on bench.py's scene (1M Gaussians, one 1920x1080 view) with a pinhole camera.  Median of --steps timed steps after --warmup, CUDA events; prints
the device name and power limit with the numbers, as one JSON line.

    python tools/bench_ut.py [--steps 20] [--warmup 5] [--distorted] [--rasterization] [--rolling-shutter]
                             [--camera ftheta]

--rasterization times the public call instead: rasterization(with_ut=True, with_eval3d=True, sh_degree=3,
packed=False) forward and backward on the same scene with SH degree 3, next to the same operators chained by hand, and
reports the difference as the public call's overhead.

--rolling-shutter times the rolling-shutter step (top to bottom; the end pose is the start pose turned by 2 degrees and
moved by 0.03) next to the global-shutter step on the same scene, alternated step by step: the operator chain, or with
--rasterization the public call.  It also times the UT projection alone under both shutters and reports its share of
each step.

--camera ftheta times the operator step through an FTheta camera (the 120-degree cross-left calibration of
tests/golden/ftheta_calibrations.json scaled to 1920 pixels wide) in the global z order and in the Euclidean order
(global_z_order=False) next to the pinhole step on the same scene, alternated step by step, with the UT projection
alone under each and its share of the step.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import gsplat_b200 as gs  # noqa: E402
from tests import scene  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--distorted", action="store_true", help="pinhole with radial and tangential coefficients")
    ap.add_argument("--rasterization", action="store_true",
                    help="time rasterization(with_ut=True, with_eval3d=True, sh_degree=3) next to the hand-chained operators")
    ap.add_argument("--rolling-shutter", action="store_true",
                    help="time the rolling-shutter step next to the global-shutter step")
    ap.add_argument("--camera", choices=("pinhole", "ftheta"), default="pinhole",
                    help="ftheta: time the FTheta step in both depth orders next to the pinhole step")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ut needs a GPU"
    if a.camera == "ftheta":
        return bench_ftheta(a)
    if a.rolling_shutter:
        return bench_rolling_shutter(a)
    if a.rasterization:
        return bench_rasterization(a)
    dev = "cuda"
    # bench.py's scene: the garden crop tiled 3x3 (about 1M Gaussians), one 1920x1080 view; colours instead of SH
    sc = scene.make_scene(scene_grid=3, sh_degree=0)
    W, H = 1920, 1080
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)  # noqa: E731
    means, quats, scales = (t(sc[k]).requires_grad_(True) for k in ("means", "quats", "scales"))
    opac = t(sc["opacities"])[None].contiguous().requires_grad_(True)
    colors = t(sc["colors"])[None].contiguous().requires_grad_(True)
    vm, K = t(sc["viewmats"][:1]), t(scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)[:1])
    co = dict(radial_coeffs=t(np.float32([[0.05, -0.02, 0.0, 0.0, 0.0, 0.0]])), tangential_coeffs=t(np.float32([[0.001, -0.001]]))) if a.distorted else {}
    tw, th = (W + 15) // 16, (H + 15) // 16

    def ut_step():
        r, m2, d, _, _ = gs.fully_fused_projection_with_ut(means.detach(), quats.detach(), scales.detach(), opac.detach()[0], vm, K, W, H, **co)
        _, ii, fl = gs.isect_tiles(m2, r, d, 16, tw, th)
        offs = gs.isect_offset_encode(ii, 1, tw, th)
        rc, ra = gs.rasterize_to_pixels_eval3d(means, quats, scales, colors, opac, vm, K, W, H, 16, offs, fl, **co)
        (rc.sum() + ra.sum()).backward()
        return fl.numel()

    def ewa_step():
        r, m2, d, con, _ = gs.fully_fused_projection(means, None, quats, scales, vm, K, W, H)
        _, ii, fl = gs.isect_tiles(m2, r, d, 16, tw, th)
        offs = gs.isect_offset_encode(ii, 1, tw, th)
        rc, ra = gs.rasterize_to_pixels(m2, con, colors, opac, W, H, 16, offs, fl)
        (rc.sum() + ra.sum()).backward()
        return fl.numel()

    res = {}
    for name, fn in (("ewa", ewa_step), ("ut", ut_step)):
        for _ in range(a.warmup):
            n = fn()
        times = []
        for _ in range(a.steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        res[name] = {"median_ms": float(np.median(times)), "n_isects": int(n)}
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    res.update(device=torch.cuda.get_device_name(0), power_limit=q.stdout.strip(), gaussians=int(means.shape[0]), width=W,
               height=H, distorted=a.distorted, steps=a.steps)
    print(json.dumps(res))


def _device_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(device=torch.cuda.get_device_name(0), power_limit=q.stdout.strip())


def bench_rasterization(a):
    """rasterization(with_ut=True, with_eval3d=True, sh_degree=3, packed=False) forward + backward against the same
    work chained by hand (UT projection, SH + clamp, isect_tiles + isect_offset_encode, eval3d compositing), alternated
    step by step so that both see the same machine state."""
    dev = "cuda"
    sc = scene.make_scene(scene_grid=3, sh_degree=3)
    W, H = 1920, 1080
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)  # noqa: E731
    means, quats, scales, opac, sh = (t(sc[k]).requires_grad_(True) for k in ("means", "quats", "scales", "opacities", "sh"))
    vm, K = t(sc["viewmats"][:1]), t(scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)[:1])
    co = dict(radial_coeffs=t(np.float32([[0.05, -0.02, 0.0, 0.0, 0.0, 0.0]])), tangential_coeffs=t(np.float32([[0.001, -0.001]]))) if a.distorted else {}
    tw, th = (W + 15) // 16, (H + 15) // 16
    N = means.shape[0]

    def public():
        rc, ra, meta = gs.rasterization(means, quats, scales, opac, sh, vm, K, W, H, sh_degree=3, packed=False, with_ut=True,
                                        with_eval3d=True, **co)
        (rc.sum() + ra.sum()).backward()
        return meta["flatten_ids"].numel()

    def chain():
        r, m2, d, _, _ = gs.fully_fused_projection_with_ut(means.detach(), quats.detach(), scales.detach(), opac.detach(), vm, K,
                                                          W, H, **co)
        feat = torch.clamp_min(gs.spherical_harmonics(3, means, vm, sh, masks=(r > 0).all(-1)) + 0.5, 0.0)
        _, ii, fl = gs.isect_tiles(m2, r, d, 16, tw, th)
        offs = gs.isect_offset_encode(ii, 1, tw, th)
        o = torch.broadcast_to(opac[None], (1, N))
        rc, ra = gs.rasterize_to_pixels_eval3d(means, quats, scales, feat, o, vm, K, W, H, 16, offs, fl, **co)
        (rc.sum() + ra.sum()).backward()
        return fl.numel()

    fns = {"rasterization": public, "hand_chain": chain}
    for fn in fns.values():
        for _ in range(a.warmup):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in fns}
    n = {}
    for _ in range(a.steps):
        for name, fn in fns.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            n[name] = fn()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1))
    res = {name: {"median_ms": float(np.median(v)), "min_ms": float(np.min(v)), "n_isects": int(n[name])} for name, v in times.items()}
    res["overhead_ms"] = res["rasterization"]["median_ms"] - res["hand_chain"]["median_ms"]
    res.update(_device_info(), gaussians=int(N), width=W, height=H, sh_degree=3, distorted=a.distorted, steps=a.steps)
    print(json.dumps(res))


def _end_pose(vm: torch.Tensor, degrees=2.0, shift=0.03) -> torch.Tensor:
    """vm [C, 4, 4] turned by `degrees` about a fixed axis and moved by `shift` in the camera frame."""
    axis = torch.tensor([0.3, 0.8, -0.5], dtype=torch.float64)
    axis = axis / axis.norm()
    k = torch.tensor([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]], dtype=torch.float64)
    th = torch.tensor(degrees, dtype=torch.float64).deg2rad()
    delta = torch.eye(4, dtype=torch.float64)
    delta[:3, :3] = torch.eye(3, dtype=torch.float64) + torch.sin(th) * k + (1 - torch.cos(th)) * (k @ k)
    delta[:3, 3] = shift * axis
    return (delta.to(vm.device) @ vm.double()).float().contiguous()


def _time(fns, steps, warmup):
    """Median and min ms of each fn, alternated step by step; its last return value."""
    for fn in fns.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    times, n = {k: [] for k in fns}, {}
    for _ in range(steps):
        for name, fn in fns.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            n[name] = fn()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1))
    return {name: {"median_ms": float(np.median(v)), "min_ms": float(np.min(v)), "out": n[name]} for name, v in times.items()}


def bench_rolling_shutter(a):
    dev = "cuda"
    sc = scene.make_scene(scene_grid=3, sh_degree=3 if a.rasterization else 0)
    W, H = 1920, 1080
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)  # noqa: E731
    means, quats, scales = (t(sc[k]).requires_grad_(True) for k in ("means", "quats", "scales"))
    opac = t(sc["opacities"]).requires_grad_(True)
    colors = t(sc["sh"] if a.rasterization else sc["colors"][None]).requires_grad_(True)
    vm, K = t(sc["viewmats"][:1]), t(scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)[:1])
    vm_rs = _end_pose(vm)
    co = dict(radial_coeffs=t(np.float32([[0.05, -0.02, 0.0, 0.0, 0.0, 0.0]])), tangential_coeffs=t(np.float32([[0.001, -0.001]]))) if a.distorted else {}
    shutters = {"global": {}, "rolling": dict(rolling_shutter=gs.RollingShutterType.ROLLING_TOP_TO_BOTTOM, viewmats_rs=vm_rs)}
    tw, th = (W + 15) // 16, (H + 15) // 16
    N = means.shape[0]

    def step(rs):
        if a.rasterization:
            rc, ra, meta = gs.rasterization(means, quats, scales, opac, colors, vm, K, W, H, sh_degree=3, packed=False,
                                            with_ut=True, with_eval3d=True, **co, **rs)
            fl = meta["flatten_ids"]
        else:
            r, m2, d, _, _ = gs.fully_fused_projection_with_ut(means.detach(), quats.detach(), scales.detach(), opac.detach(), vm,
                                                              K, W, H, **co, **rs)
            _, ii, fl = gs.isect_tiles(m2, r, d, 16, tw, th)
            offs = gs.isect_offset_encode(ii, 1, tw, th)
            o = torch.broadcast_to(opac[None], (1, N))
            rc, ra = gs.rasterize_to_pixels_eval3d(means, quats, scales, colors, o, vm, K, W, H, 16, offs, fl, **co, **rs)
        (rc.sum() + ra.sum()).backward()
        return fl.numel()

    def projection(rs):
        gs.fully_fused_projection_with_ut(means.detach(), quats.detach(), scales.detach(), opac.detach(), vm, K, W, H, **co, **rs)
        return 0

    fns = {f"{k}_step": (lambda rs=rs: step(rs)) for k, rs in shutters.items()}
    fns.update({f"{k}_projection": (lambda rs=rs: projection(rs)) for k, rs in shutters.items()})
    r = _time(fns, a.steps, a.warmup)
    res = {}
    for k in shutters:
        s, p = r[f"{k}_step"], r[f"{k}_projection"]
        res[k] = {"step_median_ms": s["median_ms"], "step_min_ms": s["min_ms"], "n_isects": int(s["out"]),
                  "projection_median_ms": p["median_ms"], "projection_share": p["median_ms"] / s["median_ms"]}
    res["rolling_over_global"] = res["rolling"]["step_median_ms"] / res["global"]["step_median_ms"]
    res.update(_device_info(), gaussians=int(N), width=W, height=H, rasterization=a.rasterization, distorted=a.distorted,
               shutter="ROLLING_TOP_TO_BOTTOM", steps=a.steps)
    print(json.dumps(res))


def bench_ftheta(a):

    dev = "cuda"
    sc = scene.make_scene(scene_grid=3, sh_degree=0)
    W, H = 1920, 1080
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)  # noqa: E731
    means, quats, scales = (t(sc[k]).requires_grad_(True) for k in ("means", "quats", "scales"))
    opac = t(sc["opacities"]).requires_grad_(True)
    colors = t(sc["colors"][None]).requires_grad_(True)
    vm, K = t(sc["viewmats"][:1]), t(scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)[:1])
    params, pp, size = scene.scaled(scene.calibrations()["cross_left_120fov"], W)
    assert size == (W, H)
    K_ft = t(np.float32([[[1, 0, pp[0]], [0, 1, pp[1]], [0, 0, 1]]]))
    ft = gs.FThetaCameraDistortionParameters(reference_poly=0, **params)
    cams = {"pinhole": (K, {}), "ftheta_z": (K_ft, dict(camera_model="ftheta", ftheta_coeffs=ft)),
            "ftheta_dist": (K_ft, dict(camera_model="ftheta", ftheta_coeffs=ft, global_z_order=False))}
    tw, th = (W + 15) // 16, (H + 15) // 16
    N = means.shape[0]

    def step(Kc, co):
        ev = {k: v for k, v in co.items() if k != "global_z_order"}  # the compositing takes no depth order
        r, m2, d, _, _ = gs.fully_fused_projection_with_ut(means.detach(), quats.detach(), scales.detach(), opac.detach(), vm,
                                                          Kc, W, H, **co)
        _, ii, fl = gs.isect_tiles(m2, r, d, 16, tw, th)
        offs = gs.isect_offset_encode(ii, 1, tw, th)
        o = torch.broadcast_to(opac[None], (1, N))
        rc, ra = gs.rasterize_to_pixels_eval3d(means, quats, scales, colors, o, vm, Kc, W, H, 16, offs, fl, **ev)
        (rc.sum() + ra.sum()).backward()
        return fl.numel()

    def projection(Kc, co):
        gs.fully_fused_projection_with_ut(means.detach(), quats.detach(), scales.detach(), opac.detach(), vm, Kc, W, H, **co)
        return 0

    fns = {f"{k}_step": (lambda c=c: step(*c)) for k, c in cams.items()}
    fns.update({f"{k}_projection": (lambda c=c: projection(*c)) for k, c in cams.items()})
    r = _time(fns, a.steps, a.warmup)
    res = {}
    for k in cams:
        s, p = r[f"{k}_step"], r[f"{k}_projection"]
        res[k] = {"step_median_ms": s["median_ms"], "step_min_ms": s["min_ms"], "n_isects": int(s["out"]),
                  "projection_median_ms": p["median_ms"], "projection_share": p["median_ms"] / s["median_ms"]}
    res.update(_device_info(), gaussians=int(N), width=W, height=H, calibration="cross_left_120fov", steps=a.steps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
