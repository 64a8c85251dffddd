"""Sparse-pixel rendering against the dense pipeline on bench.py's scene (1M Gaussians, one 1920x1080 view, seed 42).

    python tools/sparse_bench.py [--2dgs | --3dgut [--rolling-shutter]] [--steps 20] [--warmup 5] [--out FILE]

One step of each pipeline, timed on the host around a device synchronise (both pipelines read one count back to the
host, so a step is not asynchronous anyway):
  sparse: build_sparse_tile_layout + isect_tiles_sparse + rasterize_to_pixels_sparse forward + backward;
  dense:  isect_tiles(conics=None) + isect_offset_encode + rasterize_to_pixels forward + backward over the whole image
          (the same radius-AABB tile lists), the loss on the requested pixels only.
With --2dgs the same scene is projected as surfels (fully_fused_projection_2dgs, RGB + depth channel) and the pipelines
are the 2DGS ones:
  sparse: build_sparse_tile_layout + isect_tiles_sparse + rasterize_to_pixels_2dgs_sparse forward + backward;
  dense:  isect_tiles_sorted + rasterize_to_pixels_2dgs forward + backward over the whole image (the same lists), the
          loss on all five outputs at the requested pixels only.
With --3dgut the same scene (colours, not SH) is projected by fully_fused_projection_with_ut through the distorted
pinhole of tools/bench_ut.py, and the pipelines are the 3DGUT ones:
  sparse: build_sparse_tile_layout + isect_tiles_sparse + rasterize_to_pixels_eval3d_sparse forward + backward;
  dense:  isect_tiles_sorted + rasterize_to_pixels_eval3d forward + backward over the whole image (the same lists), the
          loss on the requested pixels only.
--rolling-shutter (with --3dgut) exposes the image top to bottom, the end pose being tools/bench_ut.py's (the start
pose turned by 2 degrees and moved by 0.03).
Workloads: (a) 4096 random pixels, (b) sixteen 64x64 patches, (c) every pixel.  The projection runs once, outside the
timed steps.  Prints one JSON line per workload with the median step times, and the device name and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

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


def workloads(rng):
    out = {}
    flat = rng.choice(W * H, 4096, replace=False)
    out["a_4096_random"] = np.stack([flat // W, flat % W], -1)
    ys, xs = rng.randint(0, H - 64, 16), rng.randint(0, W - 64, 16)
    yy, xx = np.meshgrid(np.arange(64), np.arange(64), indexing="ij")
    p = np.concatenate([np.stack([y + yy.ravel(), x + xx.ravel()], -1) for y, x in zip(ys, xs)])
    out["b_16_patches_64"] = np.unique(p, axis=0)  # overlapping patches: each pixel once
    yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    out["c_every_pixel"] = np.stack([yy.ravel(), xx.ravel()], -1)
    return out


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", help="also append the JSON lines to this file")
    ap.add_argument("--2dgs", dest="surfels", action="store_true", help="the 2DGS pipelines on the scene's surfels")
    ap.add_argument("--3dgut", dest="ut", action="store_true", help="the 3DGUT pipelines through a distorted pinhole")
    ap.add_argument("--rolling-shutter", action="store_true", help="with --3dgut: a top-to-bottom rolling shutter")
    args = ap.parse_args()
    if args.rolling_shutter and not args.ut:
        ap.error("--rolling-shutter needs --3dgut")
    if args.surfels and args.ut:
        ap.error("--2dgs and --3dgut are exclusive")
    if not torch.cuda.is_available():
        raise SystemExit("sparse_bench needs a GPU")
    dev = "cuda:0"
    sc = scene.make_scene(scene_grid=SCENE_GRID, sh_degree=0)
    Ks = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    N = sc["means"].shape[0]
    if args.surfels:
        return main_2dgs(args, sc, Ks, t, N, dev)
    if args.ut:
        return main_3dgut(args, sc, Ks, t, N, dev)
    with torch.no_grad():
        radii, m2, depths, conics, _ = gs.fully_fused_projection(
            t(sc["means"]), None, t(sc["quats"]), t(sc["scales"]), t(sc["viewmats"][:1]), t(Ks[:1]), W, H
        )
    colors = t(sc["colors"])[None].contiguous()
    opac = t(sc["opacities"])[None].contiguous()
    params = [x.detach().clone().requires_grad_(True) for x in (m2, conics, colors, opac)]
    info = device_info()
    lines = []

    for name, pix in workloads(np.random.RandomState(42)).items():
        pixels = t(pix.astype(np.int32))
        image_ids = torch.zeros(pixels.shape[0], device=dev, dtype=torch.int32)
        P = pixels.shape[0]
        v = torch.randn((P, 3), device=dev, generator=torch.Generator(device=dev).manual_seed(0))
        v_img = torch.zeros((1, H, W, 3), device=dev)
        v_img[0, pixels[:, 0].long(), pixels[:, 1].long()] = v
        stats = {}

        def sparse_step():
            active, amask, words, cum, pmap = gs.build_sparse_tile_layout(pixels, image_ids, 1, 16, TW, TH)
            toff, fl = gs.isect_tiles_sparse(m2, radii, depths, amask, active, 1, 16, TW, TH)
            rc, _ = gs.rasterize_to_pixels_sparse(*params, image_ids, active, toff, fl, words, cum, pmap, W, H, 16, TW, TH)
            (rc * v).sum().backward()
            stats.update(n_active=int(active.shape[0]), n_isects=int(fl.shape[0]))

        def dense_step():
            _, ids, fl = gs.isect_tiles(m2, radii, depths, 16, TW, TH)
            off = gs.isect_offset_encode(ids, 1, TW, TH)
            rc, _ = gs.rasterize_to_pixels(*params, W, H, 16, off, fl)
            (rc * v_img).sum().backward()
            stats.update(dense_isects=int(fl.shape[0]))

        sparse_ms, sparse_min = _timed(sparse_step, args.steps, args.warmup)
        dense_ms, dense_min = _timed(dense_step, args.steps, args.warmup)
        rec = dict(
            workload=name, pixels=P, n_gaussians=N, image=f"{W}x{H}", steps=args.steps, sparse_ms=round(sparse_ms, 3),
            sparse_min_ms=round(sparse_min, 3), dense_ms=round(dense_ms, 3), dense_min_ms=round(dense_min, 3),
            sparse_over_dense=round(sparse_ms / dense_ms, 3), **stats, **info,
        )
        line = json.dumps(rec)
        print(line, flush=True)
        lines.append(line)
    _write(args, lines)
    return 0


def _write(args, lines):
    if args.out:
        with open(args.out, "a") as f:
            f.write("\n".join(lines) + "\n")


def _timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts) * 1e3, min(ts) * 1e3


def main_2dgs(args, sc, Ks, t, N, dev) -> int:
    D = 4  # RGB + the depth channel that distortion and median depth are taken from
    with torch.no_grad():
        radii, m2, depths, rt, nrm = gs.fully_fused_projection_2dgs(
            t(sc["means"]), t(sc["quats"]), t(sc["scales"]), t(sc["viewmats"][:1]), t(Ks[:1]), W, H
        )
        colors = torch.cat([t(sc["colors"])[None], depths[..., None]], -1).contiguous()
        opac = t(sc["opacities"])[None].contiguous()
    params = [x.detach().clone().requires_grad_(True) for x in (m2, rt, colors, opac, nrm)]
    densify = torch.zeros_like(m2, requires_grad=True)
    info = device_info()
    lines = []
    for name, pix in workloads(np.random.RandomState(42)).items():
        pixels = t(pix.astype(np.int32))
        image_ids = torch.zeros(pixels.shape[0], device=dev, dtype=torch.int32)
        P = pixels.shape[0]
        g = torch.Generator(device=dev).manual_seed(0)
        v = [torch.randn((P, k), device=dev, generator=g) for k in (D, 1, 3, 1, 1)]
        v_img = []
        for x in v:
            img = torch.zeros((1, H, W, x.shape[-1]), device=dev)
            img[0, pixels[:, 0].long(), pixels[:, 1].long()] = x
            v_img.append(img)
        stats = {}

        def sparse_step():
            active, amask, words, cum, pmap = gs.build_sparse_tile_layout(pixels, image_ids, 1, 16, TW, TH)
            toff, fl = gs.isect_tiles_sparse(m2, radii, depths, amask, active, 1, 16, TW, TH)
            outs = gs.rasterize_to_pixels_2dgs_sparse(
                *params, densify, image_ids, active, toff, fl, words, cum, pmap, W, H, 16, TW, TH, distloss=True
            )
            sum((o * c).sum() for o, c in zip(outs, v)).backward()
            stats.update(n_active=int(active.shape[0]), n_isects=int(fl.shape[0]))

        def dense_step():
            hits = gs.ops.isect_tiles_sorted(m2, radii, depths, 16, TW, TH)
            off = hits.isect_offsets.reshape(1, TH, TW)
            outs = gs.rasterize_to_pixels_2dgs(*params, densify, W, H, 16, off, hits.flatten_ids, distloss=True)
            sum((o * c).sum() for o, c in zip(outs, v_img)).backward()
            stats.update(dense_isects=int(hits.flatten_ids.shape[0]))

        sparse_ms, sparse_min = _timed(sparse_step, args.steps, args.warmup)
        dense_ms, dense_min = _timed(dense_step, args.steps, args.warmup)
        rec = dict(
            pipeline="2dgs", workload=name, pixels=P, n_gaussians=N, image=f"{W}x{H}", channels=D, steps=args.steps,
            sparse_ms=round(sparse_ms, 3), sparse_min_ms=round(sparse_min, 3), dense_ms=round(dense_ms, 3),
            dense_min_ms=round(dense_min, 3), sparse_over_dense=round(sparse_ms / dense_ms, 3), **stats, **info,
        )
        line = json.dumps(rec)
        print(line, flush=True)
        lines.append(line)
    _write(args, lines)
    return 0


def main_3dgut(args, sc, Ks, t, N, dev) -> int:
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from bench_ut import _end_pose

    vm, K = t(sc["viewmats"][:1]), t(Ks[:1])
    # the distorted pinhole of tools/bench_ut.py --distorted
    cam = dict(radial_coeffs=t(np.float32([[0.05, -0.02, 0.0, 0.0, 0.0, 0.0]])), tangential_coeffs=t(np.float32([[0.001, -0.001]])))
    if args.rolling_shutter:
        cam.update(rolling_shutter=gs.RollingShutterType.ROLLING_TOP_TO_BOTTOM, viewmats_rs=_end_pose(vm))
    means, quats, scales = t(sc["means"]), t(sc["quats"]), t(sc["scales"])
    colors = t(sc["colors"])[None].contiguous()
    opac = t(sc["opacities"])[None].contiguous()
    with torch.no_grad():
        radii, m2, depths, _, _ = gs.fully_fused_projection_with_ut(means, quats, scales, opac[0], vm, K, W, H, **cam)
    params = [x.detach().clone().requires_grad_(True) for x in (means, quats, scales, colors, opac)]
    info = device_info()
    lines = []
    for name, pix in workloads(np.random.RandomState(42)).items():
        pixels = t(pix.astype(np.int32))
        image_ids = torch.zeros(pixels.shape[0], device=dev, dtype=torch.int32)
        P = pixels.shape[0]
        v = torch.randn((P, 3), device=dev, generator=torch.Generator(device=dev).manual_seed(0))
        v_img = torch.zeros((1, H, W, 3), device=dev)
        v_img[0, pixels[:, 0].long(), pixels[:, 1].long()] = v
        stats = {}

        def sparse_step():
            active, amask, words, cum, pmap = gs.build_sparse_tile_layout(pixels, image_ids, 1, 16, TW, TH)
            toff, fl = gs.isect_tiles_sparse(m2, radii, depths, amask, active, 1, 16, TW, TH)
            rc, _ = gs.rasterize_to_pixels_eval3d_sparse(
                *params, vm, K, image_ids, active, toff, fl, words, cum, pmap, W, H, 16, TW, TH, **cam
            )
            (rc * v).sum().backward()
            stats.update(n_active=int(active.shape[0]), n_isects=int(fl.shape[0]))

        def dense_step():
            hits = gs.ops.isect_tiles_sorted(m2, radii, depths, 16, TW, TH)
            off = hits.isect_offsets.reshape(1, TH, TW)
            rc, _ = gs.rasterize_to_pixels_eval3d(*params, vm, K, W, H, 16, off, hits.flatten_ids, **cam)
            (rc * v_img).sum().backward()
            stats.update(dense_isects=int(hits.flatten_ids.shape[0]))

        sparse_ms, sparse_min = _timed(sparse_step, args.steps, args.warmup)
        dense_ms, dense_min = _timed(dense_step, args.steps, args.warmup)
        rec = dict(
            pipeline="3dgut", camera="pinhole radial+tangential",
            shutter="rolling top to bottom" if args.rolling_shutter else "global", workload=name, pixels=P,
            n_gaussians=N, image=f"{W}x{H}", steps=args.steps, sparse_ms=round(sparse_ms, 3),
            sparse_min_ms=round(sparse_min, 3), dense_ms=round(dense_ms, 3), dense_min_ms=round(dense_min, 3),
            sparse_over_dense=round(sparse_ms / dense_ms, 3), **stats, **info,
        )
        line = json.dumps(rec)
        print(line, flush=True)
        lines.append(line)
    _write(args, lines)
    return 0


if __name__ == "__main__":
    sys.exit(main())
