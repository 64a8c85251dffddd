"""Times the per-pixel contributor queries on bench.py's scene (the garden crop tiled 3 x 3, 1M Gaussians, one
1920x1080 view, seed 42): rasterize_num_contributing_gaussians, rasterize_contributing_gaussian_ids,
rasterize_top_contributing_gaussian_ids with K = 8 and 32, and the three _sparse forms on 4096 seeded pixels, with one
rasterize_to_pixels forward on the same intersections for scale.

With --2dgs the same scene is projected as surfels (fully_fused_projection_2dgs, the lists of isect_tiles_sorted and
isect_tiles_sparse) and the six _2dgs queries are timed the same way, with one rasterize_to_pixels_2dgs forward (RGB +
depth) for scale; the record also holds the surfel walk's top-K bound.

With --3dgut the scene goes through the UT projection (fully_fused_projection_with_ut) and the distorted pinhole of
tools/bench_ut.py (radial and tangential coefficients), the lists of isect_tiles_sorted and isect_tiles_sparse
(conics=None), and the six _eval3d queries are timed the same way, with one rasterize_to_pixels_eval3d forward on the
same lists for scale; --rolling-shutter adds a top-to-bottom rolling shutter (bench_ut.py's end pose).  The record also
holds the eval3d walk's top-K bound.

    python tools/contrib_bench.py [--2dgs | --3dgut [--rolling-shutter]] [--steps 20] [--warmup 5]

Each call is timed with CUDA events after `warmup` untimed calls; the ids query includes its host read of the largest
count.  Projection, tile intersection and the sparse layout run once, outside the timed calls.  Prints one JSON line
with the median times (ms), the pair count, and the device name and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)

import gsplat_b200 as gs  # noqa: E402
from tests import scene  # noqa: E402
from tools.indices_bench import device_info, timed  # noqa: E402

W, H, SCENE_GRID, N_SPARSE = 1920, 1080, 3, 4096
TW, TH = (W + 15) // 16, (H + 15) // 16


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--2dgs", dest="surfels", action="store_true", help="the 2DGS queries on the scene's surfels")
    ap.add_argument("--3dgut", dest="ut", action="store_true", help="the 3DGUT queries through a distorted pinhole")
    ap.add_argument("--rolling-shutter", action="store_true", help="--3dgut with a top-to-bottom rolling shutter")
    args = ap.parse_args()
    if args.rolling_shutter and not args.ut:
        ap.error("--rolling-shutter needs --3dgut")
    if not torch.cuda.is_available():
        raise SystemExit("contrib_bench needs a GPU")
    dev = "cuda:0"
    sc = scene.make_scene(scene_grid=SCENE_GRID, sh_degree=0)
    Ks = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)[:1]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    vm = t(sc["viewmats"][:1])
    opac = t(sc["opacities"])[None].contiguous()
    colors = t(sc["colors"])[None].contiguous()
    rec = {"image": f"{W}x{H}", "n_gaussians": int(sc["means"].shape[0]), "sparse_pixels": N_SPARSE, "steps": args.steps}
    ms = lambda fn: timed(fn, args.steps, args.warmup)[0]  # noqa: E731
    if args.surfels:
        return main_2dgs(sc, t, vm, t(Ks), opac, colors, rec, ms, dev)
    if args.ut:
        return main_3dgut(sc, t, vm, t(Ks), opac, colors, rec, ms, dev, args.rolling_shutter)
    with torch.no_grad():
        radii, m2, depths, conics, _ = gs.fully_fused_projection(t(sc["means"]), None, t(sc["quats"]), t(sc["scales"]), vm, t(Ks), W, H)
        _, ids, fl = gs.isect_tiles(m2, radii, depths, 16, TW, TH, conics=conics, opacities=opac)
        off = gs.isect_offset_encode(ids, 1, TW, TH)
        a = (m2, conics, opac, off, fl, W, H, 16)
        counts, _ = gs.rasterize_num_contributing_gaussians(*a)
        rec["isects"] = int(fl.shape[0])
        rec["pairs"] = int(counts.sum())
        rec["max_count"] = int(counts.max())
        rec["raster_fwd_ms"] = ms(lambda: gs.rasterize_to_pixels(m2, conics, colors, opac, W, H, 16, off, fl))
        rec["num_ms"] = ms(lambda: gs.rasterize_num_contributing_gaussians(*a))
        rec["ids_ms"] = ms(lambda: gs.rasterize_contributing_gaussian_ids(*a, counts))
        for k in (8, 32):
            rec[f"top{k}_ms"] = ms(lambda: gs.rasterize_top_contributing_gaussian_ids(*a, k))

        active, amask, words, cum, pmap = _sparse_pixels(t, dev)
        s_off, s_fl = gs.isect_tiles_sparse(m2, radii, depths, amask, active, 1, 16, TW, TH)
        s = (m2, conics, opac, active, s_off, s_fl, words, cum, pmap)
        grid = (W, H, 16, TW, TH)
        s_counts, _ = gs.rasterize_num_contributing_gaussians_sparse(*s, *grid)
        rec["sparse_num_ms"] = ms(lambda: gs.rasterize_num_contributing_gaussians_sparse(*s, *grid))
        rec["sparse_ids_ms"] = ms(lambda: gs.rasterize_contributing_gaussian_ids_sparse(*s, s_counts, *grid))
        rec["sparse_top8_ms"] = ms(lambda: gs.rasterize_top_contributing_gaussian_ids_sparse(*s, *grid, 8))
    rec.update(device_info())
    print(json.dumps(rec), flush=True)
    return 0


def _sparse_pixels(t, dev):
    """the 4096 seeded pixels of one image and their sparse layout"""
    rng = np.random.RandomState(42)
    flat = rng.choice(W * H, N_SPARSE, replace=False)
    pixels = t(np.stack([flat // W, flat % W], -1).astype(np.int32))
    image_ids = torch.zeros(N_SPARSE, device=dev, dtype=torch.int32)
    return gs.build_sparse_tile_layout(pixels, image_ids, 1, 16, TW, TH)


def main_2dgs(sc, t, vm, Ks, opac, colors, rec, ms, dev) -> int:
    rec["pipeline"] = "2dgs"
    with torch.no_grad():
        radii, m2, depths, rt, nrm = gs.fully_fused_projection_2dgs(t(sc["means"]), t(sc["quats"]), t(sc["scales"]), vm, Ks,
                                                                    W, H)
        hits = gs.ops.isect_tiles_sorted(m2, radii, depths, 16, TW, TH)
        off, fl = hits.isect_offsets.reshape(1, TH, TW), hits.flatten_ids
        a = (m2, rt, opac, off, fl, W, H, 16)
        counts, _ = gs.rasterize_num_contributing_gaussians_2dgs(*a)
        rec["isects"] = int(fl.shape[0])
        rec["pairs"] = int(counts.sum())
        rec["max_count"] = int(counts.max())
        rec["surfel_top_k_bound"] = gs.ops._max_depth_samples(torch.device(dev), "gsb200_surfel_contrib_max_samples")
        rgbd = torch.cat([colors, depths[..., None]], -1).contiguous()
        densify = torch.zeros_like(m2)
        rec["raster_2dgs_fwd_ms"] = ms(lambda: gs.rasterize_to_pixels_2dgs(m2, rt, rgbd, opac, nrm, densify, W, H, 16, off, fl))
        rec["num_ms"] = ms(lambda: gs.rasterize_num_contributing_gaussians_2dgs(*a))
        rec["ids_ms"] = ms(lambda: gs.rasterize_contributing_gaussian_ids_2dgs(*a, counts))
        for k in (8, 32):
            rec[f"top{k}_ms"] = ms(lambda: gs.rasterize_top_contributing_gaussian_ids_2dgs(*a, k))

        active, amask, words, cum, pmap = _sparse_pixels(t, dev)
        s_off, s_fl = gs.isect_tiles_sparse(m2, radii, depths, amask, active, 1, 16, TW, TH)
        s = (m2, rt, opac, active, s_off, s_fl, words, cum, pmap)
        grid = (W, H, 16, TW, TH)
        s_counts, _ = gs.rasterize_num_contributing_gaussians_2dgs_sparse(*s, *grid)
        rec["sparse_num_ms"] = ms(lambda: gs.rasterize_num_contributing_gaussians_2dgs_sparse(*s, *grid))
        rec["sparse_ids_ms"] = ms(lambda: gs.rasterize_contributing_gaussian_ids_2dgs_sparse(*s, s_counts, *grid))
        for k in (8, 32):
            rec[f"sparse_top{k}_ms"] = ms(lambda: gs.rasterize_top_contributing_gaussian_ids_2dgs_sparse(*s, *grid, k))
    rec.update(device_info())
    print(json.dumps(rec), flush=True)
    return 0


def main_3dgut(sc, t, vm, Ks, opac, colors, rec, ms, dev, rolling) -> int:
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from bench_ut import _end_pose

    rec["pipeline"] = "3dgut-rolling" if rolling else "3dgut"
    cam = dict(radial_coeffs=t(np.float32([[0.05, -0.02, 0.0, 0.0, 0.0, 0.0]])),
               tangential_coeffs=t(np.float32([[0.001, -0.001]])))
    if rolling:
        cam.update(rolling_shutter=gs.RollingShutterType.ROLLING_TOP_TO_BOTTOM, viewmats_rs=_end_pose(vm))
    means, quats, scales = t(sc["means"]), t(sc["quats"]), t(sc["scales"])
    with torch.no_grad():
        radii, m2, depths, _, _ = gs.fully_fused_projection_with_ut(means, quats, scales, opac[0], vm, Ks, W, H, **cam)
        hits = gs.ops.isect_tiles_sorted(m2, radii, depths, 16, TW, TH)
        off, fl = hits.isect_offsets.reshape(1, TH, TW), hits.flatten_ids
        geo = (means, quats, scales, opac, vm, Ks)
        a = geo + (off, fl, W, H, 16)
        counts, _ = gs.rasterize_num_contributing_gaussians_eval3d(*a, **cam)
        rec["isects"] = int(fl.shape[0])
        rec["pairs"] = int(counts.sum())
        rec["max_count"] = int(counts.max())
        rec["eval3d_top_k_bound"] = gs.ops._max_depth_samples(torch.device(dev), "gsb200_eval3d_contrib_max_samples")
        rec["eval3d_fwd_ms"] = ms(lambda: gs.rasterize_to_pixels_eval3d(means, quats, scales, colors, opac, vm, Ks, W, H, 16,
                                                                        off, fl, **cam))
        rec["num_ms"] = ms(lambda: gs.rasterize_num_contributing_gaussians_eval3d(*a, **cam))
        rec["ids_ms"] = ms(lambda: gs.rasterize_contributing_gaussian_ids_eval3d(*a, counts, **cam))
        for k in (8, 32):
            rec[f"top{k}_ms"] = ms(lambda: gs.rasterize_top_contributing_gaussian_ids_eval3d(*a, k, **cam))

        active, amask, words, cum, pmap = _sparse_pixels(t, dev)
        s_off, s_fl = gs.isect_tiles_sparse(m2, radii, depths, amask, active, 1, 16, TW, TH)
        s = geo + (active, s_off, s_fl, words, cum, pmap)
        grid = (W, H, 16, TW, TH)
        s_counts, _ = gs.rasterize_num_contributing_gaussians_eval3d_sparse(*s, *grid, **cam)
        rec["sparse_num_ms"] = ms(lambda: gs.rasterize_num_contributing_gaussians_eval3d_sparse(*s, *grid, **cam))
        rec["sparse_ids_ms"] = ms(lambda: gs.rasterize_contributing_gaussian_ids_eval3d_sparse(*s, s_counts, *grid, **cam))
        for k in (8, 32):
            rec[f"sparse_top{k}_ms"] = ms(lambda: gs.rasterize_top_contributing_gaussian_ids_eval3d_sparse(*s, *grid, k,
                                                                                                          **cam))
    rec.update(device_info())
    print(json.dumps(rec), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
