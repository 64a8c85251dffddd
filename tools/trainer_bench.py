#!/usr/bin/env python
"""BASELINE configs[4] (cfg5): the train loop of the reference's examples/simple_trainer.py on synthetic
data, run on one of two backends of the SAME installed ``gsplat`` package (baseline/_ref, the unmodified
reference installed by baseline/install_ref.py):

  --backend reference   stock path: gsplat.rasterization() -> torch.ops.gsplat.rasterization_3dgs with the
                        reference's registered autograd, gsplat.losses.ssim_loss (torch conv2d path),
                        gsplat.strategy.{DefaultStrategy, MCMCStrategy} on the reference's relocation / perturb ops.
  --backend b200        the same loop after gsplat_b200.dropin.apply() (INTEGRATION.md section A).

The loop restates examples/simple_trainer.py (file:line of what each statement mirrors):
  parameters + 6 fused Adam optimizers with the sqrt(BS) rule   :292-374
  ExponentialLR on the means                                    :808-813
  per step: batch to device (pinned, non_blocking)              :880-884
            SH degree schedule                                  :905
            activations exp / sigmoid / cat(sh0, shN)           :665-689
            rasterization(packed=False, absgrad=strategy.absgrad, sparse_grad=False, ...)   :722-749
            strategy.step_pre_backward                          :934-941
            L1 + SSIM, lerp with ssim_lambda                    :951-961
            (MCMC) opacity / scale regularisation               :996-999
            loss.backward(), loss.item() for the progress bar   :1001-1003
            optimizer.step() + zero_grad(set_to_none) x6, scheduler.step()   :1133-1149
            strategy.step_post_backward                         :1155-1176
Data: the synthetic workload of bench.py (test_garden crop tiled 3x3 = 1 006 065 points, 1080p, SH3); the targets
are renders of a "ground truth" parameter set (the workload's own colours / opacities, scales x ``--gt-scale``),
the trainable splats start from perturbed values (trainer-style init: init_opa, scales shrunk, grey SH).  Densification
runs on an accelerated schedule (``--refine-start/--refine-every``; defaults of the reference are 500 / 100) so that
the 1M -> 3M growth of cfg5 happens within a bench-sized run; both backends get the same schedule and seeds.

``--with-ut`` (with ``--strategy mcmc``, the only densification the reference supports for 3DGUT) trains 3DGUT:
rasterization(with_ut=True, with_eval3d=True) through the plain pinhole; the ground truth stays the EWA render.  Both
backends need the reference package in baseline/_ref; without it the tool prints a "not_run" line.

Prints ONE JSON line.  Test / bench infrastructure: it imports oracle/refcuda.py to locate the reference.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np
import torch

W_IMG, H_IMG = 1920, 1080


def make_cameras(sc, n_views: int, dev):
    """n_views cameras: the three garden poses + small rotations about the scene's up axis."""
    from tests import scene

    Ks = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W_IMG, H_IMG)
    vms, ks = [], []
    for v in range(n_views):
        base = sc["viewmats"][v % 3].astype(np.float64)
        ang = 0.04 * (v // 3)
        c, s = math.cos(ang), math.sin(ang)
        rot = np.array([[c, -s, 0, 0], [s, c, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]], np.float64)
        vms.append((base @ rot).astype(np.float32))
        ks.append(Ks[v % 3])
    viewmats = torch.from_numpy(np.stack(vms)).to(dev)
    return torch.linalg.inv(viewmats), torch.from_numpy(np.stack(ks)).to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", choices=["reference", "b200"], required=True)
    ap.add_argument("--strategy", choices=["default", "mcmc"], default="default")
    ap.add_argument("--steps", type=int, default=600)
    ap.add_argument("--views", type=int, default=6)
    ap.add_argument("--cap", type=int, default=3_000_000)
    ap.add_argument("--refine-start", type=int, default=100)
    ap.add_argument("--refine-every", type=int, default=25)
    ap.add_argument("--grow-grad2d", type=float, default=0.0002)
    ap.add_argument("--gt-scale", type=float, default=2.0)
    ap.add_argument("--sh-degree-interval", type=int, default=20)
    ap.add_argument("--no-fused-losses", action="store_true", help="b200 backend: keep the package's torch SSIM")
    ap.add_argument("--fused-ssim-only", action="store_true", help="reference backend + ONLY the fused SSIM of gsplat_b200 (isolates the loss)")
    ap.add_argument("--breakdown", action="store_true", help="CUDA-event phase times of a few steady steps (after the run)")
    ap.add_argument("--warm", type=int, default=20, help="untimed first steps (allocator / cuDNN autotune / lazy init)")
    ap.add_argument("--grad-stats", action="store_true", help="default strategy: print quantiles of the densification statistic")
    ap.add_argument("--with-ut", action="store_true",
                    help="train 3DGUT: rasterization(with_ut=True, with_eval3d=True), MCMC only (as in the reference)")
    args = ap.parse_args()
    if args.with_ut and args.strategy != "mcmc":
        ap.error("--with-ut trains with the MCMC strategy only (the reference densifies 3DGUT with MCMC alone)")

    from oracle import refcuda
    from tests import scene

    assert torch.cuda.is_available()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    if not refcuda.package_available():
        # the reference package (baseline/_ref) drives both backends: strategies, losses and the ground truth
        print(json.dumps({"tool": "trainer_bench", "backend": args.backend, "strategy": args.strategy,
                          "with_ut": args.with_ut, "not_run": "the reference package is not installed in baseline/_ref"}))
        return
    gsplat = refcuda.import_package()
    from gsplat.strategy import DefaultStrategy, MCMCStrategy
    import gsplat.losses as glosses

    torch.manual_seed(42)
    np.random.seed(42)
    sc = scene.make_scene(scene_grid=3, sh_degree=3)
    N0 = sc["means"].shape[0]
    t = lambda a: torch.from_numpy(a).to(dev)  # noqa: E731
    camtoworlds_all, Ks_all = make_cameras(sc, args.views, dev)

    # ---- ground-truth renders with the reference's stock path (same pixels for both backends)
    with torch.no_grad():
        gt = []
        for v in range(args.views):
            rc, _, _ = gsplat.rasterization(
                t(sc["means"]), t(sc["quats"]), t(sc["scales"]) * args.gt_scale, t(sc["opacities"]), t(sc["sh"]),
                torch.linalg.inv(camtoworlds_all[v : v + 1]), Ks_all[v : v + 1], W_IMG, H_IMG, sh_degree=3, packed=False,
            )
            gt.append(rc[0].clamp(0, 1).cpu())
        pixels_host = torch.stack(gt).pin_memory()  # [V, H, W, 3] float32, as the DataLoader delivers (pin_memory=True)
        c2w_host, Ks_host = camtoworlds_all.cpu().pin_memory(), Ks_all.cpu().pin_memory()
    torch.cuda.empty_cache()

    applied = None
    if args.backend == "b200":
        from gsplat_b200 import dropin

        applied = dropin.apply(losses=not args.no_fused_losses)
    elif args.fused_ssim_only:
        from gsplat_b200 import dropin

        applied = dropin.apply(losses=True, ops=False)
    rasterization = gsplat.rendering.rasterization

    # ---- trainable splats, trainer-style init (simple_trainer.py:292-349) from perturbed ground truth
    mcmc = args.strategy == "mcmc"
    g = torch.Generator(device="cpu").manual_seed(7)
    means0 = t(sc["means"]) + (torch.randn((N0, 3), generator=g) * 0.005).to(dev)
    scales0 = torch.log(t(sc["scales"]) * args.gt_scale * (0.5 if mcmc else 0.8))
    quats0 = torch.rand((N0, 4), generator=g).to(dev)
    opac0 = torch.logit(torch.full((N0,), 0.5 if mcmc else 0.1, device=dev))
    sh_all = t(sc["sh"])
    sh00 = (sh_all[:, :1, :] * 0.7).contiguous()
    shN0 = torch.zeros((N0, 15, 3), device=dev)
    lrs = dict(means=1.6e-4, scales=5e-3, quats=1e-3, opacities=5e-2, sh0=2.5e-3, shN=2.5e-3 / 20)
    splats = torch.nn.ParameterDict(
        {k: torch.nn.Parameter(v) for k, v in dict(means=means0, scales=scales0, quats=quats0, opacities=opac0, sh0=sh00, shN=shN0).items()}
    ).to(dev)
    BS = 1
    optimizers = {
        name: torch.optim.Adam(
            [{"params": splats[name], "lr": lr * math.sqrt(BS), "name": name}], eps=1e-15 / math.sqrt(BS),
            betas=(1 - BS * (1 - 0.9), 1 - BS * (1 - 0.999)), fused=True,
        )
        for name, lr in lrs.items()
    }
    max_steps = 30_000
    scheduler = torch.optim.lr_scheduler.ExponentialLR(optimizers["means"], gamma=0.01 ** (1.0 / max_steps))

    if mcmc:
        strategy = MCMCStrategy(cap_max=args.cap, refine_start_iter=args.refine_start, refine_every=args.refine_every, verbose=False)
        strategy.check_sanity(splats, optimizers)
        state = strategy.initialize_state()
        opacity_reg, scale_reg = 0.01, 0.01
    else:
        strategy = DefaultStrategy(
            refine_start_iter=args.refine_start, refine_every=args.refine_every, grow_grad2d=args.grow_grad2d, verbose=False,
            reset_every=3000,
        )
        strategy.check_sanity(splats, optimizers)
        state = strategy.initialize_state(scene_scale=1.0)
        opacity_reg, scale_reg = 0.0, 0.0
    ssim_lambda = 0.2

    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731

    def train_step(step: int, marks=None):
        v = step % args.views
        camtoworlds = c2w_host[v : v + 1].to(dev, non_blocking=True)
        Ks = Ks_host[v : v + 1].to(dev, non_blocking=True)
        pixels = pixels_host[v : v + 1].to(dev, non_blocking=True)
        sh_degree_to_use = min(step // args.sh_degree_interval, 3)
        if marks is not None:
            marks["start"].record()
        means, quats = splats["means"], splats["quats"]
        scales = torch.exp(splats["scales"])
        opacities = torch.sigmoid(splats["opacities"])
        colors = torch.cat([splats["sh0"], splats["shN"]], 1)
        renders, alphas, info = rasterization(
            means=means, quats=quats, scales=scales, opacities=opacities, colors=colors,
            viewmats=torch.linalg.inv_ex(camtoworlds).inverse, Ks=Ks, width=W_IMG, height=H_IMG, packed=False,
            absgrad=(strategy.absgrad if isinstance(strategy, DefaultStrategy) else False), sparse_grad=False,
            rasterize_mode="classic", distributed=False, camera_model="pinhole", with_ut=args.with_ut, with_eval3d=args.with_ut,
            sh_degree=sh_degree_to_use, near_plane=0.01, far_plane=1e10, render_mode="RGB",
        )
        colors_r = renders
        if marks is not None:
            marks["fwd"].record()
        if isinstance(strategy, DefaultStrategy):
            strategy.step_pre_backward(params=splats, optimizers=optimizers, state=state, step=step, info=info)
        l1loss = glosses.l1_loss(colors_r, pixels).mean()
        ssimloss = glosses.ssim_loss(colors_r.permute(0, 3, 1, 2), pixels.permute(0, 3, 1, 2))
        loss = torch.lerp(l1loss, ssimloss, ssim_lambda)
        if opacity_reg > 0.0:
            loss = loss + opacity_reg * glosses.opacity_reg_loss(splats["opacities"])
        if scale_reg > 0.0:
            loss = loss + scale_reg * glosses.scale_reg_loss(splats["scales"])
        if marks is not None:
            marks["loss"].record()
        loss.backward()
        if marks is not None:
            marks["bwd"].record()
        loss_val = loss.item()  # the trainer formats it into the progress bar every step (:1003)
        for opt in optimizers.values():
            opt.step()
            opt.zero_grad(set_to_none=True)
        scheduler.step()
        if marks is not None:
            marks["opt"].record()
        if isinstance(strategy, DefaultStrategy):
            if len(splats["means"]) > args.cap:
                strategy.refine_stop_iter = min(strategy.refine_stop_iter, step)  # cfg5 stops growing at the cap
            strategy.step_post_backward(params=splats, optimizers=optimizers, state=state, step=step, info=info, packed=False)
        else:
            strategy.step_post_backward(
                params=splats, optimizers=optimizers, state=state, step=step, info=info, lr=scheduler.get_last_lr()[0]
            )
        if marks is not None:
            marks["post"].record()
        return loss_val, info

    # ---- run
    n_hist, loss_hist, grad_stats = [], [], None
    t0 = t_first_refine = None
    steps_1m = 0
    for step in range(args.steps):
        if step == args.warm:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
        n_before = len(splats["means"])
        if n_before != N0 and t_first_refine is None and t0 is not None:
            torch.cuda.synchronize()
            t_first_refine, steps_1m = time.perf_counter(), step - args.warm
        if args.grad_stats and not mcmc and grad_stats is None and step == args.refine_start and state.get("grad2d") is not None:
            gstat = (state["grad2d"] / state["count"].clamp_min(1))[state["count"] > 0]
            qs = torch.tensor([0.5, 0.8, 0.9, 0.95, 0.98, 0.99], device=gstat.device)
            grad_stats = {"quantiles": dict(zip(qs.tolist(), torch.quantile(gstat[:: max(1, gstat.numel() // 1_000_000)], qs).tolist())),
                          "n_seen": int(gstat.numel())}
        loss_val, info = train_step(step)
        if step % 25 == 0 or step == args.steps - 1:
            n_hist.append((step, len(splats["means"])))
            loss_hist.append((step, round(loss_val, 5)))
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    timed_steps = args.steps - args.warm
    if t_first_refine is None:
        t_first_refine, steps_1m = t1, timed_steps

    out = {
        "tool": "trainer_bench", "backend": args.backend, "strategy": args.strategy, "with_ut": args.with_ut, "steps": args.steps,
        "it_per_s_total": timed_steps / (t1 - t0),
        "steps_at_1M": steps_1m,
        "it_per_s_at_1M": (steps_1m / (t_first_refine - t0)) if steps_1m > 0 else None,
        "ms_per_step_total": (t1 - t0) / timed_steps * 1e3,
        "untimed_warm_steps": args.warm, "grad_stats": grad_stats,
        "n_gaussians_start": N0, "n_gaussians_end": len(splats["means"]), "n_hist": n_hist, "loss_hist": loss_hist,
        "n_isects_last": int(info["flatten_ids"].numel()) if info.get("flatten_ids") is not None else None,
        "path": "gsplat.rasterization() (stock: torch.ops.gsplat.rasterization_3dgs)" if args.backend == "reference"
        else "gsplat.rasterization() after gsplat_b200.dropin.apply()",
        "dropin": applied,
        "schedule": {"refine_start": args.refine_start, "refine_every": args.refine_every, "cap": args.cap,
                     "grow_grad2d": args.grow_grad2d, "views": args.views, "gt_scale": args.gt_scale},
        "max_mem_gb": torch.cuda.max_memory_allocated() / 2**30,
        "device": torch.cuda.get_device_name(0),
        "power_limit": subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                                      text=True).stdout.strip(),
    }
    if args.breakdown:
        # freeze the structure (no refinement) and time the phases of 10 steady steps with CUDA events
        strategy.refine_start_iter = 10**9  # keeps the per-step bookkeeping (DefaultStrategy._update_state, MCMC noise)
        acc = {k: 0.0 for k in ("fwd", "loss", "bwd", "opt", "post")}
        reps = 10
        for i in range(3 + reps):
            marks = {k: ev() for k in ("start", "fwd", "loss", "bwd", "opt", "post")}
            train_step(args.steps + i, marks)
            torch.cuda.synchronize()
            if i >= 3:
                order = ["start", "fwd", "loss", "bwd", "opt", "post"]
                for a, b in zip(order[:-1], order[1:]):
                    acc[b] += marks[a].elapsed_time(marks[b])
        out["breakdown_ms"] = {k: v / reps for k, v in acc.items()}
        out["breakdown_ms"]["sum"] = sum(out["breakdown_ms"].values())
        out["breakdown_n_gaussians"] = len(splats["means"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
