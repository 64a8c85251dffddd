#!/usr/bin/env python
"""Installs the UNMODIFIED reference (nerfstudio-project/gsplat v1.6.0) into baseline/_ref/ so that
``import gsplat`` there runs the reference's own Python package on its own CUDA kernels through its stock
path (gsplat.rasterization() -> torch.ops.gsplat.rasterization_3dgs, csrc/Rendering.cpp:745-1481, with the
reference's registered autograd).  Test / bench infrastructure only; gsplat_b200 never imports it.

    python baseline/install_ref.py [--force]

What it does (only where /root/reference exists, i.e. in the build container; the GPU box receives the
result because baseline/_ref is git-ignored but NOT gpurun-ignored):

 1. ``BUILD_NO_CUDA=1 pip install --no-index --no-build-isolation --no-deps --target baseline/_ref <copy>``
    from a scratch copy under /tmp (the source tree is read-only and setuptools writes egg-info in place).
    BUILD_NO_CUDA=1 is the reference's own switch (setup.py:40) for a Python-only install.
 2. compiles the reference's CUDA sources where they lie with the committed recipe oracle/build_ref.py
    (--full: 3DGS + 3DGUT + adam + relocation + camera wrappers, channels 1,3,4,6,8,21,23,24,32,128 as in the reference's pytest.ini, sm_90a, the reference's release
    flags; about 25 minutes from scratch on 8 cores, seconds when oracle/_ref/obj_full is warm) and places the result as the
    prebuilt module the package looks for first: ``gsplat/csrc.so`` (gsplat/cuda/_backend.py:30).
 3. copies what the reference's own hot-path tests need at run time: tests/ + the root conftest.py (the
    reference's GPU-CI XFAIL list) -> baseline/_ref/reference_suite/ (a rootdir of its own: the tests import each
    other as ``tests.*``), assets/test_garden.npz -> baseline/_ref/assets/ and reference_suite/assets/
    (gsplat/_helper.py:61 and tests/test_basic.py:99 resolve it relative to the package / the test file).
 4. writes baseline/_ref/nerfacc/__init__.py: the two nerfacc>=0.5.3 functions the reference's torch
    compositing twin calls (_torch_impl.py:763-766).  nerfacc is a dev dependency that is neither vendored
    nor installed here; the published algorithm (exclusive transmittance product, segment sum) is restated.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DST = os.path.join(HERE, "_ref")

NERFACC_SHIM = '''"""Minimal stand-in for the nerfacc (>=0.5.3) functions gsplat's torch compositing twins use
(gsplat/cuda/_torch_impl.py:763-766, _torch_impl_eval3d.py:418-469).  Written for the reference's own tests; not part of gsplat_b200."""
import torch


def pack_info(ray_indices, n_rays=None):
    """[n_rays, 2] = (first sample, sample count) of every ray; ray_indices sorted (nerfacc.pack_info)."""
    if n_rays is None:
        n_rays = int(ray_indices.max().item()) + 1 if ray_indices.numel() else 0
    counts = torch.bincount(ray_indices, minlength=n_rays)
    starts = torch.cumsum(counts, 0) - counts
    return torch.stack([starts, counts], dim=-1)


def render_weight_from_alpha(alphas, packed_info=None, ray_indices=None, n_rays=None, **_):
    """w_i = alpha_i * prod_{j<i, same ray} (1 - alpha_j); samples of a ray are contiguous and ordered.
    Returns (weights, transmittance) like nerfacc.render_weight_from_alpha (prefix='exclusive')."""
    if alphas.numel() == 0:
        return alphas, alphas
    if ray_indices is None:
        counts = packed_info[:, 1]
        ray_indices = torch.repeat_interleave(torch.arange(counts.numel(), device=alphas.device), counts)
    logt = torch.log1p(-alphas.double())  # float64 prefix sums; autograd flows through the casts
    csum = torch.cumsum(logt, 0) - logt  # exclusive
    first = torch.ones_like(ray_indices, dtype=torch.bool)
    first[1:] = ray_indices[1:] != ray_indices[:-1]
    seg = torch.cumsum(first.long(), 0) - 1
    start = csum[first][seg]
    trans = torch.exp(csum - start).to(alphas.dtype)
    return alphas * trans, trans


def accumulate_along_rays(weights, values=None, ray_indices=None, n_rays=None):
    src = weights[..., None] if values is None else weights[..., None] * values
    out = torch.zeros((n_rays, src.shape[-1]), device=src.device, dtype=src.dtype)
    out.index_add_(0, ray_indices, src)
    return out
'''


def main() -> int:
    if not os.path.isdir(REF):
        print("install_ref: /root/reference not present -- nothing to do (the GPU box uses the shipped baseline/_ref)")
        return 0
    force = "--force" in sys.argv
    pkg = os.path.join(DST, "gsplat")
    if force and os.path.isdir(DST):
        shutil.rmtree(DST)
    if not os.path.isdir(pkg):
        tmp = "/tmp/gsplat_ref_copy"
        shutil.rmtree(tmp, ignore_errors=True)
        shutil.copytree(
            REF, tmp, symlinks=True,
            ignore=shutil.ignore_patterns("docs", "third_party", ".git", "__pycache__"),
        )
        env = dict(os.environ, BUILD_NO_CUDA="1")
        cmd = [sys.executable, "-m", "pip", "install", "--no-index", "--no-build-isolation", "--no-deps",
               "--find-links", "/opt/wheelhouse", "--target", DST, tmp]
        r = subprocess.run(cmd, env=env, capture_output=True, text=True)
        print(r.stdout[-1500:])
        if r.returncode != 0:
            print(r.stderr[-3000:])
            return 1
        shutil.rmtree(tmp, ignore_errors=True)
    # 2. the CUDA extension, as the prebuilt module gsplat.csrc
    r = subprocess.run([sys.executable, os.path.join(ROOT, "oracle", "build_ref.py"), "--full"])
    if r.returncode != 0:
        return r.returncode
    so = os.path.join(ROOT, "oracle", "_ref", "gsplat_ref.so")
    dst_so = os.path.join(pkg, "csrc.so")
    if not os.path.exists(dst_so) or os.path.getmtime(dst_so) < os.path.getmtime(so):
        shutil.copy2(so, dst_so)
    # 3. tests + asset
    suite = os.path.join(DST, "reference_suite")
    if not os.path.isdir(os.path.join(suite, "tests")):
        shutil.copytree(os.path.join(REF, "tests"), os.path.join(suite, "tests"), ignore=shutil.ignore_patterns("__pycache__"))
        shutil.copy2(os.path.join(REF, "conftest.py"), os.path.join(suite, "conftest.py"))
        with open(os.path.join(suite, "pytest.ini"), "w") as f:
            # the reference's pytest.ini minus the plugins that are not installed here (pytest_check, pytest-env)
            f.write("[pytest]\ntestpaths = tests\npythonpath = .\nmarkers =\n    gradcheck: numerical autograd gradcheck\n")
    for d in (os.path.join(DST, "assets"), os.path.join(suite, "assets")):
        os.makedirs(d, exist_ok=True)
        shutil.copy2(os.path.join(REF, "assets", "test_garden.npz"), os.path.join(d, "test_garden.npz"))
    # 4. nerfacc stand-in
    os.makedirs(os.path.join(DST, "nerfacc"), exist_ok=True)
    with open(os.path.join(DST, "nerfacc", "__init__.py"), "w") as f:
        f.write(NERFACC_SHIM)
    print("install_ref: baseline/_ref ready:", sorted(os.listdir(DST)))
    return 0


if __name__ == "__main__":
    sys.exit(main())
