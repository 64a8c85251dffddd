"""Checks that a change leaves the existing kernels' machine code alone.

    python tools/sass_compare.py [--base REV] [--units raster.cu isect.cu ...]

Compiles the units (default: every unit of gsplat_b200/build.py) for sm_90a with the flags of build.py -- those that
exist at git revision ``--base`` (default HEAD) from the sources at that revision, all of them from the working tree --
disassembles the objects with ``cuobjdump -sass`` and compares every kernel of the base objects with the kernel of the
same name in the new ones, whichever unit it is compiled in: a kernel that moved to another file is matched with its
old self.  Names are compared demangled, with the pixel-addressing policy of the compositing kernels
(``gsb::DensePixels``) removed, so that a kernel that only gained that template argument is matched with its old self,
with ``isect_count_kernel<true / false>`` under the names the two count kernels had before they became one template,
with the unmasked ``isect_count_kernel`` and ``isect_emit_kernel`` (``MASKED`` = false) without that template argument
and the tile-mask parameters that came with it, and with the pair-query kernels ``raster_indices_kernel``,
``surfel_indices_kernel`` and ``eval3d_indices_kernel`` named by their template arguments without their parameter list
(``<false / true>`` became the ``CountSink`` / ``PairSink`` instantiations when each walk took a sink; the 2DGS and
3DGUT walks became ``pair_walk_kernel<SurfelModel, Sink, Pix>`` and ``pair_walk_kernel<Eval3dModel<Shutter, Lens>,
Sink, Pix>``, named as the kernels they were, so that they are reported as changed), and with the 3DGUT kernels
(``ut_project_kernel``, ``eval3d_fwd_kernel``, ``eval3d_bwd_kernel``) without their ``gsb::GlobalShutter`` policy, the
template argument and the trailing empty parameter they gained with the rolling shutter, and without their
``gsb::CamLens`` policy, the template argument and trailing empty parameter they gained with the FTheta lens.  Instructions and their encodings must be
identical; address and line-info comments are ignored.  A library kernel (CUB) that several units instantiate must be
identical in all of them.  Kernels that only the new objects have are listed as new.  Exit status 1 on any difference.  Needs nvcc / cuobjdump / cu++filt (no GPU).
"""
from __future__ import annotations

import argparse
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)

from gsplat_b200 import build as B  # noqa: E402

CUDA_BIN = os.path.dirname(B._nvcc()) if os.path.isabs(B._nvcc()) else "/usr/local/cuda/bin"
# cu++filt prints the policy parameter of a kernel as `T<k>`: dropped together with the policy template argument
POLICY_PARAM = re.compile(r",\s*T\d+\)$")
# isect_count_kernel<TOTALS> and isect_emit_kernel<KeyT> gained a MASKED template argument and appended parameters
# (count: N, I, image_ids, tile_mask; emit: tile_mask): <..., false> is the kernel as it was
MASKED_KERNEL = re.compile(
    r"^void (gsb::isect_(?:count|emit)_kernel)<(.*), \(bool\)0>\((.*?), (?:long, long, const long \*, )?const unsigned char \*\)$"
)
# isect_count_kernel<TOTALS>: <true> was isect_count_totals_kernel, <false> isect_count_kernel without the totals pointer
COUNT_KERNEL = re.compile(r"^void gsb::isect_count_kernel<\(bool\)([01])>\((.*), unsigned long long \*\)$")
# raster_indices_kernel<EMIT> became raster_indices_kernel<Sink, Pix> and surfel_indices_kernel<EMIT> became
# surfel_indices_kernel<Sink>: <false> is the CountSink walk, <true> the PairSink
INDICES_KERNEL = re.compile(r"^void (gsb::(?:<unnamed>::)?(?:raster|surfel|eval3d)_indices_kernel)<(.*)>\(.*\)$")
INDICES_SINK = {"(bool)0": "gsb::CountSink", "(bool)1": "gsb::PairSink"}
# surfel_indices_kernel<Sink, Pix> and eval3d_indices_kernel<Sink, Shutter, Lens, Pix> became pair_walk_kernel of the
# SurfelModel / Eval3dModel<Shutter, Lens>: renamed as they were, before the policies are removed
PAIR_WALK = re.compile(
    r"^void gsb::pair_walk_kernel<gsb::<unnamed>::(?:(SurfelModel)|Eval3dModel<([^<>]*)>), (gsb::\w+), (gsb::\w+)>(\(.*\))$"
)


def _tree_at(rev: str, dst: str) -> None:
    """gsplat_b200/csrc and include/ as of `rev`, written under dst."""
    files = subprocess.check_output(["git", "-C", ROOT, "ls-tree", "-r", "--name-only", rev, "gsplat_b200/csrc", "include"], text=True)
    for rel in files.split():
        out = os.path.join(dst, rel)
        os.makedirs(os.path.dirname(out), exist_ok=True)
        with open(out, "wb") as f:
            f.write(subprocess.check_output(["git", "-C", ROOT, "show", f"{rev}:{rel}"]))


def _compile(src_root: str, unit: str, obj: str) -> None:
    cmd = [B._nvcc(), *B.ARCH, *B.COMMON, *B.UNITS[unit], "-c", os.path.join(src_root, "gsplat_b200", "csrc", unit), "-o", obj]
    subprocess.check_call(cmd, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)


def _demangle(names):
    out = subprocess.run([os.path.join(CUDA_BIN, "cu++filt")], input="\n".join(names), capture_output=True, text=True, check=True)
    return out.stdout.splitlines()


def kernels(obj: str):
    """{normalised demangled name: [instruction lines]}"""
    text = subprocess.check_output([os.path.join(CUDA_BIN, "cuobjdump"), "-sass", obj], text=True)
    raw, cur = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            raw[cur] = []
            continue
        if cur is None:
            continue
        s = line.strip()
        if not s or s.startswith("//") or s.startswith("."):
            continue
        s = re.sub(r"^/\*[0-9a-f]{4,}\*/\s*", "", s)  # instruction address
        if s:
            raw[cur].append(re.sub(r"\s+", " ", s))
    names = list(raw)
    out = {}
    for n, d in zip(names, _demangle(names)):
        m = PAIR_WALK.match(d)
        if m:  # <Sink, Pix> of the 2DGS walk, <Sink, Shutter, Lens, Pix> of the 3DGUT one
            policies = "" if m[1] else f"{m[2]}, "
            d = f"void gsb::<unnamed>::{'surfel' if m[1] else 'eval3d'}_indices_kernel<{m[3]}, {policies}{m[4]}>{m[5]}"
        if "DensePixels" in n or "SparsePixels" in n:
            d = POLICY_PARAM.sub(")", d).replace(", gsb::DensePixels>", ">")
        m = MASKED_KERNEL.match(d)
        if m:
            d = f"void {m.group(1)}<{m.group(2)}>({m.group(3)})"
        m = COUNT_KERNEL.match(d)
        if m:
            d = f"gsb::isect_count_totals_kernel({m.group(2)}, unsigned long long *)" if m.group(1) == "1" else f"gsb::isect_count_kernel({m.group(2)})"
        if "gsb::CamLens" in d:
            # the 3DGUT kernels' lens policy (template argument and last parameter): CamLens, the runtime pinhole / fisheye
            # model, is the kernel as it was before FTheta became the other policy
            d = POLICY_PARAM.sub(")", d).replace(", gsb::CamLens>", ">")
        if "gsb::GlobalShutter" in d:
            # the 3DGUT kernels' shutter policy (template argument and last parameter): GlobalShutter is the kernel as it was
            # (a kernel with no other template argument was not a template, and demangles without its return type)
            d = POLICY_PARAM.sub(")", d).replace(", gsb::GlobalShutter>", ">")
            if "<gsb::GlobalShutter>" in d:
                d = d.replace("<gsb::GlobalShutter>", "").removeprefix("void ")
        m = INDICES_KERNEL.match(d)
        if m:
            d = f"{m.group(1)}<{INDICES_SINK.get(m.group(2), m.group(2))}>"
        out[d] = raw[n]
    return out


def kernels_of(src_root: str, units, tmp: str, tag: str):
    """{name: {instruction lines of every unit that has the kernel}} over the units present under src_root"""
    out = {}
    for unit in units:
        if not os.path.exists(os.path.join(src_root, "gsplat_b200", "csrc", unit)):
            continue
        obj = os.path.join(tmp, f"{tag}_{unit}.o")
        _compile(src_root, unit, obj)
        for name, body in kernels(obj).items():
            out.setdefault(name, set()).add(tuple(body))
    return out


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", default="HEAD")
    ap.add_argument("--units", nargs="+", default=list(B.UNITS))
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        base_root = os.path.join(tmp, "base")
        _tree_at(args.base, base_root)
        kb, kn = kernels_of(base_root, args.units, tmp, "base"), kernels_of(ROOT, args.units, tmp, "new")
    same = [k for k in kb if k in kn and kb[k] == kn[k]]
    missing = [k for k in kb if k not in kn]
    changed = [k for k in kb if k in kn and kb[k] != kn[k]]
    new = [k for k in kn if k not in kb]
    n_instr = sum(len(body) for k in same for body in kb[k])
    print(f"{' '.join(args.units)}: {len(kb)} kernels at {args.base}: {len(same)} identical ({n_instr} instructions), "
          f"{len(changed)} changed, {len(missing)} missing; {len(new)} new")
    for k in changed:
        print(f"  CHANGED {k} ({sorted(len(b) for b in kb[k])} -> {sorted(len(b) for b in kn[k])} instructions)")
    for k in missing:
        print(f"  MISSING {k}")
    for k in new:
        print(f"  new     {k}")
    bad = len(changed) + len(missing)
    print("dense kernels unchanged" if bad == 0 else f"{bad} kernels differ")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
