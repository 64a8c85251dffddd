"""One place that decides HOW the real reference's CUDA operators get into a process (test / bench
infrastructure only; gsplat_b200 never imports this).

Two physical copies of the same build exist (oracle/build_ref.py, baseline/install_ref.py):
``baseline/_ref/gsplat/csrc.so`` (the prebuilt module the reference's Python package imports) and
``oracle/_ref/gsplat_ref.so``.  Each runs TORCH_LIBRARY(gsplat) when loaded, so a process must load exactly
one of them: the package's copy whenever the package is installed (then ``import gsplat`` later in the same
process finds the library already open), the bare copy otherwise.
"""
from __future__ import annotations

import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG_DIR = os.path.join(ROOT, "baseline", "_ref")
PKG_SO = os.path.join(PKG_DIR, "gsplat", "csrc.so")
BARE_SO = os.path.join(ROOT, "oracle", "_ref", "gsplat_ref.so")

_loaded = None


def available() -> bool:
    return os.path.exists(PKG_SO) or os.path.exists(BARE_SO)


def package_available() -> bool:
    return os.path.exists(PKG_SO) and os.path.exists(os.path.join(PKG_DIR, "gsplat", "__init__.py"))


def load_ops():
    """torch.ops.gsplat.* of the reference build (no Python package import).  Returns torch.ops.gsplat."""
    global _loaded
    import torch

    if _loaded is None:
        so = PKG_SO if os.path.exists(PKG_SO) else BARE_SO
        if not os.path.exists(so):
            raise FileNotFoundError("reference CUDA build missing: run python oracle/build_ref.py where the reference sources are")
        torch.ops.load_library(so)
        _loaded = so
    return torch.ops.gsplat


def import_package():
    """``import gsplat`` = the unmodified reference package from baseline/_ref (stock path).  The nerfacc
    stand-in written by baseline/install_ref.py sits next to it."""
    if not package_available():
        raise FileNotFoundError("reference package not installed in baseline/_ref (python baseline/install_ref.py, where the reference sources are)")
    load_ops()
    if PKG_DIR not in sys.path:
        sys.path.insert(0, PKG_DIR)
    import gsplat

    if not os.path.abspath(gsplat.__file__).startswith(PKG_DIR):
        raise RuntimeError(f"'gsplat' resolved to {gsplat.__file__}, expected the copy under {PKG_DIR}")
    return gsplat
