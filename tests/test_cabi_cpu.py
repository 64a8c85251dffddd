"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol that
include/gsplat_b200.h declares, the ctypes signatures in gsplat_b200/_cabi.py agree with the header
parameter by parameter, and the product path refuses to run without a GPU (no CPU fallback)."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


def _header_functions():
    src = open(os.path.join(ROOT, "include", "gsplat_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    out = {}
    for m in re.finditer(r"\n\s*((?:const\s+)?[A-Za-z_0-9]+\s*\*?)\s*(gsb200_[a-z_0-9]+)\s*\((.*?)\)\s*;", src, flags=re.S):
        ret, name, params = m.group(1).strip(), m.group(2), m.group(3).strip()
        plist = [] if params in ("", "void") else [p.strip() for p in params.split(",")]
        out[name] = (ret, plist)
    return out


def _ctype_of(decl: str):
    from gsplat_b200 import _cabi as c

    if "*" in decl:
        return ctypes.c_char_p if decl.startswith("const char") and "(" in decl else c.c_vp
    base = decl.replace("const", "").split()[0]
    return {"int64_t": c.c_i64, "uint32_t": c.c_u32, "int": c.c_int, "float": c.c_f32, "size_t": c.c_sz}[base]


def test_library_exports_every_declared_symbol():
    from gsplat_b200 import _cabi

    funcs = _header_functions()
    assert len(funcs) >= 20
    assert set(funcs) == set(_cabi.EXPORTED_SYMBOLS), set(funcs) ^ set(_cabi.EXPORTED_SYMBOLS)
    L = _cabi.lib()
    for name in funcs:
        assert hasattr(L, name), f"{name} not exported by libgsplat_b200.so"


def test_ctypes_signatures_match_header():
    from gsplat_b200 import _cabi

    funcs = _header_functions()
    for name, (ret, params) in funcs.items():
        res, args = _cabi._SIGNATURES[name]
        assert len(args) == len(params), f"{name}: header has {len(params)} params, binding has {len(args)}"
        for i, (p, a) in enumerate(zip(params, args)):
            assert _ctype_of(p) is a, f"{name} arg {i} ({p}): binding uses {a}"
        if ret.startswith("const char"):
            assert res is ctypes.c_char_p
        else:
            assert res is _ctype_of(ret + " x")


def test_host_only_entry_points():
    from gsplat_b200 import _cabi

    L = _cabi.lib()
    assert b"sm_90a" in L.gsb200_version()


def test_shipped_binary_matches_the_sources():
    """The built library travels with the tree as a binary (git-ignored): it carries the sha256 of the sources it was
    compiled from, which must be the hash of the sources in this tree."""
    from gsplat_b200 import _cabi, build

    L = _cabi.lib()
    assert L.gsb200_source_hash().decode() == build.source_hash()
    # bits_for_count known answers: /root/reference/tests/cpp/test_mathutils.cpp:53-63
    for count, bits in [(0, 0), (1, 0), (2, 1), (3, 2), (4, 2), (5, 3), (7, 3), (8, 3), (9, 4), (8160, 13)]:
        assert _cabi.bits_for_count(count) == bits
    assert L.gsb200_raster_supports_channels(3) == 1 and L.gsb200_raster_supports_channels(6) == 0
    assert L.gsb200_raster_records_bytes(1000, 3, 64) >= 1000 * 48
    assert L.gsb200_error_string(-5).startswith(b"intersect_tile")


def test_raster_bwd_checks_gradient_records():
    """Both compositing backwards check the gradient records before anything is launched: a null or non-16-byte-aligned
    base is GSB200_E_INVALID, rows * row width of 2^32 floats or more is GSB200_E_UNSUPPORTED (the kernel addresses a
    row with a 32-bit element offset)."""
    from gsplat_b200 import _cabi

    L = _cabi.lib()
    fake = 1 << 20  # never dereferenced: every call below returns before the kernel is launched

    def dense(N, rec, absgrad=0):
        return L.gsb200_raster_bwd(
            1, N, 3, None, None, 16, 16, 16, 1, 1, fake, fake, 1, fake, fake, fake, fake, None, absgrad, rec, None
        )

    def sparse(n_rows, rec, absgrad=0):
        return L.gsb200_raster_sparse_bwd(
            n_rows, 3, None, None, 16, 16, 16, 1, 1, 1, fake, fake, fake, 1, fake, fake, fake, fake, fake, fake, fake, None,
            absgrad, rec, None,
        )

    too_many = (1 << 32) // 12 + 1  # D = 3 with absgrad: 12-float rows
    for call in (dense, sparse):
        assert call(4, None) == -1
        assert call(4, fake + 4) == -1
        assert call(too_many, fake, absgrad=1) == -2


def test_no_cpu_fallback():
    import gsplat_b200
    from gsplat_b200._cabi import GsplatB200Error

    z = torch.zeros
    with pytest.raises(GsplatB200Error):
        gsplat_b200.rasterization(z(4, 3), z(4, 4), z(4, 3), z(4), z(4, 3), torch.eye(4)[None], torch.eye(3)[None], 32, 32, packed=False)
    with pytest.raises(GsplatB200Error):
        gsplat_b200.quat_scale_to_covar_preci(z(4, 4), z(4, 3))
    with pytest.raises(GsplatB200Error):
        gsplat_b200.isect_tiles(z(1, 4, 2), z(1, 4, 2, dtype=torch.int32), z(1, 4), 16, 2, 2)


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "gsplat_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in text and "from oracle" not in text and "libgs_oracle" not in text, f


def test_argument_validation_is_reference_like():
    import gsplat_b200

    z = torch.zeros
    with pytest.raises(ValueError):
        gsplat_b200.rasterization(z(4, 3), z(4, 4), z(4, 3), z(5), z(4, 3), torch.eye(4)[None], torch.eye(3)[None], 32, 32)
    with pytest.raises(NotImplementedError):
        gsplat_b200.rasterization(z(4, 3), z(4, 4), z(4, 3), z(4), z(4, 3), torch.eye(4)[None], torch.eye(3)[None], 32, 32, with_ut=True)
    with pytest.raises(ValueError):
        gsplat_b200.rasterization(z(4, 3), z(4, 4), z(4, 3), z(4), z(4, 3), torch.eye(4)[None], torch.eye(3)[None], 32, 32, tile_size=8)
    with pytest.raises(ValueError):
        gsplat_b200.spherical_harmonics(3, z(4, 3), torch.eye(4)[None], z(4, 9, 3))


def test_rasterization_argument_validation_on_cpu():
    """Flags outside the path raise before any kernel is touched (reference: ValueError / NotImplementedError from the
    renderer-config checks, rendering.py:526-600); everything else fails loudly on non-CUDA tensors."""
    import pytest
    import torch

    import gsplat_b200 as gs
    from gsplat_b200._cabi import GsplatB200Error

    N = 10
    args = (torch.rand(N, 3), torch.rand(N, 4), torch.rand(N, 3), torch.rand(N), torch.rand(N, 3), torch.eye(4)[None],
            torch.eye(3)[None], 64, 64)
    for kw in (dict(with_ut=True), dict(with_eval3d=True), dict(camera_model="ftheta"), dict(camera_model="lidar"),
               dict(return_normals=True)):
        with pytest.raises(NotImplementedError):
            gs.rasterization(*args, **kw)
    for kw in (dict(render_mode="bogus"), dict(tile_size=8), dict(rasterize_mode="soft"), dict(sparse_grad=True, packed=False),
               dict(distributed=True)):
        with pytest.raises(ValueError):
            gs.rasterization(*args, **kw)
    with pytest.raises(ValueError):  # SH degree needs K >= (deg + 1)^2
        gs.rasterization(*args[:4], torch.rand(N, 4, 3), *args[5:], sh_degree=2)
    with pytest.raises(GsplatB200Error):
        gs.rasterization(*args)
