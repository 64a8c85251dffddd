"""CPU-side checks of the drop-in boundary: the C-ABI library loads, the binding in gsplat_b200/_cabi.py reads every
prototype of include/gsplat_b200.h with the right ctypes and the library exports each one, and the product path
refuses to run without a GPU (no CPU fallback)."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
HEADER = os.path.join(ROOT, "include", "gsplat_b200.h")

I64, U32, INT, F32, SZ, VP = (
    ctypes.c_int64, ctypes.c_uint32, ctypes.c_int, ctypes.c_float, ctypes.c_size_t, ctypes.c_void_p
)


def test_library_exports_every_declared_symbol():
    from gsplat_b200 import _cabi

    assert len(_cabi.EXPORTED_SYMBOLS) >= 80
    L = _cabi.lib()
    for name in _cabi.EXPORTED_SYMBOLS:
        assert hasattr(L, name), f"{name} not exported by libgsplat_b200.so"


def test_every_prototype_is_bound():
    """A prototype the parser misses would still be callable through ctypes, with int conversions that truncate
    pointers; so every gsb200_* name followed by '(' in the header, found without the parser's pattern, is bound."""
    from gsplat_b200 import _cabi

    assert os.path.samefile(_cabi.HEADER_PATH, HEADER)
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    declared = set(re.findall(r"\b(gsb200_\w+)\s*\(", src))
    assert declared == set(_cabi.EXPORTED_SYMBOLS), declared ^ set(_cabi.EXPORTED_SYMBOLS)


def test_ctypes_of_every_c_spelling():
    """Known answers covering every return and parameter type the header spells."""
    from gsplat_b200 import _cabi

    expected = {
        "gsb200_version": (ctypes.c_char_p, []),
        "gsb200_error_string": (ctypes.c_char_p, [INT]),
        "gsb200_bits_for_count": (U32, [I64]),
        "gsb200_raster_records_bytes": (SZ, [I64, INT, I64]),
        "gsb200_publish_totals": (INT, [VP, VP, I64, VP]),
        "gsb200_quat_scale_to_covar_preci_fwd": (INT, [I64, VP, VP, INT, VP, VP, VP]),
        "gsb200_projection_fwd": (INT, [I64] * 3 + [VP] * 7 + [U32] * 2 + [F32] * 4 + [INT] + [VP] * 6),
        "gsb200_isect_count_totals": (INT, [I64] * 2 + [VP] * 6 + [U32] * 3 + [VP] * 3),
        "gsb200_sparse_layout_finish": (INT, [I64, I64, U32, U32, I64, VP, SZ] + [VP] * 6),
        "gsb200_raster_sparse_fwd": (INT, [INT] + [VP] * 6 + [U32] * 5 + [I64] + [VP] * 3 + [I64] + [VP] * 8),
        "gsb200_project_sh_bwd": (
            INT, [I64] * 3 + [INT] + [VP] * 6 + [U32] * 2 + [F32] + [VP] * 5 + [I64, VP] * 3 + [I64] + [VP] * 7,
        ),
        "gsb200_eval3d_fwd": (
            INT, [I64] * 3 + [INT] + [VP] * 9 + [INT] + [VP] * 5 + [INT] + [U32] * 5 + [VP] * 2 + [I64] + [VP] * 4,
        ),
        "gsb200_nvls_allreduce_f32": (INT, [VP, I64, INT, INT, VP, I64, INT, VP]),
    }
    for name, sig in expected.items():
        assert _cabi._SIGNATURES[name] == sig, name


def test_functions_are_bound_as_parsed():
    from gsplat_b200 import _cabi

    L = _cabi.lib()
    for name, (res, args) in _cabi._SIGNATURES.items():
        fn = getattr(L, name)
        assert fn.restype is res and list(fn.argtypes) == args, name


def test_parse_header_refuses_unmapped_types():
    from gsplat_b200._cabi import GsplatB200Error, _parse_header

    for ctype in ("double", "uint16_t"):
        with pytest.raises(GsplatB200Error, match=rf"gsb200_f: parameter `{ctype} scale`"):
            _parse_header(f"int gsb200_f(int64_t n, {ctype} scale, void *stream);")
    with pytest.raises(GsplatB200Error, match="gsb200_g: return type `double`"):
        _parse_header("double gsb200_g(void);")


def test_parse_header_prototype_forms():
    from gsplat_b200._cabi import _parse_header

    text = """
    /* int gsb200_commented_out(int x); */
    const char *gsb200_a(void);
    size_t
    gsb200_b(
        int64_t n, const float *x,  /* comment */
        void *const *pads, float eps
    );
    """
    assert _parse_header(text) == {"gsb200_a": (ctypes.c_char_p, []), "gsb200_b": (SZ, [I64, VP, VP, F32])}


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
