"""The compositing entry points of the C ABI, checked on the CPU: gsb200_raster_records_bytes against sizes recorded
before the record-stream layout was written once for both the carving and the size query, and the return code of every
gsb200_raster_* entry, of the two surfel compositing entries and of the two pair-query entries (gsb200_raster_indices,
gsb200_surfel_indices) for invalid or early-return arguments, including which check fires first.  Every call here
returns before a kernel is launched or the device is touched: the pointers are fake and never read."""
import pytest

from gsplat_b200 import _cabi

OK, INVALID, UNSUPPORTED, WORKSPACE = 0, -1, -2, -4
FAKE = 1 << 20  # 16-byte aligned, never dereferenced
CHANNELS = (1, 2, 3, 4, 5, 8, 16, 32)

# gsb200_raster_records_bytes(n_isects, D, n_tiles) for D in CHANNELS
RECORDS_BYTES = {
    (0, 0): [512, 512, 512, 512, 512, 512, 512, 512],
    (0, 1): [512, 512, 512, 512, 512, 512, 512, 512],
    (0, 64): [768, 768, 768, 768, 768, 768, 768, 768],
    (0, 8160): [33024, 33024, 33024, 33024, 33024, 33024, 33024, 33024],
    (1, 0): [1536, 1536, 1536, 1536, 1536, 1536, 1536, 1536],
    (1, 1): [1536, 1536, 1536, 1536, 1536, 1536, 1536, 1536],
    (1, 64): [1792, 1792, 1792, 1792, 1792, 1792, 1792, 1792],
    (1, 8160): [34048, 34048, 34048, 34048, 34048, 34048, 34048, 34048],
    (255, 0): [16896, 16896, 16896, 16896, 20992, 20992, 29184, 45568],
    (255, 1): [16896, 16896, 16896, 16896, 20992, 20992, 29184, 45568],
    (255, 64): [17152, 17152, 17152, 17152, 21248, 21248, 29440, 45824],
    (255, 8160): [49408, 49408, 49408, 49408, 53504, 53504, 61696, 78080],
    (256, 0): [16896, 16896, 16896, 16896, 20992, 20992, 29184, 45568],
    (256, 1): [16896, 16896, 16896, 16896, 20992, 20992, 29184, 45568],
    (256, 64): [17152, 17152, 17152, 17152, 21248, 21248, 29440, 45824],
    (256, 8160): [49408, 49408, 49408, 49408, 53504, 53504, 61696, 78080],
    (10**6, 0): [64000512, 64000512, 64000512, 64000512, 80000512, 80000512, 112000512, 176000512],
    (10**6, 1): [64000512, 64000512, 64000512, 64000512, 80000512, 80000512, 112000512, 176000512],
    (10**6, 64): [64000768, 64000768, 64000768, 64000768, 80000768, 80000768, 112000768, 176000768],
    (10**6, 8160): [64033024, 64033024, 64033024, 64033024, 80033024, 80033024, 112033024, 176033024],
}

L = _cabi.lib()


def test_records_bytes_match_the_recorded_layout():
    for (n, tiles), want in RECORDS_BYTES.items():
        assert [L.gsb200_raster_records_bytes(n, D, tiles) for D in CHANNELS] == want, (n, tiles)
    for args in ((-1, 3, 1), (1, 0, 1), (1, -3, 1), (1, 3, -1)):
        assert L.gsb200_raster_records_bytes(*args) == 0, args


PARAMS = {
    "gsb200_raster_pack": "I D means2d conics colors opacities tw th offsets flatten_ids n_isects records stream",
    "gsb200_raster_fwd": "I N D means2d conics colors opacities backgrounds masks W H tile_size tw th offsets flatten_ids "
    "n_isects records render_colors render_alphas last_ids stream",
    "gsb200_raster_fwd_rows": "I N D row_records backgrounds masks W H tile_size tw th offsets flatten_ids n_isects records "
    "render_colors render_alphas last_ids stream",
    "gsb200_raster_bwd": "I N D backgrounds masks W H tile_size tw th offsets flatten_ids n_isects records render_alphas "
    "last_ids v_render_colors v_render_alphas absgrad v_grad_records stream",
    "gsb200_raster_sparse_fwd": "D means2d conics colors opacities backgrounds masks W H tile_size tw th n_active active_tiles "
    "tile_offsets flatten_ids n_isects tile_pixel_mask tile_pixel_cumsum pixel_map records render_colors render_alphas "
    "last_ids stream",
    "gsb200_raster_sparse_bwd": "n_rows D backgrounds masks W H tile_size tw th n_active active_tiles tile_offsets flatten_ids "
    "n_isects tile_pixel_mask tile_pixel_cumsum pixel_map records render_alphas last_ids v_render_colors v_render_alphas "
    "absgrad v_grad_records stream",
    "gsb200_surfel_raster_fwd": "I N D means2d ray_transforms colors opacities normals backgrounds masks W H tile_size tw th "
    "offsets flatten_ids n_isects render_colors render_alphas render_normals render_distort render_median last_ids "
    "median_ids stream",
    "gsb200_surfel_raster_bwd": "I N D means2d ray_transforms colors opacities normals backgrounds masks W H tile_size tw th "
    "offsets flatten_ids n_isects render_colors render_alphas last_ids median_ids v_render_colors v_render_alphas "
    "v_render_normals v_render_distort v_render_median v_means2d v_ray_transforms v_colors v_opacities v_normals v_densify "
    "v_means2d_abs stream",
}
# rows: conics [R, 3] for gsb200_raster_indices, ray transforms [R, 3, 3] for gsb200_surfel_indices
INDICES_PARAMS = ("I N means2d rows opacities transmittances W H tile_size tw th offsets flatten_ids n_isects range_start "
                  "range_end emit workspace workspace_bytes total gaussian_ids pixel_ids image_ids stream")
PARAMS["gsb200_raster_indices"] = PARAMS["gsb200_surfel_indices"] = INDICES_PARAMS
# a 16 x 16 image of one tile, one intersection, D = 3; every other pointer fake and 16-byte aligned
BASE = dict(I=1, N=4, D=3, W=16, H=16, tile_size=16, tw=1, th=1, n_isects=1, n_active=1, n_rows=4, absgrad=0,
            backgrounds=None, masks=None, v_render_alphas=None, stream=None,
            range_start=0, range_end=1, emit=1, workspace_bytes=1 << 62)

GRID_SMALL = dict(W=17)  # one 16-pixel tile column for a 17-pixel wide image

# (entry, arguments changed from BASE, expected code).  None of these reaches a launch.
CASES = [
    ("gsb200_raster_pack", dict(I=-1), INVALID),
    ("gsb200_raster_pack", dict(n_isects=-1), INVALID),
    ("gsb200_raster_pack", dict(offsets=None, n_isects=0), INVALID),
    ("gsb200_raster_pack", dict(n_isects=0), OK),
    ("gsb200_raster_pack", dict(I=0), OK),
    ("gsb200_raster_pack", dict(n_isects=0, D=6, means2d=None), OK),
    ("gsb200_raster_pack", dict(means2d=None), INVALID),
    ("gsb200_raster_pack", dict(records=None), INVALID),
    ("gsb200_raster_pack", dict(means2d=None, D=6), INVALID),
    ("gsb200_raster_pack", dict(D=6), UNSUPPORTED),
    ("gsb200_raster_pack", dict(D=0), UNSUPPORTED),

    ("gsb200_raster_fwd", dict(I=-1), INVALID),
    ("gsb200_raster_fwd", dict(N=-1), INVALID),
    ("gsb200_raster_fwd", dict(render_colors=None, I=0), INVALID),
    ("gsb200_raster_fwd", dict(last_ids=None), INVALID),
    ("gsb200_raster_fwd", dict(means2d=None), INVALID),
    ("gsb200_raster_fwd", dict(records=None, tile_size=8), INVALID),
    ("gsb200_raster_fwd", dict(tile_size=8), UNSUPPORTED),
    ("gsb200_raster_fwd", dict(tile_size=8, I=0), UNSUPPORTED),
    ("gsb200_raster_fwd", dict(I=0), OK),
    ("gsb200_raster_fwd", dict(I=0, D=6), OK),
    ("gsb200_raster_fwd", dict(W=0, D=6), OK),
    ("gsb200_raster_fwd", dict(H=0, means2d=None, n_isects=0), OK),
    ("gsb200_raster_fwd", dict(GRID_SMALL), INVALID),
    ("gsb200_raster_fwd", dict(GRID_SMALL, D=6), INVALID),
    ("gsb200_raster_fwd", dict(D=6), UNSUPPORTED),
    ("gsb200_raster_fwd", dict(D=0), UNSUPPORTED),

    ("gsb200_raster_fwd_rows", dict(I=-1), INVALID),
    ("gsb200_raster_fwd_rows", dict(offsets=None), INVALID),
    ("gsb200_raster_fwd_rows", dict(row_records=None), INVALID),
    ("gsb200_raster_fwd_rows", dict(row_records=FAKE + 4), INVALID),
    ("gsb200_raster_fwd_rows", dict(flatten_ids=None, D=5), INVALID),
    ("gsb200_raster_fwd_rows", dict(D=5), UNSUPPORTED),
    ("gsb200_raster_fwd_rows", dict(D=5, I=0), UNSUPPORTED),
    ("gsb200_raster_fwd_rows", dict(D=32, W=0), UNSUPPORTED),
    ("gsb200_raster_fwd_rows", dict(tile_size=8), UNSUPPORTED),
    ("gsb200_raster_fwd_rows", dict(I=0), OK),
    ("gsb200_raster_fwd_rows", dict(I=0, row_records=None, n_isects=0), OK),
    ("gsb200_raster_fwd_rows", dict(I=0, D=0), OK),
    ("gsb200_raster_fwd_rows", dict(GRID_SMALL), INVALID),
    ("gsb200_raster_fwd_rows", dict(D=0), UNSUPPORTED),

    ("gsb200_raster_bwd", dict(I=-1), INVALID),
    ("gsb200_raster_bwd", dict(N=-1), INVALID),
    ("gsb200_raster_bwd", dict(tile_size=8), UNSUPPORTED),
    ("gsb200_raster_bwd", dict(tile_size=8, n_isects=0), UNSUPPORTED),
    ("gsb200_raster_bwd", dict(n_isects=0), OK),
    ("gsb200_raster_bwd", dict(I=0), OK),
    ("gsb200_raster_bwd", dict(n_isects=0, offsets=None, D=6), OK),
    ("gsb200_raster_bwd", dict(offsets=None), INVALID),
    ("gsb200_raster_bwd", dict(v_render_colors=None), INVALID),
    ("gsb200_raster_bwd", dict(v_grad_records=None), INVALID),
    ("gsb200_raster_bwd", dict(v_grad_records=FAKE + 4), INVALID),
    ("gsb200_raster_bwd", dict(v_grad_records=None, D=6), INVALID),
    ("gsb200_raster_bwd", dict(N=1 << 31), UNSUPPORTED),
    ("gsb200_raster_bwd", dict(D=6), UNSUPPORTED),
    ("gsb200_raster_bwd", dict(D=0), UNSUPPORTED),

    ("gsb200_raster_sparse_fwd", dict(tile_size=8), UNSUPPORTED),
    ("gsb200_raster_sparse_fwd", dict(tile_size=8, n_isects=-1), UNSUPPORTED),
    ("gsb200_raster_sparse_fwd", dict(n_isects=-1), INVALID),
    ("gsb200_raster_sparse_fwd", dict(n_active=-1), INVALID),
    ("gsb200_raster_sparse_fwd", dict(n_active=1 << 31), INVALID),
    ("gsb200_raster_sparse_fwd", dict(active_tiles=None), INVALID),
    ("gsb200_raster_sparse_fwd", dict(GRID_SMALL), INVALID),
    ("gsb200_raster_sparse_fwd", dict(GRID_SMALL, n_active=0), INVALID),
    ("gsb200_raster_sparse_fwd", dict(n_active=0), OK),
    ("gsb200_raster_sparse_fwd", dict(n_active=0, D=6, active_tiles=None, records=None), OK),
    ("gsb200_raster_sparse_fwd", dict(records=None), INVALID),
    ("gsb200_raster_sparse_fwd", dict(render_colors=None, D=6), INVALID),
    ("gsb200_raster_sparse_fwd", dict(means2d=None), INVALID),
    ("gsb200_raster_sparse_fwd", dict(D=6), UNSUPPORTED),
    ("gsb200_raster_sparse_fwd", dict(D=0), UNSUPPORTED),

    ("gsb200_raster_sparse_bwd", dict(tile_size=8), UNSUPPORTED),
    ("gsb200_raster_sparse_bwd", dict(n_rows=-1), INVALID),
    ("gsb200_raster_sparse_bwd", dict(n_isects=-1), INVALID),
    ("gsb200_raster_sparse_bwd", dict(n_active=-1), INVALID),
    ("gsb200_raster_sparse_bwd", dict(pixel_map=None), INVALID),
    ("gsb200_raster_sparse_bwd", dict(GRID_SMALL), INVALID),
    ("gsb200_raster_sparse_bwd", dict(GRID_SMALL, n_isects=0), INVALID),
    ("gsb200_raster_sparse_bwd", dict(n_isects=0), OK),
    ("gsb200_raster_sparse_bwd", dict(n_active=0, D=6), OK),
    ("gsb200_raster_sparse_bwd", dict(records=None), INVALID),
    ("gsb200_raster_sparse_bwd", dict(v_grad_records=None), INVALID),
    ("gsb200_raster_sparse_bwd", dict(n_rows=1 << 31), UNSUPPORTED),
    ("gsb200_raster_sparse_bwd", dict(D=6), UNSUPPORTED),

    ("gsb200_surfel_raster_fwd", dict(I=-1), INVALID),
    ("gsb200_surfel_raster_fwd", dict(median_ids=None), INVALID),
    ("gsb200_surfel_raster_fwd", dict(normals=None), INVALID),
    ("gsb200_surfel_raster_fwd", dict(tile_size=8), UNSUPPORTED),
    ("gsb200_surfel_raster_fwd", dict(tile_size=8, I=0), UNSUPPORTED),
    ("gsb200_surfel_raster_fwd", dict(I=0), OK),
    ("gsb200_surfel_raster_fwd", dict(W=0, D=6), OK),
    ("gsb200_surfel_raster_fwd", dict(GRID_SMALL), INVALID),
    ("gsb200_surfel_raster_fwd", dict(GRID_SMALL, D=6), INVALID),
    ("gsb200_surfel_raster_fwd", dict(N=1 << 28), UNSUPPORTED),
    ("gsb200_surfel_raster_fwd", dict(D=6), UNSUPPORTED),
    ("gsb200_surfel_raster_fwd", dict(D=0), UNSUPPORTED),

    ("gsb200_surfel_raster_bwd", dict(I=-1), INVALID),
    ("gsb200_surfel_raster_bwd", dict(tile_size=8), UNSUPPORTED),
    ("gsb200_surfel_raster_bwd", dict(tile_size=8, n_isects=0), UNSUPPORTED),
    ("gsb200_surfel_raster_bwd", dict(n_isects=0), OK),
    ("gsb200_surfel_raster_bwd", dict(I=0, D=6), OK),
    ("gsb200_surfel_raster_bwd", dict(H=0), OK),
    ("gsb200_surfel_raster_bwd", dict(v_densify=None), INVALID),
    ("gsb200_surfel_raster_bwd", dict(v_densify=None, D=6), INVALID),
    ("gsb200_surfel_raster_bwd", dict(GRID_SMALL), INVALID),
    ("gsb200_surfel_raster_bwd", dict(N=1 << 28), UNSUPPORTED),
    ("gsb200_surfel_raster_bwd", dict(D=6), UNSUPPORTED),
]

# Both pair-query entries share their checks and pass sequence.  BASE is an emit pass (emit = 1) with a large enough
# workspace; the count pass (emit = 0) zeroes *total on the device when there are no pairs, so its early return is not
# called here.
INDICES_CASES = [
    (dict(I=-1), INVALID),
    (dict(N=-1), INVALID),
    (dict(n_isects=-1), INVALID),
    (dict(range_start=-1), INVALID),
    (dict(range_end=-1), INVALID),
    (dict(range_end=-1, tile_size=8), INVALID),
    (dict(tile_size=8), UNSUPPORTED),
    (dict(tile_size=8, n_isects=0), UNSUPPORTED),
    (dict(emit=0, total=None), INVALID),
    (dict(emit=0, total=None, n_isects=0), INVALID),
    (dict(emit=0, total=None, range_end=0), INVALID),
    (dict(emit=0, total=None, tile_size=8), UNSUPPORTED),
    (dict(total=None, workspace_bytes=1), WORKSPACE),
    (dict(n_isects=0), OK),
    (dict(I=0), OK),
    (dict(N=0), OK),
    (dict(W=0), OK),
    (dict(H=0, means2d=None), OK),
    (dict(range_end=0), OK),
    (dict(range_start=3, range_end=3), OK),
    (dict(range_start=5, range_end=2), OK),
    (dict(GRID_SMALL, range_end=0), OK),
    (dict(range_end=0, gaussian_ids=None), OK),
    (dict(n_isects=0, workspace=None), OK),
    (dict(means2d=None), INVALID),
    (dict(rows=None), INVALID),
    (dict(opacities=None), INVALID),
    (dict(transmittances=None), INVALID),
    (dict(offsets=None), INVALID),
    (dict(flatten_ids=None), INVALID),
    (dict(gaussian_ids=None), INVALID),
    (dict(pixel_ids=None), INVALID),
    (dict(image_ids=None), INVALID),
    (dict(emit=0, gaussian_ids=None, workspace_bytes=1), WORKSPACE),
    (dict(GRID_SMALL), INVALID),
    (dict(GRID_SMALL, workspace=None), INVALID),
    (dict(GRID_SMALL, emit=0), INVALID),
    (dict(means2d=None, workspace=None), INVALID),
    (dict(workspace=None), WORKSPACE),
    (dict(workspace_bytes=1), WORKSPACE),
    (dict(emit=0, workspace_bytes=1), WORKSPACE),
    (dict(workspace_bytes=1, n_isects=1 << 31), WORKSPACE),
    (dict(n_isects=(1 << 31) - 1, workspace_bytes=1), WORKSPACE),
    (dict(n_isects=1 << 31), UNSUPPORTED),
    (dict(emit=0, n_isects=1 << 31), UNSUPPORTED),
    (dict(I=1 << 31), UNSUPPORTED),
    (dict(emit=0, I=1 << 31), UNSUPPORTED),
]
CASES += [(entry, changes, code) for entry in ("gsb200_raster_indices", "gsb200_surfel_indices") for changes, code in INDICES_CASES]


def _call(entry, changes):
    args = dict(BASE, **changes)
    return getattr(L, entry)(*[args.get(p, FAKE) for p in PARAMS[entry].split()])


@pytest.mark.parametrize("entry", sorted(PARAMS))
def test_return_codes_before_launch(entry):
    assert len(PARAMS[entry].split()) == len(_cabi._SIGNATURES[entry][1])
    got = [(changes, _call(entry, changes)) for e, changes, _ in CASES if e == entry]
    want = [(changes, code) for e, changes, code in CASES if e == entry]
    assert got == want


def test_supports_channels():
    assert [D for D in range(-1, 40) if L.gsb200_raster_supports_channels(D)] == list(CHANNELS)
