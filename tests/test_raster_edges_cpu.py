"""Self-check of the adversarial single-gaussian sweep (tests/raster_edges.py) on the CPU: the float32 oracle, which
follows the reference's per-pair formula, must agree with the float64 truth within the float32 error budget on every
decided pixel, and may only differ by returning 0 on an undecided one.  The fraction of undecided pixels is bounded
per anisotropy class, so that the GPU sweep keeps checking most of what it renders."""
import numpy as np
import pytest

from oracle import gso
from tests import raster_edges as re_


@pytest.fixture(scope="module")
def sweep():
    sw = re_.make_sweep()
    return sw, re_.truth(sw)


def test_sweep_covers_the_edges(sweep):
    sw, tr = sweep
    I = sw["means2d"].shape[0]
    assert I >= 1500 and sw["isect_offsets"].shape == (I, 3, 3) and sw["flatten_ids"].shape == (I * 9,)
    for k in re_.ANISO:
        assert (sw["aniso"] == k).sum() >= 100, k
    for kind in re_.PLACEMENTS:
        assert (sw["placement"] == kind).sum() >= 100, kind
    for op in re_.OPACITIES:
        assert np.isclose(sw["opacities"][:, 0], op, rtol=1e-7, atol=0).sum() >= 100, op
    m = sw["means2d"][:, 0]
    assert ((m[:, 0] < -300) | (m[:, 0] > re_.W + 300)).sum() >= 50, "centres several hundred pixels outside"
    touched = tr["alpha"] > 0
    # pixels are touched in the partial right column and bottom row of tiles, and by gaussians centred outside
    assert touched[:, :, 32:].any(axis=(1, 2)).sum() > 200 and touched[:, 32:, :].any(axis=(1, 2)).sum() > 200
    outside = (m[:, 0] < 0) | (m[:, 0] > re_.W) | (m[:, 1] < 0) | (m[:, 1] > re_.H)
    assert (touched.any(axis=(1, 2)) & outside).sum() > 200
    # boundary-targeted gaussians put a decided pixel within 1 % of the alpha threshold
    near = tr["decided"] & touched & (tr["alpha"] < re_.ALPHA_TH * 1.01)
    assert near.any(axis=(1, 2)).sum() > 300


def test_float32_oracle_matches_float64_truth(sweep):
    sw, tr = sweep
    for D in (3, 5):
        rc, ra = gso.rasterize_to_pixels(
            sw["means2d"], sw["conics"], sw[f"colors{D}"], sw["opacities"], re_.W, re_.H, 16, sw["isect_offsets"],
            sw["flatten_ids"], sw[f"bg{D}"],
        )
        nan = tr["nan_alpha"]
        msgs = re_.check_render(sw, tr, rc, ra, D, what=f"float32 oracle D={D}", skip=nan)
        assert not msgs, "\n".join(msgs)
        # the reference's formula clamps a NaN alpha to 0.99 (fminf) and keeps the pair; the kernels reject it
        assert nan.sum() > 1000 and set(np.unique(ra[..., 0][nan]).tolist()) <= {0.0, np.float32(re_.MAX_ALPHA)}


def test_undecided_fraction_is_bounded(sweep):
    sw, tr = sweep
    rep = re_.undecided_report(sw, tr)
    print("\nundecided pixels / (touched or undecided) pixels, gaussians with an undecided pixel:")
    for k, (fp, fg) in rep.items():
        print(f"  anisotropy {k}: {fp:.4%} of pixels, {fg:.2%} of gaussians")
    for k, (fp, fg) in rep.items():
        # needles' sigma cancels between large terms: their boundaries are wide in float32
        lim_p, lim_g = 0.03, 0.35
        assert fp <= lim_p and fg <= lim_g, (k, fp, fg)
    assert (~tr["decided"]).mean() < 1e-2
