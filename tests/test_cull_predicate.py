"""The warp-level culling predicate of the compositing kernels (csrc/raster.cu block_may_touch + the extents
computed by pack_records_kernel), restated in numpy and checked on the oracle's projection of the garden scene:
it must be CONSERVATIVE (never drop a (8x4 pixel block, gaussian) pair in which some pixel reaches alpha >= 1/255)
and it is measured against the exact answer.  At BASELINE cfg3, on the oracle's projection:
63.3 % of the pairs survive the test, 58.4 % is exact, 24.3 of 32 lanes are valid in a surviving pair."""
import numpy as np

from oracle import gso
from tests import scene


def _pairs(n_sample=60000, seed=0):
    sc = scene.make_scene(scene_grid=1, sh_degree=0)
    W, H = 1920, 1080
    Ks = scene.rescale_K(sc["Ks"], sc["width"], sc["height"], W, H)[:1]
    vm = sc["viewmats"][:1]
    radii, m2, dep, con, _ = gso.fully_fused_projection(
        sc["means"], None, sc["quats"], sc["scales"], vm, Ks, W, H, 0.3, 0.01, 1e10, 0.0, False, "pinhole", sc["opacities"]
    )
    op = np.broadcast_to(sc["opacities"][None], dep.shape)
    tw, th = 120, 68
    _, ids, fl = gso.isect_tiles(m2, radii, dep, 16, tw, th, True, con, op)
    tile = ((ids >> 32) & ((1 << 13) - 1)).astype(np.int64)
    sel = np.random.RandomState(seed).choice(len(fl), min(n_sample, len(fl)), replace=False)
    g, t = fl[sel], tile[sel]
    f = lambda x: x.astype(np.float64)  # noqa: E731
    return (f(m2[0, g, 0]), f(m2[0, g, 1]), f(con[0, g, 0]), f(con[0, g, 1]), f(con[0, g, 2]), f(op[0, g]),
            (t % tw) * 16, (t // tw) * 16)


def test_block_cull_is_conservative_and_tight():
    mx, my, a, b, c, o, tx, ty = _pairs()
    thr = np.log(255.0 * o)  # q <= thr  <=>  o * exp(-q) >= 1/255,  q = (a dx^2 + c dy^2) / 2 + b dx dy
    det = a * c - b * b
    t2 = 2.0 * thr
    ex, ey = np.sqrt(t2 * c / det), np.sqrt(t2 * a / det)  # axis-aligned half extents of the ellipse
    hd = 0.5 * (a - c)
    l1 = 0.5 * (a + c) + np.sqrt(hd * hd + b * b)
    l2 = det / l1
    v1, v2 = (b, l1 - a), (l1 - c, b)
    use2 = v2[0] ** 2 + v2[1] ** 2 > v1[0] ** 2 + v1[1] ** 2
    vx, vy = np.where(use2, v2[0], v1[0]), np.where(use2, v2[1], v1[1])
    nn = np.sqrt(vx * vx + vy * vy)
    ux, uy = vx / nn, vy / nn  # unit eigenvector of the larger eigenvalue
    lu, lv = np.sqrt(t2 / l1), np.sqrt(t2 / l2)  # half lengths of the oriented box
    kept = exact = total = 0
    hx, hy = 3.5, 1.5
    for w in range(8):
        bx0, by0 = tx + (w & 1) * 8, ty + (w >> 1) * 4
        dx, dy = mx - (bx0 + 4.0), my - (by0 + 2.0)
        keep = ((np.abs(dx) <= ex + hx) & (np.abs(dy) <= ey + hy)
                & (np.abs(dx * ux + dy * uy) <= lu + hx * np.abs(ux) + hy * np.abs(uy))
                & (np.abs(dy * ux - dx * uy) <= lv + hx * np.abs(uy) + hy * np.abs(ux)))
        px = bx0[:, None] + (np.arange(32) % 8)[None] + 0.5
        py = by0[:, None] + (np.arange(32) // 8)[None] + 0.5
        ddx, ddy = mx[:, None] - px, my[:, None] - py
        q = 0.5 * (a[:, None] * ddx**2 + c[:, None] * ddy**2) + b[:, None] * ddx * ddy
        hit = ((q <= thr[:, None]) & (q >= 0)).any(1)
        assert not (hit & ~keep).any(), "the block test dropped a pair that reaches the alpha threshold"
        kept, exact, total = kept + keep.sum(), exact + hit.sum(), total + len(mx)
    assert exact > 0.3 * total  # the sample is meaningful
    assert kept <= 1.12 * exact, f"block test too loose: keeps {kept / total:.3f}, exact {exact / total:.3f}"
