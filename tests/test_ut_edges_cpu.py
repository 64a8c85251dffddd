"""The 3DGUT projection sweep of tests/ut_edges.py checks itself without a GPU: every class is present under every lens,
the exact-UT ties sit exactly on their thresholds and take the branch they are built for (culled under
require_all_sigma_points_valid, kept otherwise), the rows whose float32 transform overflows are culled, the budgets are
finite and small beside the quantities, and the truth's visibility is the oracle's on every decided row."""
import numpy as np
import pytest

from tests import ut_edges as ue


@pytest.fixture(scope="module")
def sweep():
    return {lens: ue.make_rows(lens) for lens in ue.LENSES}


def _truth(sweep, lens, name):
    return ue.truth(sweep[lens], lens, ue.params(name))


@pytest.mark.parametrize("lens", list(ue.LENSES))
def test_classes_present_and_decided(sweep, lens):
    rows = sweep[lens]
    decided = {c: 0 for c in ue.CLASSES[lens]}
    for P in ue.PARAM_SETS:
        tr = _truth(sweep, lens, P[0])
        rep = ue.undecided_report(tr)
        print(f"\n{lens} {P[0]} (rows, undecided, decided visible):", rep)
        for c in ue.CLASSES[lens]:
            n, und, _ = rep.get(c, (0, 0, 0))
            decided[c] += n - und
        msgs = ue.undecided_ceiling_msgs(tr)
        assert not msgs, "\n".join(msgs)
    for c in ue.CLASSES[lens]:
        assert (rows["cls"] == c).sum() >= 4, c
        assert decided[c] >= 4, (lens, c, decided[c])


def test_exact_ties(sweep):
    rows = sweep["pinhole"]
    m = (rows["cls"] == "margin") & rows["exact"]
    assert m.sum() == 8
    for name, margin, sel in (("exact/m0", 0.0, slice(0, 4)), ("exact/all/m0.5", 0.5, slice(4, 8))):
        tr = _truth(sweep, "pinhole", name)
        m = np.zeros_like(m)
        m[np.flatnonzero((rows["cls"] == "margin") & rows["exact"])[sel]] = True
        q = tr.q
        mx, my = ue.W * margin, ue.H * margin
        on = np.isin(q["u"], [-mx, ue.W + mx]) | np.isin(q["v"], [-my, ue.H + my])
        assert on[m].any(1).all(), "each margin tie row has a sigma point exactly on an edge"
        right = m & (on & ((q["u"] == ue.W + mx) | (q["v"] == ue.H + my))).any(1)
        left = m & ~right
        assert right.sum() == 2 and left.sum() == 2
        assert tr.decided[m].all()
        if "all" in name:
            # in_margin is half-open: a point on the far edge is invalid, one on the near edge valid
            # (with margin 0.5 the rows lie beyond the image: the off-screen test culls them all)
            assert not tr.vis[right].any() and (tr.vis[left].all() or margin > 0)
        else:
            assert tr.vis[m].all()
    m = (rows["cls"] == "margin") & rows["exact"]
    b = (rows["cls"] == "behind") & rows["exact"]
    tr = _truth(sweep, "pinhole", "exact/m0")
    assert (tr.q["z"][b] == 0).any(1).all()
    assert tr.margins["ut_valid"][b].all(), "any-valid keeps a row with a point at z == 0, (0, 0) averaged in"
    tr = _truth(sweep, "pinhole", "exact/all/m0")
    assert tr.decided[b].all() and not tr.vis[b].any()
    # a distorted sigma point whose icD is float32(0.8) in float32 as in float64: invalid (icD > 0.8 fails), so
    # all-valid culls the row and any-valid keeps it
    assert np.float32(1) + np.float32(ue.K1) == np.float32(0.8) and 1 + ue.K1 == ue.F32(0.8)
    d = (sweep["distorted"]["cls"] == "icd") & sweep["distorted"]["exact"]
    assert d.sum() == 2
    for name, vis in (("exact/m0", True), ("exact/all/m0", False)):
        tr = _truth(sweep, "distorted", name)
        assert (tr.q["icd"][d] == ue.F32(0.8)).any(1).all()
        assert tr.decided[d].all() and (tr.vis[d] == vis).all(), name
    # the exact UT's float32 weights are the float64 ones
    assert ue.weights32(ue.EXACT_UT) == (2.0, 0.25, 0.25, 0.125)


@pytest.mark.parametrize("lens", list(ue.LENSES))
def test_branches(sweep, lens):
    rows = sweep[lens]
    for P in ue.PARAM_SETS:
        tr = _truth(sweep, lens, P[0])
        ov = rows["cls"] == "overflow"
        assert not tr.vis[ov].any(), "rows whose float32 transform overflows are culled"
        dg = (rows["cls"] == "degenerate") & tr.decided & ((tr.q["qn2"] < ue.FLT_EPS) | (tr.q["smin"] < ue.FLT_EPS))
        assert not tr.vis[dg].any()
        npd = (rows["cls"] == "nonpd") & tr.decided
        if P[1] == ue.NEG_BETA_UT:
            # the negative centre weight makes these covariances indefinite: culled by det or c00 / c11
            assert (~tr.margins["pd"][npd]).sum() >= 3 and not tr.vis[npd & ~tr.margins["pd"]].any()
        # the truth's visibility is the oracle's (float32 thresholds, overflow culled) on every decided row
        dec = tr.decided
        assert (tr.vis[dec] == tr.oracle_valid[dec]).all(), P[0]


@pytest.mark.parametrize("lens", list(ue.LENSES))
def test_budgets_finite_and_small(sweep, lens):
    for name in ("exact/m0", "other/all/m0.1/clip3"):
        tr = _truth(sweep, lens, name)
        ok = tr.decided & tr.vis
        assert ok.sum() >= 10
        for k in ("means2d", "depths", "conics", "compensations"):
            b = np.asarray(tr.beta[k]).reshape(len(ok), -1)[ok]
            ref = np.abs(getattr(tr, k).reshape(len(ok), -1)[ok])
            assert np.isfinite(b).all(), k
            assert (b <= 5e-2 * np.maximum(ref, 1.0)).all(), (k, float((b / np.maximum(ref, 1.0)).max()))
