"""The 3DGUT projection (ut_project_kernel) on the adversarial sweep of tests/ut_edges.py, against its float64 truth:
for every lens and parameter set, radii exact and means2d / depths / conics / compensations within their budgets on
every decided row, culled rows all zero, and the undecided rows counted per class and bounded (ut_edges.UNDECIDED_MAX)."""
import numpy as np
import pytest
import torch

from tests import ut_edges as ue

pytestmark = pytest.mark.gpu
dev = "cuda"


@pytest.fixture(scope="module")
def gs():
    import gsplat_b200

    return gsplat_b200


@pytest.fixture(scope="module")
def sweep():
    return {lens: ue.make_rows(lens) for lens in ue.LENSES}


def _t(a):
    return torch.tensor(np.ascontiguousarray(a), device=dev)


@pytest.mark.parametrize("name", [p[0] for p in ue.PARAM_SETS])
@pytest.mark.parametrize("lens", list(ue.LENSES))
def test_projection_vs_truth(gs, sweep, lens, name):
    rows, P = sweep[lens], ue.params(name)
    tr = ue.truth(rows, lens, P)
    spec = ue.LENSES[lens]
    co = {ue.COEFF_KEYS[k]: _t(np.asarray(v, np.float32)[None]) for k, v in spec["coeffs"].items()}
    out = gs.fully_fused_projection_with_ut(
        _t(rows["means"]), _t(rows["quats"]), _t(rows["scales"]), _t(rows["opacities"]), _t(ue.VM[None]),
        _t(ue.K_of(lens)[None]), ue.W, ue.H, eps2d=P["eps2d"], near_plane=P["near"], far_plane=ue.FAR,
        radius_clip=P["clip"], calc_compensations=True, camera_model=spec["kind"], ut_params=ue.ut_namespace(P), **co,
    )
    out = [o[0].cpu().numpy() for o in out]
    rep = ue.undecided_report(tr)
    print(f"\n{lens} {name} (rows, undecided, decided visible):", rep)
    msgs = ue.check_projection(rows, tr, *out, what=f"GPU {lens} {name}")
    assert not msgs, "\n".join(msgs)
    # culled rows are all zero, decided or not
    culled = (out[0] == 0).all(-1)
    for o in out[1:]:
        assert (o.reshape(len(culled), -1)[culled] == 0).all()
    msgs = ue.undecided_ceiling_msgs(tr)
    assert not msgs, "\n".join(msgs)
