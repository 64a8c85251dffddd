"""Float64 restatement of rolling-shutter 3DGUT (test infrastructure), on top of the global-shutter oracle in
oracle/ut.py: every image row (or column) is exposed at its own pose, the start pose (viewmat) and the end pose
(viewmat_rs) interpolated at the row's relative frame time, translation linearly and rotation by slerp of the poses'
quaternions (taken from the rotation blocks from their largest component).  A sigma point is projected by a fixed-point
iteration on its frame time, starting from the start pose's projection if it is valid, else the end pose's; a pixel's
ray leaves at its row's pose; the depth and the near / far cull take the mid-frame pose; the SH view directions are
taken from the mean of the two camera positions.  Autograd differentiates the compositing as in oracle/ut.py."""
from __future__ import annotations

import math

import torch

from oracle import ut as U
from oracle.ut import F64, quat_to_rotmat

# ---- rolling shutter: ids as the reference's RollingShutterType
TOP_TO_BOTTOM, LEFT_TO_RIGHT, BOTTOM_TO_TOP, RIGHT_TO_LEFT, GLOBAL = 0, 1, 2, 3, 4
RS_ITERATIONS = 10
FLT_EPS = float(torch.finfo(torch.float32).eps)


def quat_from_rotmat(R):
    """Unit quaternion (w, x, y, z) of a rotation matrix [3, 3], from its largest component."""
    R = torch.as_tensor(R, dtype=F64)
    f = torch.stack([R[0, 0] + R[1, 1] + R[2, 2], R[0, 0] - R[1, 1] - R[2, 2], R[1, 1] - R[0, 0] - R[2, 2],
                     R[2, 2] - R[0, 0] - R[1, 1]])
    big = int(torch.argmax(f))  # the first of equal maxima, as a strict > scan
    v = torch.sqrt(f[big] + 1) * 0.5
    m = 0.25 / v
    wx, wy, wz = (R[2, 1] - R[1, 2]) * m, (R[0, 2] - R[2, 0]) * m, (R[1, 0] - R[0, 1]) * m
    xy, xz, yz = (R[1, 0] + R[0, 1]) * m, (R[0, 2] + R[2, 0]) * m, (R[2, 1] + R[1, 2]) * m
    return torch.stack([(v, wx, wy, wz), (wx, v, xy, xz), (wy, xy, v, yz), (wz, xz, yz, v)][big])


def slerp(q0, q1, a):
    """Normalised slerp of two unit quaternions at a (a tensor [P], not clamped) -> [P, 4]: the short arc, a
    component-wise lerp when cos(theta) > 1 - FLT_EPSILON."""
    a = torch.as_tensor(a, dtype=F64).reshape(-1, 1)
    c = float((q0 * q1).sum())
    if c < 0:
        q1, c = -q1, -c
    if c > 1 - FLT_EPS:
        q = q0 * (1 - a) + q1 * a
    else:
        th = math.acos(c)
        q = (torch.sin((1 - a) * th) * q0 + torch.sin(a * th) * q1) / math.sin(th)
    return q / q.norm(dim=-1, keepdim=True)


def frame_time(shutter, W, H, u, v):
    """Relative frame time of image points (u, v): that of their row (or column)."""
    u, v = torch.as_tensor(u, dtype=F64), torch.as_tensor(v, dtype=F64)
    if shutter == TOP_TO_BOTTOM:
        return torch.floor(v) / (H - 1)
    if shutter == LEFT_TO_RIGHT:
        return torch.floor(u) / (W - 1)
    if shutter == BOTTOM_TO_TOP:
        return (H - torch.ceil(v)) / (H - 1)
    return (W - torch.ceil(u)) / (W - 1)


class ShutterPoses:
    """A rolling-shutter camera's start and end poses (row-major 4x4 view matrices) as quaternions and translations;
    ``at(a)`` -> (R [P, 3, 3], t [P, 3]) at relative frame times a [P]: translation lerp, rotation slerp."""

    def __init__(self, viewmat, viewmat_rs):
        vm0, vm1 = torch.as_tensor(viewmat, dtype=F64), torch.as_tensor(viewmat_rs, dtype=F64)
        self.q0, self.q1 = quat_from_rotmat(vm0[:3, :3]), quat_from_rotmat(vm1[:3, :3])
        self.t0, self.t1 = vm0[:3, 3], vm1[:3, 3]

    def at(self, a):
        a = torch.as_tensor(a, dtype=F64).reshape(-1)
        t = (1 - a)[:, None] * self.t0 + a[:, None] * self.t1
        return quat_to_rotmat(slerp(self.q0, self.q1, a)), t


def rs_project(points, cam, poses: ShutterPoses, shutter, margin):
    """World points [P, 3] -> (uv [P, 2], valid [P], edge [P]) through a rolling shutter: start from the start pose's
    projection if valid, else the end pose's (neither: invalid, at the end pose's point); then re-project at the frame
    time of the current point until that time repeats, at most 10 times.  ``edge``: a point whose row (or column)
    coordinate came within 1e-3 pixel of a boundary on the way, where float32 may pick the neighbouring row's pose."""
    P = points.shape[0]

    def proj(a):
        R, t = poses.at(a)
        return cam.project(torch.einsum("pij,pj->pi", R, points) + t, margin)

    uv0, ok0 = proj(torch.zeros(P, dtype=F64))
    uv1, ok1 = proj(torch.ones(P, dtype=F64))
    uv = torch.where(ok0[:, None], uv0, uv1)
    valid = ok0 | ok1
    live = valid.clone()
    prev = torch.full((P,), -math.inf, dtype=F64)
    coord = 1 if shutter in (TOP_TO_BOTTOM, BOTTOM_TO_TOP) else 0
    edge = torch.zeros(P, dtype=torch.bool)
    for _ in range(RS_ITERATIONS):
        a = frame_time(shutter, cam.W, cam.H, uv[:, 0], uv[:, 1])
        x = uv[:, coord]
        edge = edge | (live & ((x - torch.round(x)).abs() < 1e-3))
        live = live & (a != prev)
        if not bool(live.any()):
            break
        prev = torch.where(live, a, prev)
        uv_n, ok_n = proj(a)
        uv = torch.where(live[:, None], uv_n, uv)
        valid = torch.where(live, ok_n, valid)
    return uv, valid, edge


def rs_sh_viewmat(viewmat, viewmat_rs):
    """[..., 4, 4] view matrices [I | -c] with c the mean of the two poses' positions -R^T t: the camera position the
    SH view directions of a rolling-shutter camera are taken from."""
    vm0, vm1 = torch.as_tensor(viewmat, dtype=F64), torch.as_tensor(viewmat_rs, dtype=F64)
    pos = lambda vm: -torch.einsum("...ji,...j->...i", vm[..., :3, :3], vm[..., :3, 3])  # noqa: E731
    out = torch.zeros(vm0.shape, dtype=F64)
    out[..., :3, :3] = torch.eye(3, dtype=F64)
    out[..., :3, 3] = -0.5 * (pos(vm0) + pos(vm1))
    out[..., 3, 3] = 1
    return out



class _RollingCamera:
    """A camera model that projects WORLD points through the rolling shutter (oracle.ut.ut_projection is run with an
    identity view matrix, so its camera-frame points are the world points); records the boundary flags."""

    def __init__(self, cam, poses, shutter):
        self.cam, self.poses, self.shutter = cam, poses, shutter
        self.W, self.H = cam.W, cam.H
        self.edge = None

    def project(self, pts, margin):
        uv, valid, edge = rs_project(pts.reshape(-1, 3), self.cam, self.poses, self.shutter, margin)
        self.edge = edge.reshape(pts.shape[:-1])
        return uv.reshape(pts.shape[:-1] + (2,)), valid.reshape(pts.shape[:-1])


def ut_projection(means, quats, scales, opacities, viewmat, cam, eps2d=0.3, near_plane=0.01, far_plane=1e10,
                  radius_clip=0.0, ut=None, viewmat_rs=None, shutter=GLOBAL):
    """oracle.ut.ut_projection under either shutter.  Rolling: sigma points through rs_project, the depth and the
    near / far cull at the mid-frame pose; ``rs_edge`` [N] marks the rows with a sigma point near a row (column)
    boundary, where float32 may take the neighbouring row's pose."""
    if shutter == GLOBAL:
        out = U.ut_projection(means, quats, scales, opacities, viewmat, cam, eps2d, near_plane, far_plane, radius_clip, ut)
        out["rs_edge"] = torch.zeros(len(out["valid"]), dtype=torch.bool)
        return out
    poses = ShutterPoses(viewmat, viewmat_rs)
    rc = _RollingCamera(cam, poses, shutter)
    out = U.ut_projection(means, quats, scales, opacities, torch.eye(4, dtype=F64), rc, eps2d, -math.inf, math.inf,
                          radius_clip, ut)
    R, t = poses.at(torch.tensor([0.5], dtype=F64))
    zc = torch.as_tensor(means, dtype=F64) @ R[0, 2] + t[0, 2]
    keep = out["valid"] & (zc >= near_plane) & (zc <= far_plane)
    for k in ("radii", "means2d", "conics"):
        out[k] = torch.where(keep[:, None], out[k], torch.zeros_like(out[k]))
    out["compensations"] = torch.where(keep, out["compensations"], torch.zeros_like(zc))
    out["depths"] = torch.where(keep, zc, torch.zeros_like(zc))
    out["valid"], out["rs_edge"] = keep, rc.edge.any(1)
    return out


def pixel_rays(viewmat, cam, viewmat_rs=None, shutter=GLOBAL):
    """World rays of every pixel centre (origins, unit directions, valid [H*W]); rolling: each pixel's ray leaves at
    the pose of its row (column)."""
    if shutter == GLOBAL:
        return U.pixel_rays(viewmat, cam)
    jj, ii = torch.meshgrid(torch.arange(cam.W, dtype=F64), torch.arange(cam.H, dtype=F64), indexing="xy")
    u, v = jj.reshape(-1) + 0.5, ii.reshape(-1) + 0.5
    d, ok = cam.unproject(u, v)
    R, t = ShutterPoses(viewmat, viewmat_rs).at(frame_time(shutter, cam.W, cam.H, u, v))
    return -torch.einsum("pji,pj->pi", R, t), torch.einsum("pji,pj->pi", R, d), ok


def eval3d_render(means, quats, scales, colors, opacities, viewmat, cam, isect_offsets, flatten_ids, C, N, image_index,
                  background=None, mask=None, viewmat_rs=None, shutter=GLOBAL):
    """oracle.ut.eval3d_render under either shutter: the same compositing of the pixels' rays of pixel_rays."""
    if shutter == GLOBAL:
        return U.eval3d_render(means, quats, scales, colors, opacities, viewmat, cam, isect_offsets, flatten_ids, C, N,
                               image_index, background, mask)
    global_rays = U.pixel_rays
    U.pixel_rays = lambda vm, c: pixel_rays(vm, c, viewmat_rs, shutter)  # the compositing takes its rays from here
    try:
        return U.eval3d_render(means, quats, scales, colors, opacities, viewmat, cam, isect_offsets, flatten_ids, C, N,
                               image_index, background, mask)
    finally:
        U.pixel_rays = global_rays
