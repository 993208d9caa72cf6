"""TEST INFRASTRUCTURE ONLY -- CPU oracle for the camera models of ray generation beyond the undistorted pinhole.

`generate_rays_camera` restates Cameras._generate_rays_from_coords (cameras/cameras.py:633-667, 793-815, 898-969) for one
PERSPECTIVE or FISHEYE camera with the radial / tangential undistortion of camera_utils.py:655-758 and the AD datasets'
rolling-shutter directions, in the reference's own torch op sequence, so that on a CPU it reproduces the reference bit
for bit (oracle/make_golden_cameras.py asserts this before writing tests/golden/camera_models.npz).  With its defaults
it is oracle.neurad_oracle.generate_rays_pinhole, bit for bit (tests/test_camera_models_cpu.py checks both against
tests/golden/raygen.npz).
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
from torch import Tensor

from oracle.neurad_oracle import normalize_with_norm

CAMERA_TYPES = ("perspective", "fisheye")


def undistort_radial_tangential(coords: Tensor, k: Tensor, eps: float = 1e-3, iterations: int = 10) -> Tensor:
    """camera_utils.radial_and_tangential_undistort (camera_utils.py:655-758): Newton's method on the forward model
    x_d = x * (1 + k1 r + k2 r^2 + k3 r^3 + k4 r^4) + 2 p1 x y + p2 (r + 2 x^2) (and y alike, p1 / p2 swapped), r = x^2 + y^2,
    from (x, y) = (x_d, y_d); a step is taken only where |det J| > eps.  k = [k1, k2, k3, k4, p1, p2] (fp32).  Each line
    keeps the reference's operation order, so the result is its bits."""
    xd, yd = coords[..., 0], coords[..., 1]
    k1, k2, k3, k4, p1, p2 = (k[..., i] for i in range(6))
    x, y = xd, yd
    for _ in range(iterations):
        r = x * x + y * y
        d = 1.0 + r * (k1 + r * (k2 + r * (k3 + r * k4)))
        res_x = d * x + 2 * p1 * x * y + p2 * (r + 2 * x * x) - xd
        res_y = d * y + 2 * p2 * x * y + p1 * (r + 2 * y * y) - yd
        dd_dr = k1 + r * (2.0 * k2 + r * (3.0 * k3 + r * 4.0 * k4))
        dd_dx, dd_dy = 2.0 * x * dd_dr, 2.0 * y * dd_dr
        jxx = d + dd_dx * x + 2.0 * p1 * y + 6.0 * p2 * x
        jxy = dd_dy * x + 2.0 * p1 * x + 2.0 * p2 * y
        jyx = dd_dx * y + 2.0 * p2 * y + 2.0 * p1 * x
        jyy = d + dd_dy * y + 2.0 * p2 * x + 6.0 * p1 * y
        det = jyx * jxy - jxx * jyy
        ok = torch.abs(det) > eps
        x = x + torch.where(ok, (res_x * jyy - res_y * jxy) / det, torch.zeros_like(det))
        y = y + torch.where(ok, (res_y * jxx - res_x * jyx) / det, torch.zeros_like(det))
    return torch.stack([x, y], dim=-1)


def generate_rays_camera(
    c2w: Tensor,
    fx: float,
    fy: float,
    cx: float,
    cy: float,
    height: int,
    width: int,
    coords: Tensor,
    time: float,
    velocity: Optional[Tensor] = None,
    rolling_shutter_time: float = 0.0,
    time_to_center_pixel: float = 0.0,
    camera_type: str = "perspective",
    distortion_params: Optional[Tensor] = None,
    rs_direction: str = "Vertical",
) -> Dict[str, Tensor]:
    """Cameras._generate_rays_from_coords for one PERSPECTIVE or FISHEYE camera: distortion_params [6] = k1..k4, p1, p2
    (undistortion skipped when all are 0, as the reference does), rs_direction "Horizontal" / "Horizontal_reversed" take the
    time offset from the column (the latter negated, its time_to_center_pixel included), anything else from the row.
    coords [...,2] = (y, x) incl. the 0.5 pixel-centre offset."""
    if camera_type not in CAMERA_TYPES:
        raise ValueError(camera_type)
    y, x = coords[..., 0], coords[..., 1]
    fx_, fy_, cx_, cy_ = (torch.full_like(x, v) for v in (fx, fy, cx, cy))
    coord = torch.stack([(x - cx_) / fx_, (y - cy_) / fy_], -1)
    coord_x_offset = torch.stack([(x - cx_ + 1) / fx_, (y - cy_) / fy_], -1)
    coord_y_offset = torch.stack([(x - cx_) / fx_, (y - cy_ + 1) / fy_], -1)
    coord_stack = torch.stack([coord, coord_x_offset, coord_y_offset], dim=0)
    if distortion_params is not None:
        k = torch.as_tensor(distortion_params, dtype=torch.float32).reshape(6)
        if (k != 0).any():
            coord_stack = undistort_radial_tangential(coord_stack, k)
    coord_stack[..., 1] *= -1  # OpenCV -> OpenGL
    directions_stack = torch.empty((3,) + x.shape + (3,))
    if camera_type == "perspective":
        directions_stack[..., 0] = coord_stack[..., 0]
        directions_stack[..., 1] = coord_stack[..., 1]
        directions_stack[..., 2] = -1.0
    else:  # equidistant mapping
        theta = torch.clip(torch.sqrt(torch.sum(coord_stack**2, dim=-1)), 0.0, math.pi)
        sin_theta = torch.sin(theta)
        directions_stack[..., 0] = coord_stack[..., 0] * sin_theta / theta
        directions_stack[..., 1] = coord_stack[..., 1] * sin_theta / theta
        directions_stack[..., 2] = -torch.cos(theta)
    directions_stack = torch.sum(directions_stack[..., None, :] * c2w[:3, :3], dim=-1)
    directions_stack, directions_norm = normalize_with_norm(directions_stack, -1)
    origins = c2w[:3, 3].expand(x.shape + (3,))
    directions = directions_stack[0]
    dx = torch.sqrt(torch.sum((directions - directions_stack[1]) ** 2, dim=-1))
    dy = torch.sqrt(torch.sum((directions - directions_stack[2]) ** 2, dim=-1))
    pixel_area = (dx * dy)[..., None]
    times = torch.full(x.shape + (1,), time)
    if velocity is not None:
        horizontal = rs_direction in ("Horizontal", "Horizontal_reversed")
        pos = coords[..., 1:2] if horizontal else coords[..., 0:1]  # column for a horizontal shutter, else row
        extent = torch.full_like(pos, float(width if horizontal else height)).long()  # int64 tensors in the reference
        time_offsets = (pos / extent - 0.5) * rolling_shutter_time + time_to_center_pixel
        if rs_direction == "Horizontal_reversed":
            time_offsets = -time_offsets
        origins = origins + velocity * time_offsets
        times = times + time_offsets
    return {
        "origins": origins,
        "directions": directions,
        "pixel_area": pixel_area,
        "times": times,
        "fars": torch.ones_like(pixel_area) * 1_000_000,
        "directions_norm": directions_norm[0],
    }
