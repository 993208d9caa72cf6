"""TEST SCAFFOLDING ONLY -- tests/fake_backend.py's CPU stand-in plus B200Backend.raygen_camera over the oracle
(oracle/camera_oracle.py), with the backend's own descriptor validation."""
import torch

from neurad_studio_b200.backend import camera_descriptor
from oracle import camera_oracle as CO
from tests.fake_backend import FakeBackend


class CameraFakeBackend(FakeBackend):
    def raygen_camera(self, cam, row0=0, row_step=1, col0=0, col_step=1, out=None):
        camera_descriptor(cam)  # the same ValueErrors as B200Backend.raygen_camera
        ys, xs = torch.meshgrid(torch.arange(row0, cam.height, row_step), torch.arange(col0, cam.width, col_step), indexing="ij")
        coords = (torch.stack([ys, xs], -1).reshape(-1, 2) + 0.5).float()
        r = CO.generate_rays_camera(cam.c2w, cam.fx, cam.fy, cam.cx, cam.cy, cam.height, cam.width, coords, cam.time, cam.velocity,
                                    cam.rolling_shutter_time, cam.time_to_center_pixel, cam.camera_type, cam.distortion_params,
                                    cam.rs_direction)
        return {"origins": r["origins"].contiguous(), "directions": r["directions"], "pixel_area": r["pixel_area"], "times": r["times"],
                "shape": tuple(ys.shape)}

    def raygen_pinhole(self, cam, row0=0, row_step=1, col0=0, col_step=1, out=None):
        return self.raygen_camera(cam, row0, row_step, col0, col_step, out)
