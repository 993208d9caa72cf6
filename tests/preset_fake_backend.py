"""TEST SCAFFOLDING ONLY -- tests/fake_backend.py with the fused render run by the host emulation of the kernels
(tests/host_emul/emul.cpp), so that the per-sensor appearance epilogue is the device code itself.  The appearance mode
reaches the emulated parameter block the way B200Backend.load_params binds it: Appearance.eps = embeddings per sensor, or 0
for one row per sensor (b200nerf_set_appearance_per_sensor)."""
import torch

from oracle import neurad_oracle as O
from tests.fake_backend import FakeBackend


class _EmulCfg:
    def __init__(self, cfg):
        self._cfg = cfg

    def __getattr__(self, k):
        if k == "embeds_per_sensor":
            return self._cfg.embeds_per_sensor if self._cfg.use_temporal_appearance else 0
        return getattr(self._cfg, k)


def emul_cfg(cfg):
    return _EmulCfg(cfg)


class PresetFakeBackend(FakeBackend):
    def render(self, rays, want_trace=False, want_intensity=False, out=None, image_width=0):
        from tests.host_emul import emul

        n = rays["origins"].shape[0]
        r = {"origins": rays["origins"].reshape(n, 3), "directions": rays["directions"].reshape(n, 3),
             "pixel_area": rays["pixel_area"].reshape(n, 1), "times": rays["times"].reshape(n, 1)}
        for k in ("nears", "fars", "sensor_idx", "is_lidar"):
            if k in rays:
                r[k] = rays[k].reshape(n, 1)
        res = emul.render(emul_cfg(self.cfg), self.params, {k: v.detach().cpu() for k, v in r.items()}, O.pdf_u, lane_mode=True)
        res = {k: res[k] for k in ("features", "depth", "accumulation", "prop_depth_0", "prop_depth_1")}
        if want_intensity:
            with torch.no_grad():
                res["intensity"], res["ray_drop_logits"] = O.decode_lidar(self.params, res["features"])
        return res
