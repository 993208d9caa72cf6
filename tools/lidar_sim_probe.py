"""Device time of a simulated lidar sweep (NeuRADModel.get_outputs_for_lidar_sweep), split into its three stages.

  python tools/lidar_sim_probe.py [--reps 30]

Prints the card's name, power limit and SM clock limit, then for a 64 x 1800 and a 128 x 2048 sweep with a non-uniform
beam table and per-beam azimuth offsets (default NeuRADConfig, random parameters, four actors) the median [min-max]
CUDA-event device time over --reps warmed calls of:
  raygen     B200Backend.raygen_lidar_sweeps for one sweep: the host validates the description, stages the descriptor
             and the tables in pinned memory and copies them without waiting, then b200nerf_raygen_lidar_sweeps runs; the
             event interval includes that host work, during which the device idles
  raygen_k   the b200nerf_raygen_lidar_sweeps launch alone on the already uploaded descriptor and tables
  render     the fused render of the sweep with the lidar head (B200Backend.render, want_intensity=True)
  epilogue   b200nerf_lidar_sweep_points: ray-drop decision, world and sensor-frame points, ordered compaction
  torch_post the viewer's torch lines on the same GPU and the same render outputs (viewer/render_state_machine.py:
             416-430: cat of depth * direction + origin and intensity, boolean index on ray_drop_prob < threshold) plus the
             sensor-frame transform of models/ad_model.py:107-113; the boolean index waits on the host
and whether the epilogue's points equal the torch lines' points.  The threshold is the median ray-drop probability of
the render, so that about half the rays are kept: at the random init no probability is below 0.5.
"""
import argparse
import ctypes
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import neurad_studio_b200 as nsb  # noqa: E402
from neurad_studio_b200 import scene  # noqa: E402
from neurad_studio_b200.backend import B200Backend  # noqa: E402
from tests import lidar_sim_cases as C  # noqa: E402


def timed(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return np.array(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lidar_sim_probe needs a CUDA device")
    dev = torch.device("cuda", 0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print(f"device: {torch.cuda.get_device_name(dev)}; nvidia-smi: {q[0] if q else 'n/a'}")
    be = B200Backend(dev)
    cfg = nsb.NeuRADConfig(n_actors=4)
    trajs = scene.make_trajectories(cfg.n_actors, cfg.duration)
    be.load_params(cfg, scene.make_params(cfg, seed=1, beta=3.0, sdf_bias=0.6, trajectories=trajs, device="cuda"))
    pose = C.pose_yaw(20.0, 0.0, 1.9, 0.0)[None]
    vel = torch.tensor([[10.0, 0.0, 0.0]])
    for beams, res in ((64, 360.0 / 1800), (128, 360.0 / 2048)):
        sensor = C.nonuniform_sensor(beams, seed=beams, azimuth_resolution_deg=res, revolution_time=0.1, sensor_idx=cfg.num_sensors - 1)
        st = {}

        def raygen():
            st["r"] = be.raygen_lidar_sweeps(sensor, pose, [4.0], vel)

        def raygen_k():
            r = st["r"]
            sw = r["sweeps"]  # the staged upload: descriptors, then the elevation table, then the offset table
            base, tab = sw.data_ptr() + sw.numel(), 4 * beams
            be._check(be.lib.b200nerf_raygen_lidar_sweeps(
                be._h, ctypes.c_void_p(sw.data_ptr()), 1, beams, r["shape"][2], float(np.deg2rad(res)), ctypes.c_void_p(base),
                ctypes.c_void_p(base + tab), *(ctypes.c_void_p(r[k].data_ptr()) for k in
                                               ("origins", "directions", "pixel_area", "times", "sensor_idx", "is_lidar", "index")),
                be._stream))

        def render():
            st["o"] = be.render(st["r"], want_intensity=True)
            st["o"]["ray_drop_prob"] = st["o"]["ray_drop_logits"].sigmoid()

        def epilogue():
            st["p"] = be.lidar_sweep_points(st["r"], st["o"]["depth"], st["o"]["intensity"], st["o"]["ray_drop_prob"], st["thr"])

        l2w = pose[0].to(dev)

        def torch_post():
            r, o = st["r"], st["o"]
            pc = torch.cat([o["depth"] * r["directions"] + r["origins"], o["intensity"]], dim=-1)
            pc = pc[o["ray_drop_prob"].squeeze(-1) < st["thr"]]
            rot_t = l2w[:3, :3].t()
            st["t"] = torch.cat([pc[:, :3] @ rot_t.t() - (rot_t @ l2w[:3, 3]), pc[:, 3:]], -1)

        raygen()
        render()
        st["thr"] = float(st["o"]["ray_drop_prob"].median())  # keeps about half the rays (the random init has no drops at 0.5)
        rows = {}
        for name, fn in (("raygen", raygen), ("raygen_k", raygen_k), ("render", render), ("epilogue", epilogue), ("torch_post", torch_post)):
            rows[name] = timed(fn, a.reps)
        be.check_status()
        m = int(st["p"]["counts"][-1])
        ours = st["p"]["points_sensor"][:m, :4]
        same_set = m == st["t"].shape[0]
        err = (ours - st["t"]).abs().max().item() if same_set and m else float("nan")
        n = st["r"]["origins"].shape[0]
        print(f"{beams} x {n // beams} sweep ({n} rays, {m} kept at ray_drop_prob < {st['thr']:.6f}):")
        for name, ts in rows.items():
            print(f"  {name:10s} {np.median(ts) * 1e3:10.1f} us  [{ts.min() * 1e3:.1f}-{ts.max() * 1e3:.1f}]")
        print(f"  torch_post / epilogue = {np.median(rows['torch_post']) / np.median(rows['epilogue']):.1f}x; "
              f"same kept set: {same_set}; max |points - torch| = {err:.2e}")


if __name__ == "__main__":
    main()
