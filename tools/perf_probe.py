"""Quick device-side timing of the fused render on a config-2 sized batch (development aid, not the bench)."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import neurad_studio_b200 as nsb
if os.environ.get('NFF_LIB'):
    from neurad_studio_b200 import build as _b
    _b.LIB_PATH = os.environ['NFF_LIB']
    _b.needs_build = lambda: False
from neurad_studio_b200 import scene
from neurad_studio_b200.backend import B200Backend

# perf_probe.py [n_actors] [reps] [--profile DIR]: with --profile the timed renders run under torch.profiler (CUDA
# activities) instead; per-kernel device times go to stdout and DIR/kernels.json, the trace to DIR/render.pt.trace.json
argv = list(sys.argv[1:])
prof_dir = None
if "--profile" in argv:
    i = argv.index("--profile")
    prof_dir = argv[i + 1]
    del argv[i:i + 2]
n_actors = int(argv[0]) if len(argv) > 0 else 0
reps = int(argv[1]) if len(argv) > 1 else 5
be = B200Backend(torch.device("cuda", 0))
cfg = nsb.NeuRADConfig(n_actors=n_actors)
trajs = scene.make_trajectories(n_actors, cfg.duration) if n_actors else None
params = scene.make_params(cfg, seed=1, beta=3.0, sdf_bias=0.6, device="cuda", trajectories=trajs)
be.load_params(cfg, params)
be.set_mlp_mode(os.environ.get('MLP_MODE', 'split'))
rays_list = []
for cam in scene.pandaset_rig():
    r = be.raygen_pinhole(cam, 1, 3, 1, 3)
    r.pop("shape")
    n = r["origins"].shape[0]
    r["sensor_idx"] = torch.full((n, 1), cam.sensor_idx, dtype=torch.long, device="cuda")
    r["is_lidar"] = torch.zeros(n, 1, dtype=torch.uint8, device="cuda")
    rays_list.append(r)
scan = scene.pandar64_scan()
r = be.raygen_lidar_points(scan)
n = r["origins"].shape[0]
r = {k: r[k] for k in ("origins", "directions", "pixel_area", "times")}
r["sensor_idx"] = torch.full((n, 1), 6, dtype=torch.long, device="cuda")
r["is_lidar"] = torch.ones(n, 1, dtype=torch.uint8, device="cuda")
rays_list.append(r)
if os.environ.get("ONE_IMAGE"):  # one 640x360 image (230 400 rays): the per-call size of get_outputs_for_camera_ray_bundle
    rays_list = rays_list[:1]
rays = {k: torch.cat([x[k] for x in rays_list]) for k in rays_list[0]}
N = rays["origins"].shape[0]
print("rays", N)
IW = int(os.environ.get("IMAGE_WIDTH", "0"))
for _ in range(2):
    be.render(rays, image_width=IW)
torch.cuda.synchronize()
if prof_dir:
    import json
    from torch.profiler import ProfilerActivity, profile

    os.makedirs(prof_dir, exist_ok=True)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            be.render(rays, image_width=IW)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if e.device_time_total > 0:
            kern[e.key] = {"calls": e.count, "total_us": e.device_time_total, "mean_us": e.device_time_total / max(e.count, 1)}
    per_render = sum(v["total_us"] for v in kern.values()) / reps
    for k, v in sorted(kern.items(), key=lambda kv: -kv[1]["total_us"]):
        print(f"{v['mean_us'] / 1e3:9.3f} ms x {v['calls']:4d}  {100 * v['total_us'] / reps / per_render:5.1f} %  {k}")
    json.dump({"rays": N, "reps": reps, "image_width": IW, "device": torch.cuda.get_device_name(), "kernels": kern},
              open(os.path.join(prof_dir, "kernels.json"), "w"), indent=1)
    prof.export_chrome_trace(os.path.join(prof_dir, "render.pt.trace.json"))
    sys.exit(0)
ts = []
for _ in range(reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); be.render(rays, image_width=IW); e1.record(); torch.cuda.synchronize()
    ts.append(e0.elapsed_time(e1))
ms = sorted(ts)[len(ts) // 2]
print(f"render: {ms:.3f} ms median of {ts}  -> {N / ms / 1e3:.2f} M rays/s; HBM-roofline frac (69.9 kB/ray, 6562.6 GB/s) = {N * 69900 / (ms * 1e-3) / 6562.6e9:.3f}")
