"""Render and training-step time under several NeuRAD presets, alternated in one call.

  python tools/preset_probe.py [--presets neurad neurader neurad-paper] [--rounds 5] [--reps 10] [--train-steps 5]

Config 2 is six PandaSet cameras at stride 3 plus one Pandar64 sweep (1 497 600 rays, image_width = 640), rendered
untraced through the default kernel pair.  Each preset gets its own backend with random parameters of its table sizes
(neurader: a 1 GB main table, 48 MB proposal tables).  Every round renders each preset `reps` times (CUDA events per
render) after one warm-up; the rounds alternate the presets.  Prints one JSON line: the card's name and power limit, and
per preset the median and range over rounds of the per-round median render time.  Writes nothing.

Each round then runs tools/train_probe.py --preset NAME (NeuRAD's 40 960 camera + 16 384 lidar ray batch, forward + losses
+ backward through the module walk, device time of the median step) once per preset, each in its own child process; the
training keys are the median and range over rounds of those step times.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:  # the timing does not depend on it
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--presets", nargs="+", default=["neurad", "neurader", "neurad-paper"])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--train-steps", type=int, default=5)
    a = ap.parse_args()

    import torch

    import neurad_studio_b200 as nsb
    from neurad_studio_b200 import scene
    from neurad_studio_b200.backend import B200Backend

    dev = torch.device("cuda", 0)
    backends, rays = {}, None
    for name in a.presets:
        cfg, _ = nsb.preset(name)
        cfg.n_actors = 0
        be = B200Backend(dev)
        be.load_params(cfg, scene.make_params(cfg, seed=1, beta=3.0, sdf_bias=0.6, device="cuda"))
        backends[name] = be
        if rays is None:
            parts = []
            for cam in scene.pandaset_rig():
                r = be.raygen_pinhole(cam, 1, 3, 1, 3)
                r.pop("shape")
                n = r["origins"].shape[0]
                r["sensor_idx"] = torch.full((n, 1), cam.sensor_idx, dtype=torch.long, device="cuda")
                r["is_lidar"] = torch.zeros(n, 1, dtype=torch.uint8, device="cuda")
                parts.append(r)
            r = be.raygen_lidar_points(scene.pandar64_scan())
            n = r["origins"].shape[0]
            r = {k: r[k] for k in ("origins", "directions", "pixel_area", "times")}
            r["sensor_idx"] = torch.full((n, 1), 6, dtype=torch.long, device="cuda")
            r["is_lidar"] = torch.ones(n, 1, dtype=torch.uint8, device="cuda")
            parts.append(r)
            rays = {k: torch.cat([x[k] for x in parts]) for k in parts[0]}
    per_round = {name: [] for name in a.presets}
    train = {name: [] for name in a.presets}
    for _ in range(a.rounds):
        for name, be in backends.items():
            be.render(rays, image_width=640)
            ts = []
            for _ in range(a.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                be.render(rays, image_width=640)
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            per_round[name].append(statistics.median(ts))
        for be in backends.values():
            be.check_status()
        for name in a.presets:
            cmd = [sys.executable, os.path.join(ROOT, "tools", "train_probe.py"), "--preset", name, "--steps", str(a.train_steps)]
            res = subprocess.run(cmd, capture_output=True, text=True, check=True)
            train[name].append(json.loads(res.stdout.strip().splitlines()[-1])["ms_total"])
    n_rays = rays["origins"].shape[0]
    res = {name: {"ms_median": round(statistics.median(v), 3), "ms_min": round(min(v), 3), "ms_max": round(max(v), 3),
                  "Mrays_per_s": round(n_rays / statistics.median(v) / 1e3, 2)} for name, v in per_round.items()}
    tr = {name: {"ms_median": round(statistics.median(v), 3), "ms_min": round(min(v), 3), "ms_max": round(max(v), 3)}
          for name, v in train.items()}
    print(json.dumps({"card": card(), "device": torch.cuda.get_device_name(), "rays": n_rays, "rounds": a.rounds,
                      "reps": a.reps, "render": res, "train_step": tr}))


if __name__ == "__main__":
    main()
