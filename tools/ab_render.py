"""A/B of two builds of the library on the render workloads: bit-identical outputs and alternated device timings.

  python tools/ab_render.py OLD.so NEW.so [--rounds R] [--reps K]

Each build runs in its own child process, loaded through NFF_LIB as tools/perf_probe.py does.  Every child renders:
  config2      the config-2 time step (six PandaSet cameras at stride 3 + one Pandar64 sweep, image_width = 640)
  config3      the same rays with 16 actors
  nears_fars   the first camera image with per-ray nears / fars (round 0 computes its edges per ray)
untraced (all outputs) and traced (the proposal stage on every 16th ray: weights, edges, indices, actor ids; once with
actor ids, which turns the early exit off, and once without).  The parent compares every array of the two builds with
np.array_equal and byte for byte (and prints, for an array that differs, its largest difference over its largest
magnitude), then prints the median and range of the per-render device time (CUDA events) of each
build and scene (config2_traced: the full config-2 step with the proposal trace but no actor ids), over R rounds that
alternate the builds, K renders each.  Exit code 1 if any array differs.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROP_TRACE = ("prop_weights_0", "prop_weights_1", "bins_s_1", "bins_e_1", "bins_s_2", "bins_e_2", "inds_1", "inds_2",
              "actor_id_0", "actor_id_1")
PROP_TRACE_NO_AID = PROP_TRACE[:-2]
SCENES = ("config2", "config3", "nears_fars")
TIMED = ("config2", "config2_traced", "config3", "nears_fars")


def child(out_dir: str, reps: int, save: bool) -> None:
    sys.path.insert(0, ROOT)
    import torch
    import neurad_studio_b200 as nsb
    from neurad_studio_b200 import build as _b
    _b.LIB_PATH = os.environ["NFF_LIB"]
    _b.needs_build = lambda: False
    from neurad_studio_b200 import scene
    from neurad_studio_b200.backend import B200Backend

    dev = torch.device("cuda", 0)

    def rig_rays():
        be = B200Backend(dev)
        cfg = nsb.NeuRADConfig(n_actors=0)
        be.load_params(cfg, scene.make_params(cfg, seed=1, beta=3.0, sdf_bias=0.6, device="cuda"))
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
        return parts

    parts = rig_rays()
    full = {k: torch.cat([x[k] for x in parts]) for k in parts[0]}
    one = dict(parts[0])
    g = torch.Generator(device="cpu").manual_seed(7)
    n1 = one["origins"].shape[0]
    one["nears"] = (torch.rand(n1, 1, generator=g) * 2.0).to(dev)
    one["fars"] = (20.0 + torch.rand(n1, 1, generator=g) * 200.0).to(dev)
    timings = {}
    for name in SCENES:
        n_act = 16 if name == "config3" else 0
        cfg = nsb.NeuRADConfig(n_actors=n_act)
        trajs = scene.make_trajectories(n_act, cfg.duration) if n_act else None
        be = B200Backend(dev)
        be.load_params(cfg, scene.make_params(cfg, seed=1, beta=3.0, sdf_bias=0.6, device="cuda", trajectories=trajs))
        be.set_mlp_mode("split")
        rays = one if name == "nears_fars" else full
        iw = 640
        for _ in range(2):
            res = be.render(rays, image_width=iw)
        torch.cuda.synchronize()
        if save:
            arrays = {f"out.{k}": v.cpu().numpy() for k, v in res.items()}
            sub = {k: v[::16].contiguous() for k, v in rays.items()}
            for tag, fields in (("trace", PROP_TRACE), ("trace_no_aid", PROP_TRACE_NO_AID)):
                tr = be.render(sub, want_trace=set(fields))
                arrays.update({f"{tag}.{k}": v.cpu().numpy() for k, v in tr.items()})
            np.savez(os.path.join(out_dir, f"{name}.npz"), **arrays)
            del arrays
        for key, trace in ((name, False), (name + "_traced", set(PROP_TRACE_NO_AID))):
            if trace and name != "config2":
                continue
            be.render(rays, want_trace=trace, image_width=iw)
            ts = []
            for _ in range(reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                be.render(rays, want_trace=trace, image_width=iw)
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            timings[key] = {"rays": rays["origins"].shape[0], "ms": ts}
        del be
        torch.cuda.empty_cache()
    with open(os.path.join(out_dir, "timings.json"), "w") as f:
        json.dump({"device": torch.cuda.get_device_name(), "timings": timings}, f)


def run_child(lib: str, out_dir: str, reps: int, save: bool) -> dict:
    env = dict(os.environ, NFF_LIB=os.path.abspath(lib))
    cmd = [sys.executable, os.path.abspath(__file__), "--child", out_dir, "--reps", str(reps)] + (["--save"] if save else [])
    subprocess.run(cmd, env=env, check=True)
    with open(os.path.join(out_dir, "timings.json")) as f:
        return json.load(f)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="*")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--child", default=None)
    ap.add_argument("--save", action="store_true")
    a = ap.parse_args()
    if a.child:
        child(a.child, a.reps, a.save)
        return 0
    if len(a.libs) != 2:
        ap.error("need OLD.so NEW.so")
    names = ("old", "new")
    ms = {n: {s: [] for s in TIMED} for n in names}
    bad = 0
    with tempfile.TemporaryDirectory() as tmp:
        dirs = {n: os.path.join(tmp, n) for n in names}
        for d in dirs.values():
            os.makedirs(d)
        device = None
        for rnd in range(a.rounds):
            for n, lib in zip(names, a.libs):
                t = run_child(lib, dirs[n], a.reps, save=rnd == 0)
                device = t["device"]
                for s in TIMED:
                    ms[n][s] += t["timings"][s]["ms"]
            if rnd == 0:
                for s in SCENES:
                    A, B = np.load(os.path.join(dirs["old"], f"{s}.npz")), np.load(os.path.join(dirs["new"], f"{s}.npz"))
                    if sorted(A.files) != sorted(B.files):
                        print(f"{s}: different arrays {sorted(A.files)} vs {sorted(B.files)}")
                        bad += 1
                        continue
                    diff = [k for k in A.files if not (np.array_equal(A[k], B[k]) and A[k].tobytes() == B[k].tobytes())]
                    bad += len(diff)
                    print(f"{s}: {len(A.files)} arrays compared, {'all identical' if not diff else 'DIFFERENT: ' + ', '.join(diff)}")
                    for k in diff:  # max |old - new| over max |old|, the tensor's scale
                        a64, b64 = A[k].astype(np.float64), B[k].astype(np.float64)
                        scale = np.nanmax(np.abs(a64)) if a64.size else 0.0
                        print(f"    {k}: max |old - new| / max |old| = {np.nanmax(np.abs(a64 - b64)) / max(scale, 1e-30):.3g}")
                    os.remove(os.path.join(dirs["old"], f"{s}.npz"))
                    os.remove(os.path.join(dirs["new"], f"{s}.npz"))
    print(f"device: {device}; per-render device time over {a.rounds} alternated rounds x {a.reps} renders")
    for s in TIMED:
        row = []
        for n in names:
            v = np.array(ms[n][s])
            row.append(f"{n} {np.median(v):8.3f} ms [{v.min():.3f}-{v.max():.3f}]")
        gain = np.median(ms["old"][s]) / np.median(ms["new"][s])
        print(f"  {s:15s} " + "   ".join(row) + f"   old/new {gain:.3f}")
    print("bit-identical" if bad == 0 else f"{bad} arrays differ")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
