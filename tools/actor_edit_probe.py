"""Cost of actor edits (DynamicActors.actor_editing) on the fused render, on one GPU.

    python tools/actor_edit_probe.py [--rounds 5] [--steps 10] [--parent-tree DIR] [--out FILE]

1. Config 3 (bench.py's config3_actors: config 2's time step, 16 rigid actors, default table sizes): the unedited render
   and the render with an all-actor translation + rotation edit, alternated round by round in one process.  Also checks
   that a render after clearing the edit is bit-identical to the first unedited one.
2. Config 2 (0 actors, bench.py's flagship step as one render): this tree against `--parent-tree` (a checkout of another
   commit with its library built), each round one child process per tree, alternated.  The children report the render
   time and a hash of the outputs, so the comparison also shows whether the two builds compute the same bits.

Times are CUDA-event times of the render call (sampling + shading kernels), median over a round's steps; the report
gives the median and range over rounds, with the card's name and power limit.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAM_RAYS = 640 * 360  # bench.py: 1920 x 1080 cameras at stride 3
EDIT = dict(lateral=1.0, longitudinal=2.0, height=0.2, rotation=0.3, index=-1.0)


def _setup(n_actors: int):
    """bench.py's time step (6 cameras + one lidar sweep at t = 1 s) with default table sizes."""
    import torch

    import neurad_studio_b200 as nsb
    from neurad_studio_b200 import scene
    from neurad_studio_b200.backend import B200Backend

    dev = torch.device("cuda", 0)
    cfg = nsb.NeuRADConfig(n_actors=n_actors)
    trajs = scene.make_trajectories(n_actors, cfg.duration) if n_actors else None
    params = scene.make_params(cfg, seed=1, beta=3.0, sdf_bias=0.6, device=dev, trajectories=trajs)
    be = B200Backend(dev)
    be.load_params(cfg, params)
    cams, scan = scene.pandaset_rig(time=1.0), scene.pandar64_scan(time=1.0, seed=0)
    n = 6 * CAM_RAYS + scan.points.shape[0]
    rays = {k: torch.empty(n, w, device=dev) for k, w in (("origins", 3), ("directions", 3), ("pixel_area", 1), ("times", 1))}
    off = 0
    for cam in cams:
        be.raygen_pinhole(cam, 1, 3, 1, 3, out={k: v[off:off + CAM_RAYS] for k, v in rays.items()})
        off += CAM_RAYS
    be.raygen_lidar_points(scan, scan.points.to(dev), out={k: v[off:] for k, v in rays.items()})
    rays["sensor_idx"] = torch.cat([torch.full((CAM_RAYS,), c.sensor_idx, dtype=torch.long) for c in cams]
                                   + [torch.full((scan.points.shape[0],), 6, dtype=torch.long)]).to(dev)
    rays["is_lidar"] = torch.cat([torch.zeros(6 * CAM_RAYS, dtype=torch.uint8), torch.ones(scan.points.shape[0], dtype=torch.uint8)]).to(dev)
    res = {k: torch.empty(n, w, device=dev) for k, w in (("features", cfg.feature_dim), ("depth", 1), ("accumulation", 1),
                                                          ("prop_depth_0", 1), ("prop_depth_1", 1))}
    return be, rays, res, n


def _time(be, rays, res, steps: int) -> float:
    import torch

    ms = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        be.render(rays, out=res, image_width=640)
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    be.check_status()
    return statistics.median(ms)


def _digest(res) -> str:
    h = hashlib.sha256()
    for k in sorted(res):
        h.update(res[k].cpu().numpy().tobytes())
    return h.hexdigest()[:16]


def _summary(xs):
    return {"median_ms": round(statistics.median(xs), 3), "min_ms": round(min(xs), 3), "max_ms": round(max(xs), 3),
            "rounds_ms": [round(x, 3) for x in xs]}


def child(steps: int) -> None:
    """Config 2 render time in this process's tree (imported from sys.path[0])."""
    be, rays, res, n = _setup(0)
    for _ in range(3):
        be.render(rays, out=res, image_width=640)
    ms = _time(be, rays, res, steps)
    print(json.dumps({"ms": ms, "digest": _digest(res), "rays": n}))


def card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # report rather than guess
        return {"error": f"{type(e).__name__}: {e}"[:200]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--parent-tree", default=None, help="another commit's tree (library built) for the config 2 comparison")
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:  # imports the tree its PYTHONPATH names
        return child(args.steps)
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("actor_edit_probe measures on a GPU; there is none")
    report = {"card": card(), "what": "CUDA-event time of one render call (sampling + shading kernels), median per round"}

    # ---- config 3: unedited vs all-actor translation + rotation edit, alternated
    be, rays, res, n = _setup(16)
    for _ in range(3):
        be.render(rays, out=res, image_width=640)
    first = _digest(res)
    be.set_actor_edit(**EDIT)
    for _ in range(3):
        be.render(rays, out=res, image_width=640)
    edited_digest = _digest(res)
    be.set_actor_edit()
    plain, edited = [], []
    for _ in range(args.rounds):
        be.set_actor_edit()
        plain.append(_time(be, rays, res, args.steps))
        be.set_actor_edit(**EDIT)
        edited.append(_time(be, rays, res, args.steps))
    be.set_actor_edit()
    be.render(rays, out=res, image_width=640)
    report["config3_16_actors"] = {
        "rays": n, "edit": EDIT, "unedited": _summary(plain), "edited": _summary(edited),
        "edited_over_unedited": round(statistics.median(edited) / statistics.median(plain), 4),
        "edit_changes_outputs": edited_digest != first, "cleared_render_bit_identical": _digest(res) == first,
    }
    del be, rays, res
    torch.cuda.empty_cache()

    # ---- config 2: this tree vs the parent tree, one child process per tree and round, alternated
    if args.parent_tree:
        trees = {"change": ROOT, "parent": os.path.abspath(args.parent_tree)}
        runs = {k: [] for k in trees}
        digests = {k: set() for k in trees}
        for _ in range(args.rounds):
            for name, tree in trees.items():
                env = dict(os.environ, PYTHONPATH=tree)
                env.pop("B200NERF_LIB", None)
                p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--steps", str(args.steps)], cwd=tree,
                                   env=env, capture_output=True, text=True)
                if p.returncode != 0:
                    raise SystemExit(f"{name} child failed:\n{p.stderr[-2000:]}")
                r = json.loads(p.stdout.strip().splitlines()[-1])
                runs[name].append(r["ms"])
                digests[name].add(r["digest"])
        report["config2_0_actors"] = {
            "parent": _summary(runs["parent"]), "change": _summary(runs["change"]),
            "change_over_parent": round(statistics.median(runs["change"]) / statistics.median(runs["parent"]), 4),
            "outputs_bit_identical": digests["parent"] == digests["change"] and len(digests["change"]) == 1,
        }
    txt = json.dumps(report, indent=1)
    print(txt)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
