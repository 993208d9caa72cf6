"""Shared bodies of the actor-edit tests (tests/test_actor_edits_cpu.py, tests/test_zz_actor_edits_gpu.py).

tests/golden/actor_edits.npz (oracle/make_golden_actor_edits.py) holds the reference's renders of one scene under the
actor edits of CASES: DynamicActors.actor_editing dicts (model_components/dynamic_actors.py:53-59, 181-249)."""
import ctypes
import os
import subprocess

import torch

from tests.helpers import cfg_from_meta, load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUTPUTS = ("features", "depth", "accumulation", "prop_depth_0", "prop_depth_1")
TRACE = ("actor_id_0", "actor_id_1", "actor_id_main")
KEYS = ("lateral", "longitudinal", "height", "rotation", "index")

_G = None


def golden():
    """(meta, cfg, params, {batch: rays}, {case: reference outputs}, {case: edit dict}, {case: batch name})."""
    global _G
    if _G is None:
        meta, g = load_golden("actor_edits.npz")
        cfg = cfg_from_meta(meta)
        rays = {b[len("ray_"):]: g[b] for b in g if b.startswith("ray_")}
        refs = {c: g[c] for c in meta["cases"]}
        _G = (meta, cfg, g["param"], rays, refs, meta["cases"], meta["batches"])
    return _G


def edit_args(edit):
    return {k: edit[k] for k in KEYS}


def rel_to_max(a, b):
    a, b = a.detach().cpu().float(), b.detach().cpu().float()
    return (a.reshape(b.shape) - b).abs().max().item() / (b.abs().max().item() + 1e-30)


def check_outputs(out, ref, ids=True):
    """The render goldens' tolerances: 1e-4 of each output's maximum (depth 2e-4); actor ids bit-exact."""
    for k in OUTPUTS:
        tol = 2e-4 if k == "depth" else 1e-4
        assert rel_to_max(out[k], ref[k]) < tol, (k, rel_to_max(out[k], ref[k]))
    if ids:
        for k in TRACE:
            n_mism = int((out[k].cpu().long().reshape(ref[k].shape) != ref[k].long()).sum())
            assert n_mism == 0, (k, n_mism)


def torch_selection(n_actors, edit):
    """The actors the reference's edit_boxes2world writes (flatten=False), by its own indexing; None: no edit."""
    if edit["longitudinal"] == 0.0 and edit["lateral"] == 0.0 and edit["rotation"] == 0.0:
        return None
    idx = torch.arange(n_actors)
    if edit["index"] == -1.0:
        return idx.tolist()
    return idx[torch.tensor([min(edit["index"], n_actors - 1)], dtype=torch.int)].tolist()


# ------------------------------------------------------------------------------------------- host emulation
def emul_lib(tmp_dir):
    src = os.path.join(ROOT, "tests", "host_emul", "emul_actor_edit.cpp")
    so = os.path.join(tmp_dir, "libemul_actor_edit.so")
    subprocess.check_call(["g++", "-std=c++20", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, src])
    lib = ctypes.CDLL(so)
    lib.emul_resolve_actor_edit.restype = ctypes.c_int
    lib.emul_resolve_actor_edit.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    lib.emul_actor_edit_frames.restype = ctypes.c_int
    lib.emul_actor_edit_frames.argtypes = [ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 7 + [ctypes.c_int] + [ctypes.c_void_p] * 7
    return lib


def emul_resolve(lib, n_actors, edit):
    e = (ctypes.c_double * 5)(*[float(edit[k]) for k in KEYS])
    first, last = ctypes.c_int(), ctypes.c_int()
    ok = lib.emul_resolve_actor_edit(n_actors, e, ctypes.byref(first), ctypes.byref(last))
    return bool(ok), first.value, last.value


def emul_frames(lib, params, rays, edit):
    """(frames [N,A,3,4], valid [N,A], lane candidates [N,A] bool, candidates' world->box [N,A,3,4])."""
    p = {k: v.float().contiguous() for k, v in params.items() if k.startswith("dynamic_actors.") and v.is_floating_point()}
    present = params["dynamic_actors.actor_present_at_time"].to(torch.uint8).contiguous()
    n_t, n_a = present.shape
    n = rays["origins"].shape[0]
    t = rays["times"].reshape(n).float().contiguous()
    o, d = rays["origins"].float().contiguous(), rays["directions"].float().contiguous()
    pad = params["dynamic_actors.actor_padding"].float().contiguous()
    frames, valid = torch.zeros(n, n_a, 12), torch.zeros(n, n_a, dtype=torch.int32)
    cand, cand_w2b = torch.zeros(n, n_a, dtype=torch.int32), torch.zeros(n, n_a, 12)
    e = (ctypes.c_double * 5)(*[float(edit[k]) for k in KEYS])
    ptr = lambda x: x.data_ptr()  # noqa: E731
    rc = lib.emul_actor_edit_frames(n_a, n_t, ptr(p["dynamic_actors.unique_timestamps"]), ptr(p["dynamic_actors.actor_rotations_6d"]),
                                    ptr(p["dynamic_actors.actor_positions"]), ptr(present), ptr(p["dynamic_actors.actor_sizes"]),
                                    ptr(pad), e, n, ptr(t), ptr(o), ptr(d), ptr(frames), ptr(valid), ptr(cand), ptr(cand_w2b))
    assert rc == 0, rc
    return frames.view(n, n_a, 3, 4), valid.bool(), cand.bool(), cand_w2b.view(n, n_a, 3, 4)


def world2box(b2w):
    """utils/poses.py:42-55 in float64: [.., 3, 4] -> [.., 3, 4]."""
    R, t = b2w[..., :3, :3].double(), b2w[..., :3, 3:].double()
    Ri = R.transpose(-2, -1)
    return torch.cat([Ri, -Ri @ t], dim=-1)


# ------------------------------------------------------------------------------------------- scene for property tests
def constant_rotation_scene(cfg_n_actors=6, seed=21, layout="torch"):
    """Actors whose rotation does not change over time (make_trajectories: a fixed yaw per actor), so that an edit's
    world-frame shift R d is the same at every keyframe and can be baked into the keyframe positions on the host."""
    import neurad_studio_b200 as nsb
    from neurad_studio_b200 import scene

    cfg = nsb.small_config(n_actors=cfg_n_actors, log2_main=14, log2_prop=13)
    trajs = scene.make_trajectories(cfg.n_actors, cfg.duration, seed=seed)
    if layout == "torch":
        params = scene.make_params(cfg, seed=seed, beta=4.0, sdf_bias=0.5, trajectories=trajs)
    else:
        params = scene.make_params_tcnn(cfg, seed=seed, beta=4.0, trajectories=trajs)
    rays = scene.random_rays(2048, cfg, seed=seed + 1, trajectories=trajs)
    return cfg, params, rays


def shifted_positions(params, lateral, longitudinal, index=-1):
    """actor_positions + R d per keyframe (R from the keyframe's own 6-D rotation, computed like the kernels' Gram-Schmidt
    in float64 then rounded): the keyframe trajectories of an unedited scene that the edit (lateral, longitudinal) of
    actor `index` (-1: all) renders."""
    r6 = params["dynamic_actors.actor_rotations_6d"].double()
    a1 = torch.nn.functional.normalize(r6[..., :3], dim=-1)
    a2 = r6[..., 3:] - (a1 * r6[..., 3:]).sum(-1, keepdim=True) * a1
    a2 = torch.nn.functional.normalize(a2, dim=-1)
    a3 = torch.cross(a1, a2, dim=-1)
    R = torch.stack([a1, a2, a3], dim=-2)  # rows, as rotation_6d_to_matrix
    d = torch.tensor([lateral, longitudinal, 0.0], dtype=torch.float64)
    pos = params["dynamic_actors.actor_positions"].double() + R @ d
    out = params["dynamic_actors.actor_positions"].clone()
    sel = slice(None) if index == -1 else slice(index, index + 1)
    out[:, sel] = pos[:, sel].float()
    return out
