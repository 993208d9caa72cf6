"""CPU: actor edits (DynamicActors.actor_editing, model_components/dynamic_actors.py:181-249) against the reference.

- The oracle renders every edited case of tests/golden/actor_edits.npz as the reference did.
- The host emulation of the edited frame builders (actor_frame<true>, lane_actor_candidates<true>) gives the reference's
  edited world->box transforms, and its ray-line cull uses the edited box centres.
- The host-side index resolution (resolve_actor_edit) selects the actors the reference's own indexing selects, and
  rejects an index below -n_actors.
- The mirror and the reference plugin hand the edit dict to the backend: in eval mode as it is, in training mode zeros.
"""
import math

import pytest
import torch

from oracle import actor_edit_oracle as AE
from oracle import neurad_oracle as O
from oracle import ref_import
from oracle.convert import to_oracle_cfg
from tests import actor_edit_cases as C
from tests.test_reference_plugin import plugin  # noqa: F401  (fixture: the plugin registered through the reference)

needs_reference = pytest.mark.skipif(not ref_import.reference_available(), reason="the reference tree is not present")


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return C.emul_lib(str(tmp_path_factory.mktemp("emul_actor_edit")))


@pytest.mark.parametrize("case", list(C.golden()[5]))
def test_oracle_reproduces_reference(case):
    meta, cfg, params, rays, refs, edits, batches = C.golden()
    r, ref = rays[batches[case]], refs[case]
    unedited = O.boxes2world_at
    with torch.no_grad():
        out = AE.nff_outputs(params, to_oracle_cfg(cfg), r["origins"], r["directions"], r["pixel_area"], r["times"],
                             r["sensor_idx"], r["is_lidar"], want_trace=True, edit=edits[case])
    assert O.boxes2world_at is unedited  # the edit applies only inside the call
    out.update(out.pop("trace"))
    for k in C.OUTPUTS:
        assert C.rel_to_max(out[k], ref[k]) < 1e-6, k
    for k in C.TRACE:
        assert torch.equal(out[k].long(), ref[k].long()), k


def test_golden_cases_cover_the_quirks():
    _, _, _, _, refs, edits, _ = C.golden()
    assert torch.equal(refs["height_only"]["features"], refs["none"]["features"])  # a height alone is no edit
    assert not torch.equal(refs["height_lateral"]["boxes2world"][..., 2, 3], refs["lateral"]["boxes2world"][..., 2, 3])
    # training mode: the reference's get_boxes2world ignores the edit
    assert torch.equal(C.golden()[4]["none"]["boxes2world"], load_train_boxes())


def load_train_boxes():
    from tests.helpers import load_golden

    return load_golden("actor_edits.npz")[1]["train"]["boxes2world"]


@pytest.mark.parametrize("case", list(C.golden()[5]))
def test_emulated_frames_match_reference_boxes(emul, case):
    """actor_frame<true> gives the reference's edited world->box at every ray time; the lane cull keeps exactly the actors
    whose EDITED centre is near the ray line (up to the kernel's 1e-3 slack) and stores the same transform."""
    meta, cfg, params, rays, refs, edits, batches = C.golden()
    r = rays[batches[case]]
    frames, valid, cand, cand_w2b = C.emul_frames(emul, params, r, edits[case])
    want = C.world2box(refs[case]["boxes2world"])
    assert (frames.double() - want).abs().max().item() < 2e-5
    assert torch.equal(cand_w2b[cand], frames[cand])
    centre = refs[case]["boxes2world"][..., :3, 3].double()
    bounds = params["dynamic_actors.actor_sizes"] / 2 + params["dynamic_actors.actor_padding"]
    radius = bounds.double().norm(dim=-1)
    v = centre - r["origins"].double()[:, None, :]
    dist = torch.linalg.norm(torch.cross(v, r["directions"].double()[:, None, :].expand_as(v), dim=-1), dim=-1)
    assert not (cand & ~valid).any()
    assert (cand | ~(valid & (dist < 0.999 * radius))).all(), "an actor near the ray line was culled"
    assert (~cand | (dist < 1.002 * radius)).all(), "a far actor was kept"
    if case == "onto":  # the rays aimed beside actors 2 and 3 reach them only through the edited centre
        lo, hi = meta["onto_rays"]
        assert cand[lo:hi, 2:4].any(-1).all()
        unedited = C.world2box(refs["none"]["boxes2world"])
        assert not torch.equal(unedited[lo:hi], want[lo:hi])


@pytest.mark.parametrize("n_actors", [1, 2, 6])
@pytest.mark.parametrize("index", [-1.0, 0.0, 1.0, 2.0, 2.9, 5.0, 5.5, 9.0, 1e9, -0.5, -1.5, -2.0, -5.0, -6.0, -6.5])
@pytest.mark.parametrize("shift", [dict(lateral=0.5), dict(rotation=0.2), dict(height=0.5), dict(height=0.5, longitudinal=-0.1), {}])
def test_index_resolution_matches_reference_indexing(emul, n_actors, index, shift):
    edit = {"lateral": 0.0, "longitudinal": 0.0, "height": 0.0, "rotation": 0.0, "index": index, **shift}
    ok, first, last = C.emul_resolve(emul, n_actors, edit)
    try:
        want = C.torch_selection(n_actors, edit)
    except IndexError:
        assert not ok and first == last == 0
        return
    assert ok
    assert list(range(first, last)) == ([] if want is None else want)


@pytest.mark.parametrize("index", [-7.0, -7.9, -100.0, float("nan")])
def test_index_below_minus_n_actors_is_rejected(emul, index):
    edit = {"lateral": 0.5, "longitudinal": 0.0, "height": 0.0, "rotation": 0.0, "index": index}
    if not math.isnan(index):
        with pytest.raises(IndexError):
            C.torch_selection(6, edit)
    assert C.emul_resolve(emul, 6, edit) == (False, 0, 0)
    assert C.emul_resolve(emul, 0, edit) == (True, 0, 0)  # no actors: nothing to edit, nothing to reject


# ------------------------------------------------------------------------------------------- Python glue
class _EditRecorder:
    """Stands in for B200Backend.set_actor_edit."""

    def __init__(self):
        self.calls = []

    def __call__(self, **kw):
        self.calls.append({k: kw.get(k, d) for k, d in zip(C.KEYS, (0.0, 0.0, 0.0, 0.0, -1.0))})


def test_mirror_forwards_actor_editing(monkeypatch):
    import neurad_studio_b200 as nsb
    from neurad_studio_b200 import nerfstudio_api as api
    from tests.fake_backend import FakeBackend

    be = FakeBackend()
    rec = _EditRecorder()
    be.set_actor_edit = rec
    monkeypatch.setattr(api, "get_backend", lambda device: be)
    model = api.NeuRADModel(nsb.small_config(n_actors=2, log2_main=10, log2_prop=10))
    assert model.dynamic_actors.actor_editing == {"lateral": 0.0, "longitudinal": 0.0, "rotation": 0.0, "index": -1.0, "height": 0.0}
    edit = {"lateral": 1.0, "longitudinal": -2.0, "rotation": 0.3, "index": 1.0, "height": 0.25}
    model.dynamic_actors.actor_editing.update(edit)
    model.eval()
    model._bind()
    assert rec.calls[-1] == {k: edit[k] for k in C.KEYS}
    model.train()
    model._bind()
    assert rec.calls[-1] == {"lateral": 0.0, "longitudinal": 0.0, "height": 0.0, "rotation": 0.0, "index": -1.0}


@needs_reference
def test_plugin_forwards_the_reference_dict(plugin, monkeypatch):  # noqa: F811
    """B200NeuRADModel reads the reference model's own dynamic_actors.actor_editing at render time: the dict the viewer
    sliders' callbacks and ADPipeline._update_actor_fids write.  Training mode sends no edit."""
    from neurad_studio_b200 import nerfstudio_api
    from tests.fake_backend import FakeBackend
    from tests.test_reference_plugin import _build_model

    be = FakeBackend()
    rec = _EditRecorder()
    be.set_actor_edit = rec
    monkeypatch.setattr(nerfstudio_api, "get_backend", lambda device: be)
    model, _, _ = _build_model(plugin, n_actors=3)
    model.eval()
    da = model.dynamic_actors
    da.actor_lateral_shift.cb_hook(type("Slider", (), {"value": 1.5})())  # the viewer slider's callback
    da.actor_editing.update({"rotation": -0.25, "index": 2})
    model._b200_bind()
    assert rec.calls[-1] == {"lateral": 1.5, "longitudinal": 0.0, "height": 0.0, "rotation": -0.25, "index": 2}
    model.train()
    model._b200_bind()
    assert rec.calls[-1] == {"lateral": 0.0, "longitudinal": 0.0, "height": 0.0, "rotation": 0.0, "index": -1.0}


def test_backend_sends_only_changes():
    from neurad_studio_b200.backend import B200Backend

    class Lib:
        def __init__(self):
            self.calls = []

        def b200nerf_set_actor_edit(self, h, *a):
            self.calls.append(a)
            return 0

    be = B200Backend.__new__(B200Backend)
    be.lib, be._h, be.cfg = Lib(), None, type("Cfg", (), {"n_actors": 3})()
    be.set_actor_edit()  # the defaults: nothing to send
    be.set_actor_edit(lateral=1.0, index=2)
    be.set_actor_edit(lateral=1.0, index=2.0)
    assert be.lib.calls == [(1.0, 0.0, 0.0, 0.0, 2.0)] and be.actor_edit_active
    be.set_actor_edit(height=0.5)  # a height alone is no edit, but it is a change of state
    assert be.lib.calls[-1] == (0.0, 0.0, 0.5, 0.0, -1.0) and not be.actor_edit_active


def test_autograd_refuses_edited_forward():
    from neurad_studio_b200 import autograd as AG

    class Ctx:
        edited = True

    with pytest.raises(RuntimeError, match="actor edit"):
        AG._refuse_edited(Ctx())
    Ctx.edited = False
    AG._refuse_edited(Ctx())
