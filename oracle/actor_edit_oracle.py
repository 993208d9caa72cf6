"""TEST INFRASTRUCTURE ONLY -- CPU oracle of NeuRAD's actor edits (DynamicActors.actor_editing).

``DynamicActors.get_boxes2world`` (model_components/dynamic_actors.py:251-268) passes the interpolated box poses through
``edit_boxes2world`` (:181-249) in eval mode.  ``edit_boxes2world`` below restates that edit for the flatten=False branch
NeuRAD's encodings use, with the reference's torch op sequence (so it reproduces the reference bit for bit on a CPU, which
oracle/make_golden_actor_edits.py asserts).  ``nff_outputs`` renders an edited scene by applying it at the same place
the reference does, to every pose oracle/neurad_oracle.py's ``boxes2world_at`` returns, and is otherwise that oracle.
"""
from __future__ import annotations

import math
from contextlib import contextmanager
from typing import Optional

import torch
from torch import Tensor

from . import neurad_oracle as O

NO_EDIT = {"lateral": 0.0, "longitudinal": 0.0, "rotation": 0.0, "index": -1.0, "height": 0.0}


def edit_boxes2world(b2w: Tensor, edit: Optional[dict]) -> Tensor:
    """b2w [Q,A,3,4] (box -> world), `edit` the actor_editing dict (None: no edit).  Only longitudinal, lateral and rotation
    decide whether anything is edited (a height alone is ignored); index -1 selects every actor, otherwise the torch.int
    tensor [min(index, A - 1)] indexes the actor axis.  The shift is in the box frame with the unedited rotation; the yaw
    multiplies from the left."""
    if edit is None or (edit["longitudinal"] == 0.0 and edit["lateral"] == 0.0 and edit["rotation"] == 0.0):
        return b2w
    n = b2w.shape[1]
    sel = torch.arange(n) if edit["index"] == -1.0 else torch.tensor([min(edit["index"], n - 1)], dtype=torch.int)
    b2w = b2w.clone()
    shift = torch.tensor([edit["lateral"], edit["longitudinal"], edit["height"], 1.0])
    b2w[:, sel, :, 3] = b2w[:, sel] @ shift
    r = edit["rotation"]
    if r != 0.0:
        yaw = torch.tensor([[math.cos(r), -math.sin(r), 0.0], [math.sin(r), math.cos(r), 0.0], [0.0, 0.0, 1.0]])
        b2w[:, sel, :3, :3] = yaw @ b2w[:, sel, :3, :3]
    return b2w


@contextmanager
def edited_boxes(edit: Optional[dict]):
    """Within the block, neurad_oracle's box poses are the edited ones (the reference's eval-mode get_boxes2world)."""
    orig = O.boxes2world_at

    def boxes2world_at(params, query_times):
        b2w, valid = orig(params, query_times)  # [Q,A,4,4]
        out = b2w.clone()
        out[..., :3, :] = edit_boxes2world(b2w[..., :3, :], None if edit is None else {**NO_EDIT, **edit})
        return out, valid

    O.boxes2world_at = boxes2world_at
    try:
        yield
    finally:
        O.boxes2world_at = orig


def nff_outputs(params, cfg, *args, edit: Optional[dict] = None, **kw):
    """neurad_oracle.nff_outputs (get_nff_outputs, eval) of the scene with the actor edit `edit` applied."""
    with edited_boxes(edit):
        return O.nff_outputs(params, cfg, *args, **kw)
