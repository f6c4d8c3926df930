"""CPU-side checks of the cyclone tracker: the public import, the argument validation of `ab_track_boxes` (which
needs no GPU because it happens before any launch) and the input checks of `Tracker.step`."""

import ctypes as C
from datetime import datetime

import pytest
import torch

from aurora_b200 import cabi
from aurora_b200.batch import Batch, Metadata
from tests import fixtures as fx

FAKE = 0x1000  # a non-null pointer; validation fails before anything could dereference it


def test_public_import():
    from aurora_b200 import Aurora, Batch, Tracker, rollout  # noqa: F401

    import aurora_b200

    assert "Tracker" in aurora_b200.__all__


def _box(**kw):
    b = cabi.AbTrackBox(plane=FAKE, h=64, w=128, ld=128, op=cabi.AB_TRACK_MAX, rows_off=0, n_rows=3, cols_off=3, n_cols=3)
    for k, v in kw.items():
        setattr(b, k, v)
    return b


def _call(boxes, box_bytes=None, index=FAKE, values=FAKE, counts=FAKE, masks=FAKE):
    lib = cabi.lib()
    arr = (cabi.AbTrackBox * max(len(boxes), 1))(*boxes)
    size = C.sizeof(cabi.AbTrackBox) if box_bytes is None else box_bytes
    status = lib.ab_track_boxes(arr, len(boxes), C.c_size_t(size), C.c_void_p(index), C.c_void_p(values),
                                C.c_void_p(counts), C.c_void_p(masks), None)
    return status, lib.ab_last_error().decode()


def test_track_boxes_rejects_null_pointers():
    assert _call([_box()], index=None)[0] == -1
    status, msg = _call([_box()], values=None)
    assert status == -1 and "null argument" in msg
    status, msg = _call([_box(plane=None)])
    assert status == -1 and "null plane" in msg
    status, msg = _call([_box(op=cabi.AB_TRACK_WINDMAX)])
    assert status == -1 and "plane2" in msg
    status, msg = _call([_box(op=cabi.AB_TRACK_MINIMA)], masks=None)
    assert status == -1 and "masks" in msg


def test_track_boxes_rejects_oversized_boxes():
    status, msg = _call([_box(n_rows=cabi.AB_TRACK_MAX_SIDE + 1)])
    assert status == -3 and "101 x 101" in msg
    status, _ = _call([_box(n_cols=cabi.AB_TRACK_MAX_SIDE + 1)])
    assert status == -3
    status, msg = _call([_box()] * (cabi.AB_TRACK_MAX_BOXES + 1))
    assert status == -3 and "at most 32" in msg


def test_track_boxes_rejects_unknown_operations_and_bad_lists():
    status, msg = _call([_box(), _box(op=7)])
    assert status == -1 and "box 1: unknown operation 7" in msg
    status, msg = _call([_box(n_rows=0)])
    assert status == -1 and "bad index lists" in msg
    status, msg = _call([_box(ld=100)])
    assert status == -1 and "bad plane extent" in msg


def test_track_boxes_checks_the_descriptor_size():
    status, msg = _call([_box()], box_bytes=C.sizeof(cabi.AbTrackBox) - 8)
    assert status == -1 and "sizeof(AbTrackBox)" in msg
    assert _call([])[0] == 0  # an empty list is a no-op


def _batch(b=1, levels=fx.LEVELS13):
    return fx.make_batch(fx.CONFIGS["tiny"], 16, 32, levels=levels, b=b)


def test_step_refuses_cpu_batches():
    from aurora_b200 import Tracker

    with pytest.raises(cabi.AbError, match="needs the prediction on a CUDA device"):
        Tracker(10.0, 20.0, datetime(2020, 6, 1)).step(_batch())


def test_step_refuses_batch_size_two():
    from aurora_b200 import Tracker

    with pytest.raises(RuntimeError, match="^Predictions don't have batch size one.$"):
        Tracker(10.0, 20.0, datetime(2020, 6, 1)).step(_batch(b=2))


def test_step_needs_700_hpa_1d_coordinates_and_whole_grids():
    from aurora_b200 import Tracker

    tr = Tracker(10.0, 20.0, datetime(2020, 6, 1))
    with pytest.raises(ValueError, match="700 is not in list"):
        tr.step(_batch(levels=fx.LEVELS4))
    b = _batch()
    lat2, lon2 = torch.meshgrid(b.metadata.lat, b.metadata.lon, indexing="ij")
    b2 = Batch(b.surf_vars, b.static_vars, b.atmos_vars,
               Metadata.derived(lat2, lon2, b.metadata.time, b.metadata.atmos_levels))
    with pytest.raises(ValueError, match="1-D latitudes and longitudes"):
        tr.step(b2)
    b.slab_plans = [object()]
    with pytest.raises(ValueError, match="gather the latitude bands first"):
        tr.step(b)
    assert tr.fails == 0 and len(tr.tracked_lats) == 1
