"""CPU-side checks of the ensemble scorer: the public import, the argument validation of `ab_ensemble_score_fields`
and its workspace query (which needs no GPU because it happens before any launch), the input checks of
`EnsembleScorer.step` and the schema of an empty result."""

import ctypes as C
from datetime import timedelta

import numpy as np
import pytest

from aurora_b200 import cabi
from aurora_b200.batch import Batch, Metadata
from tests import fixtures as fx

FAKE = 0x1000  # a non-null, 16-byte aligned pointer; validation fails before anything could dereference it


def test_public_import():
    from aurora_b200 import EnsembleScorer  # noqa: F401

    import aurora_b200

    assert "EnsembleScorer" in aurora_b200.__all__


def _field(m=8, **kw):
    f = cabi.AbEnsembleField(truth=FAKE, clim=FAKE, n_members=m, h=16, w=32, ld_member=32, ld_truth=32, ld_clim=32,
                             levels=13, member_level_stride=512, truth_level_stride=512, clim_level_stride=512)
    for k in range(m):
        f.members[k] = FAKE + 16 * 4096 * k
    for k, v in kw.items():
        setattr(f, k, v)
    return f


def _call(fields, field_bytes=None, weights=FAKE, sums=FAKE, workspace=FAKE, workspace_bytes=1 << 30):
    lib = cabi.lib()
    arr = (cabi.AbEnsembleField * max(len(fields), 1))(*fields)
    size = C.sizeof(cabi.AbEnsembleField) if field_bytes is None else field_bytes
    status = lib.ab_ensemble_score_fields(arr, len(fields), C.c_size_t(size), C.c_void_p(weights), C.c_void_p(sums),
                                          C.c_void_p(workspace), C.c_size_t(workspace_bytes), None)
    return status, lib.ab_last_error().decode()


def _query(fields, field_bytes=None):
    lib = cabi.lib()
    arr = (cabi.AbEnsembleField * max(len(fields), 1))(*fields)
    size = C.sizeof(cabi.AbEnsembleField) if field_bytes is None else field_bytes
    n = C.c_size_t()
    status = lib.ab_ensemble_score_workspace_bytes(arr, len(fields), C.c_size_t(size), C.byref(n))
    return status, lib.ab_last_error().decode()


def test_descriptor_size_and_constants():
    assert C.sizeof(cabi.AbEnsembleField) == 64 * 8 + 2 * 8 + 3 * 8 + 7 * 4 + 4
    assert (cabi.AB_ENS_MAX_MEMBERS, cabi.AB_ENS_MAX_FIELDS, cabi.AB_ENS_SUMS) == (64, 16, 10)
    for name in ("ab_ensemble_score_workspace_bytes", "ab_ensemble_score_fields"):
        assert name in cabi.EXPORTS and hasattr(cabi.lib(), name)


def test_rejects_null_pointers():
    for kw in ({"weights": None}, {"sums": None}, {"workspace": None}):
        status, msg = _call([_field()], **kw)
        assert status == -1 and "null argument" in msg, kw
    f = _field()
    f.members[5] = None
    for bad in (f, _field(truth=None)):
        for status, msg in (_call([bad]), _query([bad])):
            assert status == -1 and "field 0: null member or truth" in msg
    f = _field(m=3)
    f.members[3] = None  # past n_members: unused
    assert _query([f])[0] == 0
    lib = cabi.lib()
    assert lib.ab_ensemble_score_fields(None, 1, C.c_size_t(C.sizeof(cabi.AbEnsembleField)), C.c_void_p(FAKE),
                                        C.c_void_p(FAKE), C.c_void_p(FAKE), C.c_size_t(1 << 30), None) == -1
    assert "null argument" in lib.ab_last_error().decode()
    arr = (cabi.AbEnsembleField * 1)(_field())
    assert lib.ab_ensemble_score_workspace_bytes(arr, 1, C.c_size_t(C.sizeof(cabi.AbEnsembleField)), None) == -1
    assert "null argument" in lib.ab_last_error().decode()


def test_checks_the_descriptor_size_and_count():
    for check in (_call, _query):
        status, msg = check([_field()], field_bytes=C.sizeof(cabi.AbEnsembleField) - 8)
        assert status == -1 and "sizeof(AbEnsembleField)" in msg
        status, msg = check([_field()] * (cabi.AB_ENS_MAX_FIELDS + 1))
        assert status == -3 and "at most 16 are supported" in msg
    assert _query([_field()] * cabi.AB_ENS_MAX_FIELDS)[0] == 0
    assert _call([], weights=None, sums=None, workspace=None)[0] == 0  # an empty list is a no-op
    assert cabi.ensemble_score_workspace_bytes([]) == 0


@pytest.mark.parametrize("m", [-1, 0, 1, 65, 1000])
def test_rejects_member_counts_outside_2_to_64(m):
    f = _field(m=8, n_members=m)
    for status, msg in (_call([_field(), f]), _query([_field(), f])):
        if m < 2:
            assert status == -1 and f"field 1: {m} members, an ensemble needs at least 2" in msg
        else:
            assert status == -3 and f"field 1: {m} members, at most 64 are supported" in msg
    assert _query([_field(m=2)])[0] == 0 and _query([_field(m=64)])[0] == 0


def test_rejects_bad_extents_pitches_and_strides():
    for kw in ({"h": 0}, {"w": 0}, {"levels": 0}, {"h": -3}):
        for status, msg in (_call([_field(), _field(**kw)]), _query([_field(), _field(**kw)])):
            assert status == -1 and "field 1: bad extent" in msg, kw
    for kw in ({"ld_member": 31}, {"ld_truth": 16}, {"ld_clim": 0}):
        for status, msg in (_call([_field(**kw)]), _query([_field(**kw)])):
            assert status == -1 and "row pitch smaller than the width" in msg, kw
    assert cabi.ensemble_score_workspace_bytes([_field(clim=None, ld_clim=0)]) > 0  # no climatology: pitch unused
    for kw in ({"member_level_stride": -512}, {"truth_level_stride": -1}, {"clim_level_stride": -4}):
        for status, msg in (_call([_field(**kw)]), _query([_field(**kw)])):
            assert status == -1 and "negative level stride" in msg, kw


def test_rejects_a_small_workspace():
    fields = [_field(), _field(m=50, h=721, w=1440, ld_member=1440, ld_truth=1440, ld_clim=1440, levels=1)]
    need = cabi.ensemble_score_workspace_bytes(fields)
    # 13 planes of 16 x 32 are one work item each; at M = 50 a work item is 262144 // 52 // 1440 = 3 rows of 1440
    assert need == (13 + -(-721 // 3)) * 10 * 8
    status, msg = _call(fields, workspace_bytes=need - 1)
    assert status == -1 and f"workspace of {need - 1} bytes, {need} needed" in msg
    status, msg = _call(fields, sums=FAKE + 4)
    assert status == -1 and "8-byte aligned" in msg
    with pytest.raises(cabi.AbError, match="field 0: bad extent"):
        cabi.ensemble_score_workspace_bytes([_field(w=0)])


# ---- EnsembleScorer.step refusals -------------------------------------------------------------------------------------
def _batch(h=16, w=32, b=1, levels=fx.LEVELS4, seed=0):
    return fx.make_batch(fx.CONFIGS["tiny"], h, w, levels=levels, b=b, seed=seed)


def _restamp(x: Batch, time=None, lat=None, lon=None, levels=None, step=None) -> Batch:
    md = x.metadata
    return Batch(x.surf_vars, x.static_vars, x.atmos_vars,
                 Metadata(md.lat if lat is None else lat, md.lon if lon is None else lon,
                          md.time if time is None else time, md.atmos_levels if levels is None else levels,
                          md.rollout_step if step is None else step))


def _member(seed=0, b=1, levels=fx.LEVELS4):
    """A CPU batch shaped like a prediction (one history slice), every entry valid at the same time."""
    x = _batch(b=b, levels=levels, seed=seed)
    one = lambda d: {k: v[:, -1:] for k, v in d.items()}  # noqa: E731
    return _restamp(Batch(one(x.surf_vars), x.static_vars, one(x.atmos_vars), x.metadata),
                    time=(x.metadata.time[0],) * b)


def _truth(seed=9, **kw):
    return _restamp(_batch(seed=seed), **kw)


def test_step_refuses_one_member_or_too_many():
    from aurora_b200 import EnsembleScorer

    sc = EnsembleScorer()
    with pytest.raises(ValueError, match="needs at least 2 members, got 1"):
        sc.step(_member(), _truth())
    with pytest.raises(ValueError, match="needs at least 2 members, got 1"):
        sc.step([_member()], _truth())
    with pytest.raises(ValueError, match="needs at least one Batch"):
        sc.step([], _truth())
    with pytest.raises(ValueError, match="scores at most 64 members, got 65"):
        sc.step([_member(b=64), _member(seed=1)], _truth())


def test_step_refuses_cpu_members_and_float64_fields():
    from aurora_b200 import EnsembleScorer

    with pytest.raises(cabi.AbError, match="needs the member on a CUDA device"):
        EnsembleScorer().step([_member(0), _member(1)], _truth())
    with pytest.raises(cabi.AbError, match="needs the member on a CUDA device"):
        EnsembleScorer().step(_member(b=4), _truth())
    t = _truth()  # a float64 member is refused on the GPU (tests/test_ensemble_scorer_gpu.py)
    t.surf_vars["msl"] = t.surf_vars["msl"].double()
    with pytest.raises(TypeError, match="needs float32 fields, the truth has torch.float64"):
        EnsembleScorer().step([_member(0), _member(1)], t)


def test_step_refuses_members_that_disagree():
    from aurora_b200 import EnsembleScorer

    sc, a = EnsembleScorer(), _member(0)
    t0 = a.metadata.time[0]
    with pytest.raises(ValueError, match="the members are valid at different times"):
        sc.step([a, _restamp(_member(1), time=(t0 + timedelta(hours=6),))], _truth())
    with pytest.raises(ValueError, match="the members are valid at different times"):
        sc.step(_restamp(_member(b=2), time=(t0, t0 + timedelta(hours=6))), _truth())
    with pytest.raises(ValueError, match="members differ in rollout_step: 0 and 2"):
        sc.step([a, _restamp(_member(1), step=2)], _truth())
    with pytest.raises(ValueError, match="members differ in grid"):
        sc.step([a, _restamp(_member(1), lat=a.metadata.lat * 0.5)], _truth())
    with pytest.raises(ValueError, match="members differ in grid"):
        sc.step([a, _restamp(_member(1), lon=a.metadata.lon + 1.0)], _truth())
    with pytest.raises(ValueError, match="members differ in levels"):
        sc.step([a, _member(1, levels=(100, 250, 500, 1000))], _truth())
    b = _member(1)
    del b.surf_vars["msl"]
    with pytest.raises(ValueError, match="members differ in variables"):
        sc.step([a, b], _truth())


def test_step_refuses_truths_and_climatologies_that_do_not_fit():
    from aurora_b200 import EnsembleScorer

    ens = [_member(0), _member(1)]
    t0 = ens[0].metadata.time[0]
    with pytest.raises(ValueError, match="the truth is valid at"):
        EnsembleScorer().step(ens, _truth(time=(t0 + timedelta(hours=6),)))
    two = _restamp(_batch(b=2, seed=3), time=(t0, t0))
    with pytest.raises(ValueError, match=r"needs a truth of batch size 1, it has \[2\]"):
        EnsembleScorer().step(ens, two)
    with pytest.raises(ValueError, match=r"needs a climatology of batch size 1, it has \[2\]"):
        EnsembleScorer(climatology=two).step(ens, _truth())
    with pytest.raises(ValueError, match=r"the truth lacks the pressure levels \[500\]"):
        EnsembleScorer().step(ens, _restamp(_batch(levels=(100, 250, 850), seed=1), time=(t0,)))
    with pytest.raises(ValueError, match="the climatology's latitudes differ"):
        EnsembleScorer(climatology=_truth(lat=ens[0].metadata.lat * 0.5)).step(ens, _truth())


def test_step_refuses_2d_coordinates_and_sharded_bands():
    from aurora_b200 import EnsembleScorer

    ens, truth = [_member(0), _member(1)], _truth()
    md = ens[1].metadata
    lat2, lon2 = np.meshgrid(md.lat.numpy(), md.lon.numpy(), indexing="ij")
    import torch

    flat = Batch(ens[1].surf_vars, ens[1].static_vars, ens[1].atmos_vars,
                 Metadata.derived(torch.from_numpy(lat2), torch.from_numpy(lon2), md.time, md.atmos_levels))
    with pytest.raises(ValueError, match="1-D latitudes and longitudes"):
        EnsembleScorer().step([ens[0], flat], truth)
    ens[1].slab_plans = [object()]
    with pytest.raises(ValueError, match="needs a whole-grid member; gather the latitude bands first"):
        EnsembleScorer().step(ens, truth)


def test_empty_results_schema():
    from aurora_b200 import EnsembleScorer
    from aurora_b200.scorer import ENSEMBLE_COLUMNS

    df = EnsembleScorer().results()
    assert tuple(df.columns) == ENSEMBLE_COLUMNS == (
        "time", "rollout_step", "variable", "level", "members", "ens_rmse", "ens_bias", "spread", "ssr", "crps",
        "crps_skill", "crps_spread", "acc", "count")
    assert len(df) == 0
    assert str(df["time"].dtype) == "datetime64[ns]"
    assert [str(df[c].dtype) for c in ("rollout_step", "members", "count")] == ["int64"] * 3
    assert all(df[c].dtype == np.float64 for c in ("level", "ens_rmse", "ens_bias", "spread", "ssr", "crps",
                                                   "crps_skill", "crps_spread", "acc"))
