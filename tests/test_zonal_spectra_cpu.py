"""CPU-side checks of the zonal spectra: the public import, the argument validation of `ab_zonal_spectra` and its
workspace query (which needs no GPU because it happens before any launch), the input checks of `ZonalSpectra` and
its `step`, and the schema of an empty result."""

import ctypes as C

import numpy as np
import pytest
import torch

from aurora_b200 import cabi
from aurora_b200.batch import Batch, Metadata
from tests import fixtures as fx

FAKE = 0x1000  # a non-null, 16-byte aligned pointer; validation fails before anything could dereference it


def test_public_import():
    from aurora_b200 import ZonalSpectra  # noqa: F401

    import aurora_b200

    assert "ZonalSpectra" in aurora_b200.__all__


def _field(**kw):
    f = cabi.AbSpectrumField(x=FAKE, level_stride=16 * 32, h=16, w=32, ld=32, levels=13)
    for k, v in kw.items():
        setattr(f, k, v)
    return f


def _rows(bands):
    return (C.c_int32 * (2 * max(len(bands), 1)))(*(r for b in bands for r in b))


def _call(fields, bands=((0, 16),), field_bytes=None, weights=FAKE, out=FAKE, workspace=FAKE,
          workspace_bytes=1 << 30, band_rows=True):
    lib = cabi.lib()
    arr = (cabi.AbSpectrumField * max(len(fields), 1))(*fields)
    size = C.sizeof(cabi.AbSpectrumField) if field_bytes is None else field_bytes
    status = lib.ab_zonal_spectra(arr, len(fields), C.c_size_t(size), _rows(bands) if band_rows else None,
                                  len(bands), C.c_void_p(weights), C.c_void_p(out), C.c_void_p(workspace),
                                  C.c_size_t(workspace_bytes), None)
    return status, lib.ab_last_error().decode()


def _query(fields, bands=((0, 16),), field_bytes=None, band_rows=True):
    lib = cabi.lib()
    arr = (cabi.AbSpectrumField * max(len(fields), 1))(*fields)
    size = C.sizeof(cabi.AbSpectrumField) if field_bytes is None else field_bytes
    n = C.c_size_t()
    status = lib.ab_zonal_spectra_workspace_bytes(arr, len(fields), C.c_size_t(size),
                                                  _rows(bands) if band_rows else None, len(bands), C.byref(n))
    return status, lib.ab_last_error().decode()


def _both(fields, **kw):
    call_kw = {k: v for k, v in kw.items()}
    query_kw = {k: v for k, v in kw.items() if k in ("bands", "field_bytes", "band_rows")}
    return [_call(fields, **call_kw), _query(fields, **query_kw)]


def test_descriptor_size_and_constants():
    assert C.sizeof(cabi.AbSpectrumField) == 8 + 8 + 4 * 4
    assert (cabi.AB_SPEC_MAX_FIELDS, cabi.AB_SPEC_MAX_BANDS, cabi.AB_SPEC_MAX_WIDTH) == (64, 8, 4096)
    for name in ("ab_zonal_spectra_workspace_bytes", "ab_zonal_spectra"):
        assert name in cabi.EXPORTS and hasattr(cabi.lib(), name)


def test_rejects_null_pointers():
    for kw in ({"weights": None}, {"out": None}, {"workspace": None}):
        status, msg = _call([_field()], **kw)
        assert status == -1 and "null argument" in msg, kw
    for status, msg in _both([_field(x=None)]):
        assert status == -1 and "field 0: null x" in msg
    for status, msg in _both([_field()], band_rows=False):
        assert status == -1 and "null argument" in msg
    lib = cabi.lib()
    assert lib.ab_zonal_spectra(None, 1, C.c_size_t(C.sizeof(cabi.AbSpectrumField)), _rows([(0, 1)]), 1,
                                C.c_void_p(FAKE), C.c_void_p(FAKE), C.c_void_p(FAKE), C.c_size_t(1 << 30), None) == -1
    assert "null argument" in lib.ab_last_error().decode()
    arr = (cabi.AbSpectrumField * 1)(_field())
    assert lib.ab_zonal_spectra_workspace_bytes(arr, 1, C.c_size_t(C.sizeof(cabi.AbSpectrumField)), _rows([(0, 1)]),
                                                1, None) == -1
    assert "null argument" in lib.ab_last_error().decode()


def test_checks_the_descriptor_size_and_count():
    for status, msg in _both([_field()], field_bytes=C.sizeof(cabi.AbSpectrumField) - 4):
        assert status == -1 and "sizeof(AbSpectrumField)" in msg
    for status, msg in _both([_field()] * (cabi.AB_SPEC_MAX_FIELDS + 1)):
        assert status == -3 and "at most 64 are supported" in msg
    assert _query([_field()] * cabi.AB_SPEC_MAX_FIELDS)[0] == 0
    assert _call([], weights=None, out=None, workspace=None)[0] == 0  # an empty list is a no-op
    assert cabi.zonal_spectra_workspace_bytes([], [(0, 1)]) == 0


def test_rejects_bad_extents_pitches_strides_and_mixed_grids():
    for kw in ({"h": 0}, {"w": 0}, {"levels": 0}, {"h": -3}):
        for status, msg in _both([_field(**kw)]):
            assert status == -1 and "field 0: bad extent" in msg, kw
    for status, msg in _both([_field(ld=31)]):
        assert status == -1 and "row pitch 31 smaller than the width 32" in msg
    for status, msg in _both([_field(level_stride=-512)]):
        assert status == -1 and "negative level stride" in msg
    for kw in ({"h": 17}, {"w": 64, "ld": 64}):
        for status, msg in _both([_field(), _field(**kw)]):
            assert status == -1 and "field 1 is" in msg and "one call takes one grid" in msg, kw


@pytest.mark.parametrize("w", [7, 14, 49, 4097, 4100, 5000, 6000, 8192, 1441])
def test_rejects_unsupported_widths(w):
    for status, msg in _both([_field(w=w, ld=w)]):
        assert status == -3 and f"width {w}: supported are widths up to 4096" in msg


@pytest.mark.parametrize("w", [1, 2, 3, 4, 5, 8, 9, 25, 27, 32, 64, 90, 120, 125, 900, 1024, 1440, 2048, 3600, 4000,
                               4096])
def test_accepts_supported_widths(w):
    # one band of 16 rows is one work item of w // 2 + 3 values per plane
    assert cabi.zonal_spectra_workspace_bytes([_field(w=w, ld=w)], [(0, 16)]) == 13 * (w // 2 + 3) * 8


def test_rejects_bad_bands():
    for status, msg in _both([_field()], bands=()):
        assert status == -1 and "n_bands 0 < 1" in msg
    for status, msg in _both([_field()], bands=[(0, 16)] * 9):
        assert status == -3 and "9 bands in one call, at most 8 are supported" in msg
    for bands in ([(5, 4)], [(-1, 3)], [(0, 17)], [(0, 16), (3, 2)]):
        for status, msg in _both([_field()], bands=bands):
            assert status == -1 and "rows [" in msg and "outside [0, 16]" in msg, bands
    assert _query([_field()], bands=[(0, 16)] * 8)[0] == 0


def test_workspace_size_and_small_workspace():
    # 3 bands of 16, 0 and 33 rows: 1 + 0 + 2 work items of 32 rows per plane
    fields = [_field(), _field(levels=1)]
    bands = [(0, 16), (4, 4), (0, 16)]
    need = cabi.zonal_spectra_workspace_bytes(fields, bands)
    assert need == 14 * 2 * (32 // 2 + 3) * 8
    big = [_field(h=721, w=1440, ld=1440, levels=1)]
    assert cabi.zonal_spectra_workspace_bytes(big, [(0, 721)]) == 23 * 723 * 8
    status, msg = _call(fields, bands=bands, workspace_bytes=need - 1)
    assert status == -1 and f"workspace of {need - 1} bytes, {need} needed" in msg
    status, msg = _call(fields, bands=bands, out=FAKE + 4)
    assert status == -1 and "8-byte aligned" in msg
    with pytest.raises(cabi.AbError, match="field 0: bad extent"):
        cabi.zonal_spectra_workspace_bytes([_field(w=0)], [(0, 1)])


# ---- ZonalSpectra refusals ------------------------------------------------------------------------------------------
def _batch(h=16, w=32, b=1, seed=0, lat=None, lon=None):
    x = fx.make_batch(fx.CONFIGS["tiny"], h, w, levels=fx.LEVELS4, b=b, seed=seed)
    md = x.metadata
    # `derived` skips Metadata's own coordinate checks, as coordinates that went through a rollout do
    return Batch(x.surf_vars, x.static_vars, x.atmos_vars,
                 Metadata.derived(md.lat if lat is None else lat, md.lon if lon is None else lon, md.time,
                                  md.atmos_levels, md.rollout_step))


def test_constructor_refuses_bad_bands():
    from aurora_b200 import ZonalSpectra

    assert ZonalSpectra().bands == {"global": (-90.0, 90.0)}
    assert len(ZonalSpectra(bands={str(i): (-10, 10) for i in range(8)}).bands) == 8
    with pytest.raises(ValueError, match="at most 8 bands, got 9"):
        ZonalSpectra(bands={str(i): (-10, 10) for i in range(9)})
    with pytest.raises(ValueError, match="non-empty dict"):
        ZonalSpectra(bands={})
    for band in ((20, -20), (-91, 0), (0, 90.5), (-100, -95)):
        with pytest.raises(ValueError, match=r"needs -90 <= lo <= hi <= 90"):
            ZonalSpectra(bands={"b": band})


def test_step_refuses_cpu_tensors_and_non_float32_fields():
    from aurora_b200 import ZonalSpectra

    with pytest.raises(cabi.AbError, match="needs the batch on a CUDA device"):
        ZonalSpectra().step(_batch())
    x = _batch()
    x.surf_vars["msl"] = x.surf_vars["msl"].double()
    with pytest.raises(cabi.AbError, match="needs the batch on a CUDA device"):  # the device is checked first
        ZonalSpectra().step(x)
    x = _batch()  # a non-float32 field on the GPU is refused there (tests/test_zonal_spectra_gpu.py)
    with pytest.raises(TypeError, match="needs a str label, got int"):
        ZonalSpectra().step(x, label=3)
    with pytest.raises(TypeError, match="needs a str label, got NoneType"):
        ZonalSpectra().step(x, label=None)


def test_step_refuses_2d_coordinates_and_sharded_bands():
    from aurora_b200 import ZonalSpectra

    x = _batch()
    md = x.metadata
    lat2, lon2 = np.meshgrid(md.lat.numpy(), md.lon.numpy(), indexing="ij")
    flat = Batch(x.surf_vars, x.static_vars, x.atmos_vars,
                 Metadata.derived(torch.from_numpy(lat2), torch.from_numpy(lon2), md.time, md.atmos_levels))
    with pytest.raises(ValueError, match="1-D latitudes and longitudes"):
        ZonalSpectra().step(flat)
    x.slab_plans = [object()]
    with pytest.raises(ValueError, match="needs a whole-grid batch; gather the latitude bands first"):
        ZonalSpectra().step(x)


def _grid_error(lat=None, lon=None, w=32):
    from aurora_b200 import ZonalSpectra

    with pytest.raises(ValueError) as e:
        ZonalSpectra()._grid(_batch(w=w, lat=lat, lon=lon))
    return str(e.value)


def test_step_refuses_grids_the_kernel_does_not_take():
    lat = torch.linspace(90, -90, 16)
    for bad in (lat.flip(0).roll(1), torch.cat([lat[:8], lat[7:15]]), torch.zeros(16)):
        assert "strictly monotonic latitudes" in _grid_error(lat=bad)
    lon = torch.linspace(0, 360, 33)[:-1]
    for bad in (lon.flip(0), lon * 0.5, torch.cat([lon[:-1], lon[-1:] + 0.02]), torch.linspace(0, 360, 32)):
        assert "32 longitudes equally spaced by 11.25 degrees" in _grid_error(lon=bad)
    for w in (7, 4097, 4116):
        assert f"no prime factor above 5; this one has {w}" in _grid_error(lon=torch.linspace(0, 360, w + 1)[:-1],
                                                                          w=w)


def test_grid_accepts_the_supported_grids_and_labels_wavelengths():
    from aurora_b200 import ZonalSpectra

    sp = ZonalSpectra(bands={"global": (-90, 90), "tropics": (-20, 20), "nh": (20, 90), "none": (0.1, 0.2)})
    for w in (1440, 3600, 900, 32, 64, 90, 120):
        lon = torch.linspace(0, 360, w + 1)[:-1] if w != 3600 else torch.arange(3600) * 0.1 - 180  # float32 0.1 deg
        lat = torch.linspace(90, -90, 721) if w == 1440 else torch.linspace(-89.5, 89.5, 10)
        md = Metadata.derived(lat, lon, (fx.make_batch(fx.CONFIGS["tiny"], 4, 4, b=1).metadata.time[0],), (100,))
        rows, wl = sp._grid(Batch({}, {}, {}, md))
        assert wl.shape == (4, w // 2 + 1)
        assert np.isinf(wl[:3, 0]).all() and np.isnan(wl[3]).all()
        if w == 1440:
            assert rows == [(0, 721), (280, 441), (0, 281), (0, 0)]  # lat = 90 - 0.25 r, inclusive ends
            cos = np.cos(np.deg2rad(np.linspace(90, -90, 721)))
            assert wl[0, 1] == pytest.approx(2 * np.pi * 6371 * (cos ** 2).sum() / cos.sum())
            assert wl[1, 1] > wl[0, 1] > wl[2, 1]


def test_empty_results_schema():
    from aurora_b200 import ZonalSpectra
    from aurora_b200.spectra import COLUMNS

    df = ZonalSpectra().results()
    assert tuple(df.columns) == COLUMNS == (
        "time", "rollout_step", "label", "member", "variable", "level", "band", "wavenumber", "wavelength_km",
        "power", "rows")
    assert len(df) == 0
    assert str(df["time"].dtype) == "datetime64[ns]"
    assert [str(df[c].dtype) for c in ("rollout_step", "member", "wavenumber", "rows")] == ["int64"] * 4
    assert all(df[c].dtype == np.float64 for c in ("level", "wavelength_km", "power"))
    assert [str(df[c].dtype) for c in ("label", "variable", "band")] == ["category"] * 3
