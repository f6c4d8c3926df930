"""Golden data for the host-side tests that compare with the UNMODIFIED reference classes (`aurora.Batch`,
`aurora.normalisation`, `aurora.model.swin3d`): run the reference once on the deterministic inputs of the tests
(tests/reference_cases.py) and store what they compare against.  Needs a reference checkout on the path:

    PYTHONPATH=<reference checkout>:tests/_shims:. python tests/golden/make_reference_golden.py

Outputs
    normalisation_ref.json   the reference's per-variable locations / scales
    batch_ref.npz            normalise / normalise + unnormalise / crop(3) of the `tiny_air` batch (16 x 30, 13 levels)
    regrid_ref.npz           Batch.regrid of the `tiny` batch (17 x 32, b = 2) to 5.0 / 11.25 / 7.3 degrees
                             (both: coordinates in full, fields on the fixed sub-grid `reference_cases.sample`)
    windows_ref.json         SHA-256 of the window gather indices (int32), of the mask group ids (uint8) and of the
                             additive mask tensor (float32) of 4 x 30 random geometries
"""

import json
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))

import aurora  # noqa: E402  (the reference)
from aurora import normalisation as rn  # noqa: E402
from aurora.model import swin3d as ref  # noqa: E402
from aurora.model.util import maybe_adjust_windows  # noqa: E402

from tests import reference_cases as rc  # noqa: E402


def to_ref(b):
    return aurora.Batch(dict(b.surf_vars), dict(b.static_vars), dict(b.atmos_vars),
                        aurora.Metadata(lat=b.metadata.lat, lon=b.metadata.lon, time=b.metadata.time,
                                        atmos_levels=b.metadata.atmos_levels))


def flat(tag, rb, out):
    out[f"{tag}/shape"] = np.array(rb.spatial_shape)
    out[f"{tag}/lat"] = rb.metadata.lat.numpy()
    out[f"{tag}/lon"] = rb.metadata.lon.numpy()
    for grp in ("surf_vars", "static_vars", "atmos_vars"):
        out[f"{tag}/{grp}"] = np.array(list(getattr(rb, grp)))
        for k, v in getattr(rb, grp).items():
            out[f"{tag}/{grp}/{k}"] = rc.sample(v).numpy()


def main():
    (HERE / "normalisation_ref.json").write_text(json.dumps(
        {"locations": {k: float(v) for k, v in rn.locations.items()},
         "scales": {k: float(v) for k, v in rn.scales.items()}}, indent=0, sort_keys=True) + "\n")

    out = {}
    rb = to_ref(rc.batch_case())
    flat("normalise", rb.normalise(surf_stats={}), out)
    flat("roundtrip", rb.normalise(surf_stats={}).unnormalise(surf_stats={}), out)
    flat("crop3", rb.crop(3), out)
    np.savez_compressed(HERE / "batch_ref.npz", **out)

    out = {}
    rb = to_ref(rc.regrid_case())
    for res in rc.REGRID_RES:
        flat(str(res), rb.regrid(res), out)
    np.savez_compressed(HERE / "regrid_ref.npz", **out)

    out = {}
    for chunk in range(rc.WINDOW_CHUNKS):
        for i, (res, shifted, warped) in enumerate(rc.window_geometries(chunk)):
            c, h, w = res
            ss0 = tuple(s // 2 for s in rc.WS0) if shifted else (0, 0, 0)
            ws, ss = maybe_adjust_windows(rc.WS0, ss0, res)
            x = (torch.arange(c * h * w, dtype=torch.float64) + 1).view(1, c, h, w, 1)
            if any(ss):
                x = torch.roll(x, shifts=(-ss[0], -ss[1], -ss[2]), dims=(1, 2, 3))
            x = ref.pad_3d(x, ((-c) % ws[0], (-h) % ws[1], (-w) % ws[2]))
            idx = ref.window_partition_3d(x, ws).reshape(-1, ws[0] * ws[1] * ws[2]).long().numpy() - 1
            out[f"{chunk}/{i}/idx"] = rc.sha(idx.astype(np.int32))
            if any(ss):
                ref.compute_3d_shifted_window_mask.cache_clear()
                try:
                    mask, img = ref.compute_3d_shifted_window_mask(c, h, w, ws, ss, torch.device("cpu"), torch.float32, warped)
                except RuntimeError:  # the reference's own `.view` fails on some degenerate grids (swin3d.py:355)
                    out[f"{chunk}/{i}/mask_fails"] = True
                    continue
                grp = ref.window_partition_3d(img, ws).reshape(-1, ws[0] * ws[1] * ws[2]).to(torch.uint8).numpy()
                out[f"{chunk}/{i}/grp"] = rc.sha(grp)
                out[f"{chunk}/{i}/mask"] = rc.sha(mask.contiguous().numpy())
    (HERE / "windows_ref.json").write_text(json.dumps(out, indent=0, sort_keys=True) + "\n")


if __name__ == "__main__":
    main()
