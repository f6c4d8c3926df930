"""CPU-side checks of the C-ABI library: it builds for sm_90a, loads, exports every symbol that
include/aurora_b200.h declares, validates arguments without touching a GPU, and its window index
arithmetic (one __host__ __device__ routine shared with the attention kernel) is bit-exact against
the reference-derived goldens."""

import ctypes as C
import hashlib
import json
import re
from pathlib import Path

import numpy as np
import pytest

from aurora_b200 import cabi

ROOT = Path(__file__).resolve().parent.parent
GOLD = Path(__file__).parent / "golden"
WS0 = (2, 6, 12)


def test_library_exports_every_declared_symbol():
    header = (ROOT / "include" / "aurora_b200.h").read_text()
    declared = set(re.findall(r"\b(ab_[a-z0-9_]+)\s*\(", header))
    assert declared == set(cabi.EXPORTS), declared ^ set(cabi.EXPORTS)
    lib = cabi.lib()
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.ab_version() == cabi.ABI_VERSION


def test_argument_validation_needs_no_gpu():
    lib = cabi.lib()
    g = cabi.AbGemm()
    assert lib.ab_gemm_bf16(C.byref(g), None) == -1
    assert b"bad shape" in lib.ab_last_error()
    a = cabi.AbWindowAttention()
    assert lib.ab_window_attention(C.byref(a), None) == -1
    with pytest.raises(cabi.AbError):
        cabi.window_geometry((4, 8, 8), (2, 6, 12), (2, 3, 6))  # shift >= window


def test_window_geometry():
    assert cabi.window_geometry((4, 180, 360), WS0, (1, 3, 6)) == (1800, 144, True)
    assert cabi.window_geometry((4, 45, 90), WS0, (0, 0, 0)) == (128, 144, False)
    assert cabi.window_geometry((4, 4, 8), WS0, (1, 3, 6)) == (2, 64, True)  # clamped to (2,4,8), C shift only
    assert cabi.window_geometry((4, 1, 2), WS0, (1, 3, 6)) == (2, 4, True)


def _cases():
    z = np.load(GOLD / "windows.npz")
    return sorted(k[4:] for k in z.files if k.startswith("idx_"))


@pytest.mark.parametrize("tag", _cases())
def test_host_index_map_bit_exact_vs_reference_golden(tag):
    z = np.load(GOLD / "windows.npz")
    dims, sh, wp = tag.split("_")
    res = tuple(int(v) for v in dims.split("x"))
    ss0 = tuple(s // 2 for s in WS0) if sh == "s" else (0, 0, 0)
    idx, grp = cabi.window_index_map_host(res, WS0, ss0, wp == "w")
    np.testing.assert_array_equal(idx, z[f"idx_{tag}"])
    if f"grp_{tag}" in z.files:
        np.testing.assert_array_equal(grp, z[f"grp_{tag}"])


def test_host_index_map_production_checksums():
    hashes = json.loads((GOLD / "windows_hashes.json").read_text())
    for key, want in hashes.items():
        kind, dims, sh, _ = key.split("_")
        res = tuple(int(v) for v in dims.split("x"))
        ss0 = tuple(s // 2 for s in WS0) if sh == "s" else (0, 0, 0)
        idx, grp = cabi.window_index_map_host(res, WS0, ss0, True)
        got = idx if kind == "idx" else grp
        assert hashlib.sha256(got.tobytes()).hexdigest() == want, key


def test_ctypes_mirrors_have_the_library_struct_sizes():
    """Every descriptor struct is mirrored by hand in aurora_b200/cabi.py: its size must equal sizeof() as the library
    was compiled (catches a field added on one side only, or a padding difference)."""
    lib = cabi.lib()
    mirrors = [cabi.AbGemm, cabi.AbWindowAttention, cabi.AbLnModResidual, cabi.AbFieldIn, cabi.AbFieldOut, cabi.AbHaloPush,
               cabi.AbSwinBlock, cabi.AbGemmLn, cabi.AbPatchMergeLn, cabi.AbPatchSplitLn, cabi.AbOp]
    for which, struct in enumerate(mirrors):
        assert lib.ab_struct_size(which) == C.sizeof(struct), (struct.__name__, lib.ab_struct_size(which), C.sizeof(struct))
    assert lib.ab_struct_size(len(mirrors)) == -1


def test_run_ops_validates_without_a_gpu():
    lib = cabi.lib()
    assert lib.ab_run_ops(None, 0, None) == -1
    ops = (cabi.AbOp * 1)()
    ops[0].kind = 99
    assert lib.ab_run_ops(ops, 1, None) == -1 and b"unknown operation kind 99" in lib.ab_last_error()
    assert lib.ab_run_ops(ops, 0, None) == 0   # an empty list is a no-op
