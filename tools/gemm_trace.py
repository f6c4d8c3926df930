"""Phase trace of the wgmma GEMM (gemm_bf16_tn_kernel): where a tile's time goes, per warp role.

    python tools/gemm_trace.py [--source FILE] [--iters N]

1. Builds a copy of the library with `gemm.cu` (or `--source`, e.g. an earlier version of it) compiled twice, with and
   without -DAB_GEMM_TRACE, into build/trace/ (the other objects are the in-tree build's); the in-tree library is not
   touched.  With the switch the kernel sums clock64() cycles per phase in registers and writes one record per CTA.
2. Runs the Swin backbone shapes of the 0.25-degree model at full size on seeded operands, as tools/gemm_shapes.py
   does: qkv / proj / fc1 of stages 1 and 2, stage-1 fc2, stage-3 fc1.
3. Prints one JSON line per shape: ms per launch of the untraced and the traced kernel (the trace's own overhead),
   the effective SM clock (clock64 cycles over %globaltimer ns, per CTA), and per tile in microseconds:
     tile_us          CTA time over the tiles the CTA ran
     producer         empty_bar waits of the TMA producer
     full_first       full_bar wait of a tile's first k-block    |
     full_rest        full_bar waits of its other k-blocks        |
     order            order_bar wait (ping-pong), lag waits       |  per math warp, over the tiles
                      (staggered)                                 |
     wait1 / wait0    wgmma_wait<1> / <0>                         |  that warp's warpgroup took
     epilogue         the whole epilogue, of which                |
       store_wait     waits for a store buffer                    |
       bias_wait      waits for the bias values                   |
       math_store     the rest: bias, GELU, packing, stores       |
   plus the card line (name, power limit, max SM clock) from the same run.
   AB_GEMM_SCHEDULE=pingpong|cooperative|staggered in the environment traces that schedule (N > 128 shapes).

Writes build/trace/ only; needs a GPU to run.
"""

from __future__ import annotations

import argparse
import ctypes as C
import hashlib
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

from aurora_b200 import _build, cabi  # noqa: E402
from gemm_shapes import card, describe, time_shape  # noqa: E402

TRACE_DIR = ROOT / "build" / "trace"

# (name, m, n, k, gelu): the 0.25-degree Aurora backbone, 4 levels x 180 x 360 tokens at stage 1, D = 512 / 1024 / 2048
SHAPES = [
    ("s1_qkv", 259200, 1536, 512, False),
    ("s1_proj", 259200, 512, 512, False),
    ("s1_fc1", 259200, 2048, 512, True),
    ("s1_fc2", 259200, 512, 2048, False),
    ("s2_qkv", 64800, 3072, 1024, False),
    ("s2_proj", 64800, 1024, 1024, False),
    ("s2_fc1", 64800, 4096, 1024, True),
    ("s3_fc1", 16200, 8192, 2048, True),
]

CTA_WORDS = 6  # timer start / end, clock start / end, producer empty waits, producer tiles
SLOTS = ["full_first", "full_rest", "order", "wait1", "wait0", "epilogue", "store_wait", "bias_wait", "tiles"]


def build_libs(source: Path) -> tuple[Path, Path]:
    """(untraced, traced) libraries with `source` as gemm.cu, cached by content under build/trace/."""
    _build.build()  # the other objects
    src = source.read_bytes()
    tag = hashlib.sha256(src + _build.source_hash().encode()).hexdigest()[:16]
    out = TRACE_DIR / tag
    libs = (out / "libplain.so", out / "libtraced.so")
    if all(p.exists() for p in libs):
        return libs
    out.mkdir(parents=True, exist_ok=True)
    gemm_src = out / "gemm.cu"  # next to its objects, so that compile errors name it; includes come from csrc
    gemm_src.write_bytes(src)
    others = [str(_build.OBJ_DIR / (s.stem + ".o")) for s in _build.sources() if s.name != "gemm.cu"]
    nvcc = _build._nvcc()
    for lib, defs in zip(libs, ([], ["-DAB_GEMM_TRACE"])):
        obj = lib.with_suffix(".o")
        cmd = [nvcc, *_build.NVCC_FLAGS, *defs, "-I", str(_build.CSRC), "-c", str(gemm_src), "-o", str(obj)]
        subprocess.run(cmd, check=True)
        subprocess.run([nvcc, "-shared", *_build.NVCC_FLAGS[:2], "-o", str(lib), str(obj), *others], check=True)
    return libs


def load(path: Path) -> C.CDLL:
    """The library at `path`, set up as cabi.lib() sets up the in-tree one."""
    h = C.CDLL(str(path))
    h.ab_version.restype = C.c_int
    assert h.ab_version() == cabi.ABI_VERSION
    h.ab_last_error.restype = C.c_char_p
    h.ab_launch_count.restype = C.c_ulonglong
    for name in cabi.EXPORTS:
        if name not in ("ab_version", "ab_last_error", "ab_launch_count"):
            getattr(h, name).restype = C.c_int
    return h


def key_of(m: int, n: int, k: int, gelu: bool) -> tuple:
    return (m, n, k, "bfloat16", True, cabi.AB_ACT_GELU_ERF if gelu else cabi.AB_ACT_NONE, False, "bfloat16", False)


def summarise(rec: torch.Tensor, words: int) -> dict:
    """Per-tile microseconds of each phase from the CTA records of one or more launches (rows: CTAs)."""
    rec = rec.double()
    ns = rec[:, 1] - rec[:, 0]
    cyc = rec[:, 3] - rec[:, 2]
    ghz = (cyc / ns).mean().item()
    cta_tiles = rec[:, 5]
    out = {"sm_clock_mhz": round(1e3 * ghz, 0), "tile_us": round((ns / cta_tiles).mean().item() / 1e3, 3),
           "producer": round((rec[:, 4] / cta_tiles).mean().item() / ghz / 1e3, 3)}
    warps = rec[:, CTA_WORDS:words].reshape(rec.shape[0], -1, len(SLOTS))
    tiles = warps[..., SLOTS.index("tiles")]
    keep = tiles > 0
    for i, name in enumerate(SLOTS[:-1]):
        out[name] = round((warps[..., i][keep] / tiles[keep]).mean().item() / ghz / 1e3, 3)
    out["math_store"] = round(out["epilogue"] - out["store_wait"] - out["bias_wait"], 3)
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--source", type=Path, default=_build.CSRC / "gemm.cu", help="gemm.cu to trace")
    ap.add_argument("--label", default="tree")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--build-only", action="store_true")
    args = ap.parse_args()
    plain_so, traced_so = build_libs(args.source.resolve())
    if args.build_only:
        print(json.dumps({"kind": "built", "plain": str(plain_so), "traced": str(traced_so)}))
        return
    if not torch.cuda.is_available():
        raise SystemExit("tools/gemm_trace.py needs a CUDA device")
    print(json.dumps({**card(), "label": args.label}), flush=True)
    plain, traced = load(plain_so), load(traced_so)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    buf = torch.zeros(sms * 512, dtype=torch.int64, device="cuda")
    words = traced.ab_gemm_trace(C.c_void_p(buf.data_ptr()))
    assert words == CTA_WORDS + 8 * len(SLOTS), words

    saved = cabi._lib
    try:
        for name, m, n, k, gelu in SHAPES:
            key = key_of(m, n, k, gelu)
            cabi._lib = plain
            ms_plain = time_shape(key, args.iters)
            cabi._lib = traced
            buf.zero_()
            ms_traced = time_shape(key, args.iters)  # the records left in buf are the last launch's
            rec = buf[: sms * words].view(sms, words).cpu()
            rec = rec[rec[:, 5] > 0]  # the CTAs of the launch
            flop = 2.0 * m * n * k
            print(json.dumps({"kind": "trace", "label": args.label, "shape": name, **describe(key),
                              "ms_plain": round(ms_plain, 4), "ms_traced": round(ms_traced, 4),
                              "tflops_plain": round(flop / ms_plain / 1e9, 1),
                              "overhead": round(ms_traced / ms_plain - 1.0, 4), **summarise(rec, words)}), flush=True)
    finally:
        cabi._lib = saved


if __name__ == "__main__":
    main()
