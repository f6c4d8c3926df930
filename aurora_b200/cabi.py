"""ctypes binding of ``libaurora_b200.so`` (the C ABI declared in ``include/aurora_b200.h``).

PyTorch owns every buffer; this module only forwards raw device pointers, sizes and the current
CUDA stream.  There is no CPU fallback: if the library is missing it is built (``nvcc`` required),
and if it cannot be loaded every call raises.
"""

from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from aurora_b200 import _build

__all__ = [
    "lib", "AbError", "check", "ptr", "stream_ptr", "launch_count", "gemm", "window_attention", "window_geometry",
    "window_index_map", "ln_mod_residual", "patch_merge_ln", "patch_split_ln", "perceiver_attention",
    "linear_small", "patchify", "unpatchify", "AbFieldIn", "AbFieldOut", "ipc_export", "ipc_open", "ipc_close",
    "halo_push", "halo_wait", "AbSwinBlock", "swin_block", "swin_block_workspace_bytes", "gemm_ln_supported",
    "gemm_ln_residual", "AbTrackBox", "track_boxes", "AbScoreField", "score_workspace_bytes", "score_fields",
    "AbEnsembleField", "ensemble_score_workspace_bytes", "ensemble_score_fields", "AbSpectrumField",
    "zonal_spectra_workspace_bytes", "zonal_spectra",
]

ABI_VERSION = 2  # == AB_ABI_VERSION in include/aurora_b200.h
AB_ACT_NONE = 0
AB_ACT_GELU_ERF = 1


class AbError(RuntimeError):
    """A call into libaurora_b200.so returned a negative status."""


class AbGemm(C.Structure):
    _fields_ = [
        ("a", C.c_void_p),
        ("w", C.c_void_p),
        ("bias", C.c_void_p),
        ("residual", C.c_void_p),
        ("out_f32", C.c_void_p),
        ("out_bf16", C.c_void_p),
        ("m", C.c_int32),
        ("n", C.c_int32),
        ("k", C.c_int32),
        ("lda", C.c_int32),
        ("ldw", C.c_int32),
        ("ldr", C.c_int32),
        ("ld_f32", C.c_int32),
        ("ld_bf16", C.c_int32),
        ("act", C.c_int32),
        ("in_dtype", C.c_int32),
        ("out_dtype", C.c_int32),
        ("peer_push", C.c_void_p),
    ]


AB_DT_BF16, AB_DT_F16 = 0, 1
_DT = {torch.bfloat16: AB_DT_BF16, torch.float16: AB_DT_F16}


def _dt(t: torch.Tensor) -> int:
    try:
        return _DT[t.dtype]
    except KeyError:
        raise AbError(f"expected a bf16 or fp16 tensor, got {t.dtype}") from None


_lib: Optional[C.CDLL] = None


def lib() -> C.CDLL:
    """Load (building first if needed) the shared library.  Raises if that is impossible."""
    global _lib
    if _lib is None:
        path = _build.LIB_PATH
        _build.build()  # no-op when the library matches the sources (content hash); never load a stale binary
        handle = C.CDLL(str(path))
        handle.ab_version.restype = C.c_int
        if handle.ab_version() != ABI_VERSION:
            raise AbError(f"libaurora_b200.so has ABI version {handle.ab_version()}, this binding expects {ABI_VERSION}")
        handle.ab_last_error.restype = C.c_char_p
        handle.ab_launch_count.restype = C.c_ulonglong
        for name in EXPORTS:
            if name in ("ab_version", "ab_last_error", "ab_launch_count"):
                continue
            getattr(handle, name).restype = C.c_int
        _lib = handle
    return _lib


# Every symbol include/aurora_b200.h declares (tests check that the library exports all of them).
EXPORTS = [
    "ab_version",
    "ab_last_error",
    "ab_launch_count",
    "ab_gemm_bf16",
    "ab_window_attention",
    "ab_window_geometry",
    "ab_window_index_map",
    "ab_window_index_map_host",
    "ab_ln_mod_residual",
    "ab_patch_merge_ln",
    "ab_patch_split_ln",
    "ab_perceiver_attention",
    "ab_linear_small_f32",
    "ab_patchify",
    "ab_unpatchify",
    "ab_ipc_export",
    "ab_ipc_open",
    "ab_ipc_close",
    "ab_halo_push",
    "ab_halo_wait",
    "ab_swin_block",
    "ab_swin_block_workspace_bytes",
    "ab_gemm_ln_supported",
    "ab_gemm_ln_residual",
    "ab_run_ops",
    "ab_struct_size",
    "ab_track_boxes",
    "ab_score_workspace_bytes",
    "ab_score_fields",
    "ab_ensemble_score_workspace_bytes",
    "ab_ensemble_score_fields",
    "ab_zonal_spectra_workspace_bytes",
    "ab_zonal_spectra",
]
AB_IPC_HANDLE_BYTES = 64
AB_HALO_CTRL_BYTES = 256
AB_MAX_FIELDS = 64
AB_IN_PLAIN, AB_IN_CLAMP_MIN0, AB_IN_CLAMP_LOG_COMBINE = 0, 1, 2
AB_IN_NAN_TO_ZERO, AB_IN_DENSITY, AB_IN_SIN_DEG, AB_IN_COS_DEG = 3, 4, 5, 6


# Optional per-call device timing (bench.py's roofline leg): when PROFILE is a dict, every op wrapper
# records a CUDA-event pair on the current stream under its kernel name.
PROFILE: Optional[dict] = None

# Plan recording: when RECORD is a list, the wrappers that `ab_run_ops` can replay (gemm, swin_block, ln_mod_residual,
# patch_merge_ln, patch_split_ln) append their filled descriptor as (AB_OP_* kind, struct) INSTEAD of launching; the
# caller turns the list into an `AbOp` array with `make_program` and replays it with `run_ops` (one C call).
RECORD: Optional[list] = None
AB_OP_GEMM, AB_OP_SWIN_BLOCK, AB_OP_LN_MOD_RESIDUAL, AB_OP_PATCH_MERGE_LN, AB_OP_PATCH_SPLIT_LN = 1, 2, 3, 4, 5


class _Timed:
    def __init__(self, name: str, work: float = 0.0, nbytes: float = 0.0):
        self.name, self.work, self.nbytes = name, work, nbytes

    def __enter__(self):
        if PROFILE is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e1 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def __exit__(self, *exc):
        if PROFILE is not None:
            self.e1.record()
            PROFILE.setdefault(self.name, []).append((self.e0, self.e1, self.work, self.nbytes))
        return False


def check(status: int, what: str = "") -> None:
    if status != 0:
        msg = lib().ab_last_error().decode("utf-8", "replace")
        raise AbError(f"{what or 'libaurora_b200'} failed with status {status}: {msg}")


def ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    """Device pointer of a CUDA tensor (None passes through as NULL)."""
    if t is None:
        return None
    if not t.is_cuda:
        raise AbError("libaurora_b200 operates on CUDA tensors only (got a CPU tensor); there is no CPU path")
    return t.data_ptr()


def stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def launch_count() -> int:
    return int(lib().ab_launch_count())


def _ld(t: torch.Tensor) -> int:
    assert t.dim() == 2 and t.stride(1) == 1, "expected a row-major 2-D view"
    return t.stride(0) if t.shape[0] > 1 else max(t.stride(0), t.shape[1])


def gemm(
    a: torch.Tensor,
    w: torch.Tensor,
    *,
    bias: Optional[torch.Tensor] = None,
    residual: Optional[torch.Tensor] = None,
    out_f32: Optional[torch.Tensor] = None,
    out_bf16: Optional[torch.Tensor] = None,
    act: int = AB_ACT_NONE,
    peer_push=None,
) -> None:
    """``out = act(a @ w.T + bias) + residual`` on the wgmma GEMM (a, w bf16; outputs preallocated).
    `peer_push` (an `AbHaloPush`): the epilogue also stores the boundary rows it names into neighbouring GPUs' memory."""
    assert a.dtype == w.dtype, (a.dtype, w.dtype)
    m, k = a.shape
    n, k2 = w.shape
    assert k == k2, f"K mismatch {k} vs {k2}"
    g = AbGemm()
    g.a, g.w = ptr(a), ptr(w)
    g.bias = ptr(bias)
    g.residual = ptr(residual)
    g.out_f32 = ptr(out_f32)
    g.out_bf16 = ptr(out_bf16)
    g.m, g.n, g.k = m, n, k
    g.lda, g.ldw = _ld(a), _ld(w)
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.numel() == n and bias.is_contiguous()
    if residual is not None:
        assert residual.dtype == torch.float32 and residual.shape == (m, n)
        g.ldr = _ld(residual)
    if out_f32 is not None:
        assert out_f32.dtype == torch.float32 and out_f32.shape == (m, n)
        g.ld_f32 = _ld(out_f32)
    g.in_dtype = _dt(a)
    if out_bf16 is not None:
        assert out_bf16.shape == (m, n)
        g.ld_bf16 = _ld(out_bf16)
        g.out_dtype = _dt(out_bf16)
    g.act = act
    if peer_push is not None:
        g.peer_push = C.addressof(peer_push)
    # compulsory HBM bytes: A and W once, every output once, the residual once
    nb = 2.0 * m * k + 2.0 * n * k + m * n * ((4.0 if out_f32 is not None else 0.0) + (2.0 if out_bf16 is not None else 0.0)
                                              + (4.0 if residual is not None else 0.0))
    if RECORD is not None:
        RECORD.append((AB_OP_GEMM, g))
        return
    with _Timed("gemm", work=2.0 * m * n * k, nbytes=nb):
        check(lib().ab_gemm_bf16(C.byref(g), C.c_void_p(stream_ptr())), "ab_gemm_bf16")


class AbWindowAttention(C.Structure):
    _fields_ = [
        ("qkv", C.c_void_p),
        ("pad_qkv", C.c_void_p),
        ("out", C.c_void_p),
        ("bias", C.c_void_p),
        ("batch", C.c_int32),
        ("res", C.c_int32 * 3),
        ("window", C.c_int32 * 3),
        ("shift", C.c_int32 * 3),
        ("num_heads", C.c_int32),
        ("head_dim", C.c_int32),
        ("warped", C.c_int32),
        ("slab_h_begin", C.c_int32),
        ("slab_h_rows", C.c_int32),
        ("slab_halo", C.c_int32),
        ("reserved_", C.c_int32),
        ("halo_kv", C.c_void_p),
        ("halo_ctrl", C.c_void_p),
    ]


class AbLnModResidual(C.Structure):
    _fields_ = [
        ("y", C.c_void_p),
        ("scale", C.c_void_p),
        ("shift", C.c_void_p),
        ("residual", C.c_void_p),
        ("add_rows", C.c_void_p),
        ("out_f32", C.c_void_p),
        ("out_bf16", C.c_void_p),
        ("rows", C.c_int64),
        ("res_div", C.c_int64),
        ("res_mod", C.c_int64),
        ("add_mod", C.c_int64),
        ("dim", C.c_int32),
        ("ld_y", C.c_int32),
        ("ld_res", C.c_int32),
        ("ld_f32", C.c_int32),
        ("ld_bf16", C.c_int32),
        ("eps", C.c_float),
        ("in_dtype", C.c_int32),
        ("out_dtype", C.c_int32),
    ]


class AbPatchMergeLn(C.Structure):
    _fields_ = [("x", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p), ("out_bf16", C.c_void_p),
                ("batch", C.c_int32), ("c", C.c_int32), ("h", C.c_int32), ("w", C.c_int32), ("d", C.c_int32),
                ("eps", C.c_float)]


class AbPatchSplitLn(C.Structure):
    _fields_ = [("y_bf16", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p), ("out_bf16", C.c_void_p),
                ("batch", C.c_int32), ("c", C.c_int32), ("h", C.c_int32), ("w", C.c_int32), ("d", C.c_int32),
                ("crop_h", C.c_int32), ("crop_w", C.c_int32), ("eps", C.c_float)]


class AbFieldIn(C.Structure):
    _fields_ = [
        ("ptr", C.c_void_p),
        ("stride_t", C.c_int64),
        ("loc", C.c_float),
        ("scale", C.c_float),
        ("const_value", C.c_float),
        ("transform", C.c_int32),
        ("w0", C.c_float),
        ("w1", C.c_float),
        ("wb", C.c_float),
    ]


class AbFieldOut(C.Structure):
    _fields_ = [
        ("ptr", C.c_void_p),
        ("prev", C.c_void_p),
        ("loc", C.c_float),
        ("scale", C.c_float),
        ("col", C.c_int32),
        ("mod_col", C.c_int32),
        ("clamp_min0", C.c_int32),
        ("clamp_max1", C.c_int32),
        ("cos_col", C.c_int32),
        ("dens_col", C.c_int32),
        ("mask", C.c_void_p),
        ("mask_min", C.c_float),
    ]

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.mod_col = self.cos_col = self.dens_col = -1


def _i3(v):
    return (C.c_int32 * 3)(*[int(x) for x in v])


def _s():
    return C.c_void_p(stream_ptr())


def window_geometry(res, window, shift) -> tuple[int, int, bool]:
    """(windows per batch element, tokens per clamped window, mask applies) — host only."""
    nw, nt, sh = C.c_int32(), C.c_int32(), C.c_int32()
    check(lib().ab_window_geometry(_i3(res), _i3(window), _i3(shift), C.byref(nw), C.byref(nt), C.byref(sh)),
          "ab_window_geometry")
    return nw.value, nt.value, bool(sh.value)


def window_index_map(res, window, shift, warped: bool = True, device="cuda"):
    """Materialise the in-kernel gather map / group ids (test hook)."""
    nw, nt, _ = window_geometry(res, window, shift)
    idx = torch.empty(nw * nt, dtype=torch.int32, device=device)
    grp = torch.empty(nw * nt, dtype=torch.uint8, device=device)
    check(lib().ab_window_index_map(_i3(res), _i3(window), _i3(shift), C.c_int32(int(warped)),
                                    C.c_void_p(ptr(idx)), C.c_void_p(ptr(grp)), _s()), "ab_window_index_map")
    return idx.view(nw, nt), grp.view(nw, nt)


def window_index_map_host(res, window, shift, warped: bool = True):
    """The same index arithmetic evaluated on the host (numpy arrays); needs no GPU."""
    import numpy as np

    nw, nt, _ = window_geometry(res, window, shift)
    idx = np.empty(nw * nt, dtype=np.int32)
    grp = np.empty(nw * nt, dtype=np.uint8)
    check(lib().ab_window_index_map_host(_i3(res), _i3(window), _i3(shift), C.c_int32(int(warped)),
                                         idx.ctypes.data_as(C.c_void_p), grp.ctypes.data_as(C.c_void_p)),
          "ab_window_index_map_host")
    return idx.reshape(nw, nt), grp.reshape(nw, nt)


def window_attention(qkv: torch.Tensor, out: torch.Tensor, *, batch: int, res, window, shift, num_heads: int,
                     pad_qkv: Optional[torch.Tensor] = None, bias: Optional[torch.Tensor] = None,
                     warped: bool = True, slab: Optional[tuple[int, int]] = None,
                     halo_kv: Optional[torch.Tensor] = None, halo_ctrl: Optional[int] = None) -> None:
    """`slab=(h_begin, h_rows)`: qkv / out hold only those rows of the global grid `res` (latitude sharding);
    `halo_kv` is bf16 [2, C, halo, W, 2D]: K | V of the rows above / below the slab (cyclic)."""
    assert qkv.dtype == torch.bfloat16 and out.dtype == torch.bfloat16 and qkv.is_contiguous() and out.is_contiguous()
    d = num_heads * 64
    tokens = batch * res[0] * res[1] * res[2] if slab is None else res[0] * slab[1] * res[2]
    assert qkv.shape == (tokens, 3 * d) and out.shape == (tokens, d), (qkv.shape, out.shape, tokens, d)
    a = AbWindowAttention()
    a.qkv, a.out = ptr(qkv), ptr(out)
    if pad_qkv is not None:
        assert pad_qkv.dtype == torch.bfloat16 and pad_qkv.numel() == 3 * d and pad_qkv.is_contiguous()
    a.pad_qkv = ptr(pad_qkv)
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.is_contiguous()
    a.bias = ptr(bias)
    a.batch = batch
    a.res, a.window, a.shift = _i3(res), _i3(window), _i3(shift)
    a.num_heads, a.head_dim, a.warped = num_heads, 64, int(warped)
    if slab is not None:
        a.slab_h_begin, a.slab_h_rows = int(slab[0]), int(slab[1])
        if halo_kv is not None:
            assert halo_kv.dtype == torch.bfloat16 and halo_kv.is_contiguous() and halo_kv.dim() == 5
            assert halo_kv.shape[0] == 2 and halo_kv.shape[1] == res[0] and halo_kv.shape[3] == res[2]
            assert halo_kv.shape[4] == 2 * d
            a.slab_halo = halo_kv.shape[2]
            a.halo_kv = ptr(halo_kv)
            a.halo_ctrl = halo_ctrl  # peer transport: the kernel waits for the neighbours' pushes itself
    nw, nt, _ = window_geometry(res, window, shift)
    with _Timed("window_attention", work=4.0 * batch * nw * num_heads * nt * nt * 64, nbytes=8.0 * tokens * d):
        check(lib().ab_window_attention(C.byref(a), _s()), "ab_window_attention")


def ln_mod_residual(y: torch.Tensor, *, scale=None, shift=None, residual=None, add_rows=None, out_f32=None,
                    out_bf16=None, eps: float = 1e-5, res_div: int = 1, res_mod: int = 0) -> None:
    assert y.dim() == 2
    rows, dim = y.shape
    a = AbLnModResidual()
    a.y = ptr(y)
    a.in_dtype = _dt(y)
    a.ld_y = _ld(y)
    for t in (scale, shift):
        assert t is None or (t.dtype == torch.float32 and t.numel() == dim and t.is_contiguous())
    a.scale, a.shift = ptr(scale), ptr(shift)
    if residual is not None:
        assert residual.dtype == torch.float32 and residual.shape[1] == dim
        a.residual, a.ld_res = ptr(residual), _ld(residual)
        if res_mod == 0:
            assert residual.shape[0] == rows
        else:
            assert residual.shape[0] >= res_mod
    if add_rows is not None:
        assert add_rows.dtype == torch.float32 and add_rows.shape[1] == dim and add_rows.is_contiguous()
        a.add_rows, a.add_mod = ptr(add_rows), add_rows.shape[0]
    if out_f32 is not None:
        assert out_f32.dtype == torch.float32 and out_f32.shape == (rows, dim)
        a.out_f32, a.ld_f32 = ptr(out_f32), _ld(out_f32)
    if out_bf16 is not None:
        assert out_bf16.shape == (rows, dim)
        a.out_bf16, a.ld_bf16 = ptr(out_bf16), _ld(out_bf16)
        a.out_dtype = _dt(out_bf16)
    a.rows, a.dim, a.eps = rows, dim, eps
    a.res_div, a.res_mod = res_div, res_mod
    nb = rows * dim * (2.0 + (4.0 if residual is not None and res_mod == 0 else 0.0)
                       + (4.0 if out_f32 is not None else 0.0) + (2.0 if out_bf16 is not None else 0.0)
                       + (4.0 if add_rows is not None else 0.0))
    if RECORD is not None:
        RECORD.append((AB_OP_LN_MOD_RESIDUAL, a))
        return
    with _Timed("ln_mod_residual", nbytes=nb):
        check(lib().ab_ln_mod_residual(C.byref(a), _s()), "ab_ln_mod_residual")


def patch_merge_ln(x: torch.Tensor, gamma, beta, out: torch.Tensor, *, batch, c, h, w, d, eps=1e-5) -> None:
    assert x.dtype == torch.float32 and x.is_contiguous() and x.numel() == batch * c * h * w * d
    assert out.dtype == torch.bfloat16 and out.is_contiguous()
    assert out.numel() == batch * c * ((h + 1) // 2) * ((w + 1) // 2) * 4 * d
    if RECORD is not None:
        m = AbPatchMergeLn(x=ptr(x), gamma=ptr(gamma), beta=ptr(beta), out_bf16=ptr(out), batch=batch, c=c, h=h, w=w, d=d, eps=eps)
        RECORD.append((AB_OP_PATCH_MERGE_LN, m))
        return
    check(lib().ab_patch_merge_ln(C.c_void_p(ptr(x)), C.c_void_p(ptr(gamma)), C.c_void_p(ptr(beta)),
                                  C.c_void_p(ptr(out)), batch, c, h, w, d, C.c_float(eps), _s()), "ab_patch_merge_ln")


def patch_split_ln(y: torch.Tensor, gamma, beta, out: torch.Tensor, *, batch, c, h, w, d, crop_h, crop_w,
                   eps=1e-5) -> None:
    assert y.dtype == torch.bfloat16 and y.is_contiguous() and y.numel() == batch * c * h * w * 2 * d
    assert out.dtype == torch.bfloat16 and out.is_contiguous()
    assert out.numel() == batch * c * (2 * h - crop_h) * (2 * w - crop_w) * (d // 2)
    if RECORD is not None:
        sp = AbPatchSplitLn(y_bf16=ptr(y), gamma=ptr(gamma), beta=ptr(beta), out_bf16=ptr(out), batch=batch, c=c, h=h, w=w,
                            d=d, crop_h=crop_h, crop_w=crop_w, eps=eps)
        RECORD.append((AB_OP_PATCH_SPLIT_LN, sp))
        return
    check(lib().ab_patch_split_ln(C.c_void_p(ptr(y)), C.c_void_p(ptr(gamma)), C.c_void_p(ptr(beta)),
                                  C.c_void_p(ptr(out)), batch, c, h, w, d, crop_h, crop_w, C.c_float(eps), _s()),
          "ab_patch_split_ln")


def perceiver_attention(q: torch.Tensor, kv: torch.Tensor, out: torch.Tensor, *, nloc: int, num_heads: int,
                        head_dim: int) -> None:
    assert q.dtype == torch.float32 and q.is_contiguous() and q.dim() == 2
    lq, d = q.shape
    assert d == num_heads * head_dim
    assert kv.dim() == 2 and kv.shape[1] == 2 * d and kv.shape[0] % nloc == 0
    lk = kv.shape[0] // nloc
    assert out.dtype == kv.dtype and out.shape == (lq * nloc, d)
    check(lib().ab_perceiver_attention(C.c_void_p(ptr(q)), C.c_void_p(ptr(kv)), C.c_void_p(ptr(out)),
                                       C.c_int64(nloc), lq, lk, num_heads, head_dim, _ld(kv), _ld(out), _dt(kv),
                                       _s()),
          "ab_perceiver_attention")


def linear_small(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, *, silu_in=False,
                 silu_out=False) -> torch.Tensor:
    assert x.dtype == torch.float32 and w.dtype == torch.float32 and x.is_contiguous() and w.is_contiguous()
    rows, k = x.shape
    n, k2 = w.shape
    assert k == k2
    y = torch.empty(rows, n, dtype=torch.float32, device=x.device)
    check(lib().ab_linear_small_f32(C.c_void_p(ptr(x)), C.c_void_p(ptr(w)), C.c_void_p(ptr(bias)),
                                    C.c_void_p(ptr(y)), rows, n, k, int(silu_in), int(silu_out), _s()),
          "ab_linear_small_f32")
    return y


def patchify(fields: list, t_hist: int, h: int, w: int, p: int, out: torch.Tensor) -> None:
    assert out.dim() == 2 and out.shape[0] == (h // p) * (w // p)
    arr = (AbFieldIn * len(fields))(*fields)
    check(lib().ab_patchify(arr, len(fields), t_hist, h, w, p, C.c_void_p(ptr(out)), _ld(out), _dt(out), _s()),
          "ab_patchify")


def unpatchify(fields: list, y: torch.Tensor, h: int, w: int, p: int) -> None:
    assert y.dtype == torch.float32 and y.dim() == 2 and y.shape[0] == (h // p) * (w // p)
    arr = (AbFieldOut * len(fields))(*fields)
    check(lib().ab_unpatchify(arr, len(fields), C.c_void_p(ptr(y)), _ld(y), h, w, p, _s()), "ab_unpatchify")


# ---- peer-memory halo exchange (csrc/halo.cu) ------------------------------------------------------------------
class AbHaloPush(C.Structure):
    _fields_ = [
        ("local", C.c_void_p),
        ("above_slot", C.c_void_p),
        ("below_slot", C.c_void_p),
        ("above_flag", C.c_void_p),
        ("below_flag", C.c_void_p),
        ("ctrl", C.c_void_p),
        ("c", C.c_int32),
        ("rows", C.c_int32),
        ("w", C.c_int32),
        ("slot_rows", C.c_int32),
        ("rows_to_above", C.c_int32),
        ("rows_to_below", C.c_int32),
        ("src_tok_bytes", C.c_int64),
        ("tok_off_bytes", C.c_int64),
        ("tok_bytes", C.c_int64),
    ]


def ipc_export(t: torch.Tensor) -> tuple[bytes, int]:
    """(IPC handle bytes, offset of `t` inside its allocation) for a CUDA tensor of THIS process."""
    h = (C.c_uint8 * AB_IPC_HANDLE_BYTES)()
    off = C.c_uint64()
    check(lib().ab_ipc_export(C.c_void_p(ptr(t)), h, C.byref(off)), "ab_ipc_export")
    return bytes(h), int(off.value)


def ipc_open(handle: bytes) -> int:
    """Map another process's allocation; returns its base address in this process."""
    assert len(handle) == AB_IPC_HANDLE_BYTES
    h = (C.c_uint8 * AB_IPC_HANDLE_BYTES).from_buffer_copy(handle)
    base = C.c_void_p()
    check(lib().ab_ipc_open(h, C.byref(base)), "ab_ipc_open")
    return int(base.value)


def ipc_close(base: int) -> None:
    check(lib().ab_ipc_close(C.c_void_p(base)), "ab_ipc_close")


def halo_push(local: torch.Tensor, *, above_slot: int, below_slot: int, above_flag: int, below_flag: int, ctrl: int,
              slot_rows: int, rows_to_above: int, rows_to_below: int, col_from: int = 0) -> None:
    """`local` [C, rows, W, K] contiguous (2-byte elements); columns [col_from, K) of the first `rows_to_above` /
    last `rows_to_below` rows go to the neighbours.  The slot / flag arguments are raw (peer) addresses."""
    assert local.dim() == 4 and local.is_contiguous()
    es = local.element_size()
    a = AbHaloPush()
    a.local = ptr(local)
    a.above_slot, a.below_slot, a.above_flag, a.below_flag, a.ctrl = above_slot, below_slot, above_flag, below_flag, ctrl
    a.c, a.rows, a.w = local.shape[0], local.shape[1], local.shape[2]
    a.slot_rows, a.rows_to_above, a.rows_to_below = slot_rows, rows_to_above, rows_to_below
    a.src_tok_bytes = local.shape[3] * es
    a.tok_off_bytes = col_from * es
    a.tok_bytes = (local.shape[3] - col_from) * es
    with _Timed("halo_push", nbytes=float(a.c) * (rows_to_above + rows_to_below) * a.w * a.tok_bytes):
        check(lib().ab_halo_push(C.byref(a), _s()), "ab_halo_push")


def halo_wait(ctrl: int) -> None:
    with _Timed("halo_wait"):
        check(lib().ab_halo_wait(C.c_void_p(ctrl), _s()), "ab_halo_wait")


# ---- whole-block entry point (csrc/block.cu) ----------------------------------------------------------------------
class AbSwinBlock(C.Structure):
    _fields_ = [
        ("x_f32", C.c_void_p), ("x_b16", C.c_void_p), ("out_b16", C.c_void_p),
        ("w_qkv", C.c_void_p), ("w_proj", C.c_void_p), ("w_fc1", C.c_void_p), ("w_fc2", C.c_void_p),
        ("b_qkv", C.c_void_p), ("b_proj", C.c_void_p), ("b_fc1", C.c_void_p), ("b_fc2", C.c_void_p),
        ("pad_qkv", C.c_void_p),
        ("scale1", C.c_void_p), ("shift1", C.c_void_p), ("scale2", C.c_void_p), ("shift2", C.c_void_p),
        ("workspace", C.c_void_p), ("halo_push", C.POINTER(AbHaloPush)), ("halo_kv", C.c_void_p),
        ("dim", C.c_int32), ("hidden", C.c_int32), ("num_heads", C.c_int32),
        ("res", C.c_int32 * 3), ("window", C.c_int32 * 3), ("shift", C.c_int32 * 3),
        ("ld_out_b16", C.c_int32), ("out_b16_dtype", C.c_int32),
        ("slab_h_begin", C.c_int32), ("slab_h_rows", C.c_int32), ("halo_rows", C.c_int32),
        ("eps", C.c_float), ("fuse_ln", C.c_int32), ("fuse_push", C.c_int32),
    ]


def swin_block_workspace_bytes(tokens: int, dim: int, hidden: int) -> int:
    n = C.c_size_t()
    check(lib().ab_swin_block_workspace_bytes(C.c_int64(tokens), dim, hidden, C.byref(n)), "ab_swin_block_workspace_bytes")
    return int(n.value)


def swin_block(desc: AbSwinBlock) -> None:
    """One whole Swin3DTransformerBlock in place on the token stream (see include/aurora_b200.h)."""
    if RECORD is not None:
        RECORD.append((AB_OP_SWIN_BLOCK, desc))
        return
    check(lib().ab_swin_block(C.byref(desc), _s()), "ab_swin_block")


# ---- projection with adaLN + residual in the epilogue (csrc/gemm_ln.cu) -------------------------------------------
class AbGemmLn(C.Structure):
    _fields_ = [
        ("a", C.c_void_p), ("w", C.c_void_p), ("bias", C.c_void_p), ("scale", C.c_void_p), ("shift", C.c_void_p),
        ("residual", C.c_void_p), ("out_f32", C.c_void_p), ("out_16", C.c_void_p),
        ("m", C.c_int32), ("n", C.c_int32), ("k", C.c_int32),
        ("lda", C.c_int32), ("ldw", C.c_int32), ("ldr", C.c_int32), ("ld_f32", C.c_int32), ("ld_16", C.c_int32),
        ("in_dtype", C.c_int32), ("out_dtype", C.c_int32), ("eps", C.c_float),
    ]


def gemm_ln_supported(n: int) -> bool:
    return bool(lib().ab_gemm_ln_supported(int(n)))


def gemm_ln_residual(a: torch.Tensor, w: torch.Tensor, *, bias=None, scale=None, shift=None, residual=None, out_f32=None,
                     out_bf16=None, eps: float = 1e-5) -> None:
    """``out = residual + LN(a @ w.T + bias) * scale + shift`` in one kernel (N = 512 or 1024)."""
    assert a.dtype == w.dtype
    m, k = a.shape
    n, k2 = w.shape
    assert k == k2
    g = AbGemmLn()
    g.a, g.w, g.bias, g.scale, g.shift = ptr(a), ptr(w), ptr(bias), ptr(scale), ptr(shift)
    for t in (bias, scale, shift):
        assert t is None or (t.dtype == torch.float32 and t.numel() == n and t.is_contiguous())
    g.m, g.n, g.k, g.lda, g.ldw = m, n, k, _ld(a), _ld(w)
    if residual is not None:
        assert residual.dtype == torch.float32 and residual.shape == (m, n)
        g.residual, g.ldr = ptr(residual), _ld(residual)
    if out_f32 is not None:
        assert out_f32.dtype == torch.float32 and out_f32.shape == (m, n)
        g.out_f32, g.ld_f32 = ptr(out_f32), _ld(out_f32)
    g.in_dtype = _dt(a)
    if out_bf16 is not None:
        assert out_bf16.shape == (m, n)
        g.out_16, g.ld_16, g.out_dtype = ptr(out_bf16), _ld(out_bf16), _dt(out_bf16)
    g.eps = eps
    nb = 2.0 * m * k + 2.0 * n * k + m * n * ((4.0 if residual is not None else 0.0) + (4.0 if out_f32 is not None else 0.0)
                                              + (2.0 if out_bf16 is not None else 0.0))
    with _Timed("gemm_ln", work=2.0 * m * n * k, nbytes=nb):
        check(lib().ab_gemm_ln_residual(C.byref(g), _s()), "ab_gemm_ln_residual")


# ---- whole-stage replay (ab_run_ops) ------------------------------------------------------------------------------
class _AbOpUnion(C.Union):
    _fields_ = [("gemm", AbGemm), ("block", AbSwinBlock), ("ln", AbLnModResidual), ("merge", AbPatchMergeLn),
                ("split", AbPatchSplitLn)]


class AbOp(C.Structure):
    _fields_ = [("kind", C.c_int32), ("reserved_", C.c_int32), ("u", _AbOpUnion)]


_OP_FIELD = {AB_OP_GEMM: "gemm", AB_OP_SWIN_BLOCK: "block", AB_OP_LN_MOD_RESIDUAL: "ln", AB_OP_PATCH_MERGE_LN: "merge",
             AB_OP_PATCH_SPLIT_LN: "split"}


def make_program(recorded: list):
    """`recorded` = [(AB_OP_* kind, descriptor struct), ...] as collected under RECORD -> (AbOp array, keep-alive list)."""
    arr = (AbOp * len(recorded))()
    for i, (kind, desc) in enumerate(recorded):
        arr[i].kind = kind
        setattr(arr[i].u, _OP_FIELD[kind], desc)   # copies the struct; pointers inside keep pointing at caller-owned memory
    return arr, [d for _, d in recorded]


def run_ops(program) -> None:
    check(lib().ab_run_ops(program, len(program), _s()), "ab_run_ops")


# ---- tropical-cyclone tracking boxes (csrc/tracker.cu) ------------------------------------------------------------
AB_TRACK_MINIMA, AB_TRACK_MAX, AB_TRACK_MIN, AB_TRACK_WINDMAX = 0, 1, 2, 3
AB_TRACK_MAX_SIDE = 101
AB_TRACK_MAX_BOXES = 32


class AbTrackBox(C.Structure):
    _fields_ = [
        ("plane", C.c_void_p), ("plane2", C.c_void_p),
        ("h", C.c_int32), ("w", C.c_int32), ("ld", C.c_int32), ("op", C.c_int32),
        ("rows_off", C.c_int32), ("n_rows", C.c_int32), ("cols_off", C.c_int32), ("n_cols", C.c_int32),
        ("mask_off", C.c_int64),
    ]


def track_boxes(boxes: list, index: torch.Tensor, values: torch.Tensor, counts: torch.Tensor,
                masks: Optional[torch.Tensor]) -> None:
    """One launch over `boxes` (`AbTrackBox` list); `index` int32, `values` f32 and `counts` int32 [len(boxes)],
    `masks` uint8, all on the device."""
    assert index.dtype == torch.int32 and values.dtype == torch.float32 and counts.dtype == torch.int32
    assert values.numel() >= len(boxes) and counts.numel() >= len(boxes)
    arr = (AbTrackBox * len(boxes))(*boxes)
    check(lib().ab_track_boxes(arr, len(boxes), C.c_size_t(C.sizeof(AbTrackBox)), C.c_void_p(ptr(index)),
                               C.c_void_p(ptr(values)), C.c_void_p(ptr(counts)), C.c_void_p(ptr(masks)), _s()),
          "ab_track_boxes")


# ---- latitude-weighted scores (csrc/score.cu) ---------------------------------------------------------------------
AB_SCORE_MAX_FIELDS = 64
AB_SCORE_SUMS = 8  # W, sum w d, sum w d^2, sum w |d|, sum w af ao, sum w af^2, sum w ao^2, count


class AbScoreField(C.Structure):
    _fields_ = [
        ("pred", C.c_void_p), ("truth", C.c_void_p), ("clim", C.c_void_p),
        ("pred_level_stride", C.c_int64), ("truth_level_stride", C.c_int64), ("clim_level_stride", C.c_int64),
        ("h", C.c_int32), ("w", C.c_int32),
        ("ld_pred", C.c_int32), ("ld_truth", C.c_int32), ("ld_clim", C.c_int32),
        ("levels", C.c_int32),
    ]


def score_workspace_bytes(fields: list) -> int:
    arr = (AbScoreField * max(len(fields), 1))(*fields)
    n = C.c_size_t()
    check(lib().ab_score_workspace_bytes(arr, len(fields), C.c_size_t(C.sizeof(AbScoreField)), C.byref(n)),
          "ab_score_workspace_bytes")
    return int(n.value)


def score_fields(fields: list, row_weights: torch.Tensor, sums: torch.Tensor, workspace: torch.Tensor) -> None:
    """One call over `fields` (`AbScoreField` list): `row_weights` float64 [h], `sums` float64 [planes, 8] (a view with
    contiguous rows), `workspace` of at least `score_workspace_bytes(fields)` bytes, all on the device."""
    assert row_weights.dtype == torch.float64 and sums.dtype == torch.float64 and sums.is_contiguous()
    arr = (AbScoreField * max(len(fields), 1))(*fields)
    nbytes = workspace.numel() * workspace.element_size()
    check(lib().ab_score_fields(arr, len(fields), C.c_size_t(C.sizeof(AbScoreField)), C.c_void_p(ptr(row_weights)),
                                C.c_void_p(ptr(sums)), C.c_void_p(ptr(workspace)), C.c_size_t(nbytes), _s()),
          "ab_score_fields")


AB_ENS_MAX_MEMBERS = 64
AB_ENS_MAX_FIELDS = 16
# W, sum w (xm - y), sum w (xm - y)^2, sum w s^2, sum w crps skill, sum w crps spread, sum w af ao, sum w af^2,
# sum w ao^2, count
AB_ENS_SUMS = 10


class AbEnsembleField(C.Structure):
    _fields_ = [
        ("members", C.c_void_p * AB_ENS_MAX_MEMBERS), ("truth", C.c_void_p), ("clim", C.c_void_p),
        ("member_level_stride", C.c_int64), ("truth_level_stride", C.c_int64), ("clim_level_stride", C.c_int64),
        ("n_members", C.c_int32), ("h", C.c_int32), ("w", C.c_int32),
        ("ld_member", C.c_int32), ("ld_truth", C.c_int32), ("ld_clim", C.c_int32),
        ("levels", C.c_int32),
    ]


def ensemble_score_workspace_bytes(fields: list) -> int:
    arr = (AbEnsembleField * max(len(fields), 1))(*fields)
    n = C.c_size_t()
    check(lib().ab_ensemble_score_workspace_bytes(arr, len(fields), C.c_size_t(C.sizeof(AbEnsembleField)),
                                                  C.byref(n)), "ab_ensemble_score_workspace_bytes")
    return int(n.value)


def ensemble_score_fields(fields: list, row_weights: torch.Tensor, sums: torch.Tensor,
                          workspace: torch.Tensor) -> None:
    """One call over `fields` (`AbEnsembleField` list): `row_weights` float64 [h], `sums` float64 [planes, 10] (a view
    with contiguous rows), `workspace` of at least `ensemble_score_workspace_bytes(fields)` bytes, all on the device."""
    assert row_weights.dtype == torch.float64 and sums.dtype == torch.float64 and sums.is_contiguous()
    arr = (AbEnsembleField * max(len(fields), 1))(*fields)
    nbytes = workspace.numel() * workspace.element_size()
    check(lib().ab_ensemble_score_fields(arr, len(fields), C.c_size_t(C.sizeof(AbEnsembleField)),
                                         C.c_void_p(ptr(row_weights)), C.c_void_p(ptr(sums)),
                                         C.c_void_p(ptr(workspace)), C.c_size_t(nbytes), _s()),
          "ab_ensemble_score_fields")


# ---- latitude-band zonal power spectra (csrc/spectra.cu) ------------------------------------------------------------
AB_SPEC_MAX_FIELDS = 64
AB_SPEC_MAX_BANDS = 8
AB_SPEC_MAX_WIDTH = 4096


class AbSpectrumField(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("level_stride", C.c_int64),
        ("h", C.c_int32), ("w", C.c_int32), ("ld", C.c_int32), ("levels", C.c_int32),
    ]


def _band_rows(bands: list) -> C.Array:
    return (C.c_int32 * (2 * max(len(bands), 1)))(*(r for band in bands for r in band))


def zonal_spectra_workspace_bytes(fields: list, bands: list) -> int:
    """`bands`: [(r0, r1)] row ranges."""
    arr = (AbSpectrumField * max(len(fields), 1))(*fields)
    n = C.c_size_t()
    check(lib().ab_zonal_spectra_workspace_bytes(arr, len(fields), C.c_size_t(C.sizeof(AbSpectrumField)),
                                                 _band_rows(bands), len(bands), C.byref(n)),
          "ab_zonal_spectra_workspace_bytes")
    return int(n.value)


def zonal_spectra(fields: list, bands: list, row_weights: torch.Tensor, out: torch.Tensor,
                  workspace: torch.Tensor) -> None:
    """One call over `fields` (`AbSpectrumField` list of one grid) and `bands` ([(r0, r1)] row ranges): `row_weights`
    float64 [h], `out` float64 [planes, n_bands * (w // 2 + 3)] (a view with contiguous rows), `workspace` of at least
    `zonal_spectra_workspace_bytes(fields, bands)` bytes, all on the device."""
    assert row_weights.dtype == torch.float64 and out.dtype == torch.float64 and out.is_contiguous()
    arr = (AbSpectrumField * max(len(fields), 1))(*fields)
    nbytes = workspace.numel() * workspace.element_size()
    check(lib().ab_zonal_spectra(arr, len(fields), C.c_size_t(C.sizeof(AbSpectrumField)), _band_rows(bands),
                                 len(bands), C.c_void_p(ptr(row_weights)), C.c_void_p(ptr(out)),
                                 C.c_void_p(ptr(workspace)), C.c_size_t(nbytes), _s()),
          "ab_zonal_spectra")
