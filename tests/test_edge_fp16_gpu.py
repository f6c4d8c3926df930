"""The 16-bit kernels of the encoder / decoder path against float64 references of the same operation, fp16 and bf16
side by side.  The encoder and decoder run with fp16 operands by default (`AuroraEngine(edge_dtype="fp16")`), so every
fp16 instantiation below is on the production path.

Each reference decodes the 16-bit values the kernel reads, upcasts them to float64 and computes the operation there.
Bounds depend on the output type:
* 16-bit outputs: at most one ulp of the output type at the reference value (`_ulp`, fp16 subnormals included), plus
  an absolute floor only where the kernel's fp32 sum can cancel; each floor is derived where it is used.
* fp32 outputs: relative 1e-5 plus an absolute term scaled by the magnitude of the terms summed for that element.
fp16 stores saturate finite overflow and +-inf to +-65504 and keep NaN; bf16 and fp32 keep the value.  NaN must come
out exactly where the float64 reference (and torch.clamp in the reference model) puts it.

Measured on an H100 80GB HBM3 at a 700 W power limit, the largest error over the whole file was 0.50 of the bound on
16-bit outputs (the output rounding itself), 0.09 on fp32 outputs and 0.80 on the float32 angle remainder."""

import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
F16, BF16, F32 = torch.float16, torch.bfloat16, torch.float32
DTYPES = {"fp16": F16, "bf16": BF16}
FP16_MAX = 65504.0
FLT_MAX = float(np.finfo(np.float32).max)
NAN, INF = float("nan"), float("inf")
SENTINEL = -1000.0  # exactly representable in every output type
_FORMAT = {F16: (10, -14), BF16: (7, -126), F32: (23, -126)}  # (mantissa bits, smallest normal exponent)


# ------------------------------------------------------------------------------------------------
# comparison helpers
# ------------------------------------------------------------------------------------------------
def _ulp(x: torch.Tensor, dtype) -> torch.Tensor:
    """Spacing of `dtype` at |x| (float64): 2^(e - mantissa bits) with e the binade of |x|, clamped to the smallest
    normal exponent, so subnormals and 0 get the subnormal spacing (2^-24 for fp16)."""
    mant, emin = _FORMAT[dtype]
    ax = x.double().abs()
    e = torch.frexp(torch.where(torch.isfinite(ax) & (ax > 0), ax, torch.ones_like(ax))).exponent - 1
    e = torch.where(ax > 0, e, torch.full_like(e, emin)).clamp(min=emin)
    return torch.exp2((e - mant).double())


def _nan_and_inf(o: torch.Tensor, ref: torch.Tensor, rounded: torch.Tensor, what: str) -> torch.Tensor:
    nan_o, nan_r = torch.isnan(o), torch.isnan(ref)
    assert torch.equal(nan_o, nan_r), (f"{what}: NaN placement differs at {int((nan_o != nan_r).sum())} elements, "
                                       f"first {torch.nonzero(nan_o != nan_r)[:4].tolist()}, "
                                       f"kernel there {o[nan_o != nan_r][:4].tolist()}")
    inf_r = torch.isinf(rounded)
    assert torch.equal(o[inf_r], rounded[inf_r]), f"{what}: overflow to inf differs"
    return ~nan_r & ~inf_r


def _report(err, tol, fin, what):
    ratio = torch.where(fin, err / tol, torch.zeros_like(err))
    worst = float(ratio.max()) if ratio.numel() else 0.0
    if not worst <= 1.0:
        i = int(torch.argmax(torch.nan_to_num(ratio, nan=INF)))
        raise AssertionError(f"{what}: error {float(err.flatten()[i]):.3e} > bound {float(tol.flatten()[i]):.3e} "
                             f"(worst error / bound {worst:.2f}, element {i})")
    return worst


def _check16(out: torch.Tensor, ref: torch.Tensor, floor=0.0, what: str = "") -> float:
    """16-bit `out` against float64 `ref`: NaN exactly where ref is NaN; fp16 saturates ref to +-65504 first; where ref
    rounds to +-inf in bf16 the same inf; elsewhere |out - ref| <= ulp(ref) + floor."""
    dtype = out.dtype
    ref = ref.double()
    if dtype == F16:
        ref = ref.clamp(-FP16_MAX, FP16_MAX)  # keeps NaN
    o = out.double()
    fin = _nan_and_inf(o, ref, ref.to(dtype).double(), what)
    err = torch.where(fin, (o - ref).abs(), torch.zeros_like(o))
    tol = _ulp(ref, dtype) + floor
    return _report(err, tol.expand_as(err), fin, what)


def _check32(out: torch.Tensor, ref: torch.Tensor, atol, what: str = "") -> float:
    """fp32 `out` against float64 `ref`: NaN / inf where ref has them, elsewhere |out - ref| <= 1e-5 |ref| + atol."""
    ref = ref.double()
    o = out.double()
    fin = _nan_and_inf(o, ref, ref.float().double(), what)
    err = torch.where(fin, (o - ref).abs(), torch.zeros_like(o))
    tol = 1e-5 * torch.where(fin, ref.abs(), torch.zeros_like(ref)) + atol + _ulp(ref, F32)
    return _report(err, tol.expand_as(err), fin, what)


def _round16(x32: torch.Tensor, dtype) -> torch.Tensor:
    """What a 16-bit store of the fp32 value must hold: round to nearest even; fp16 saturates at +-65504, NaN stays."""
    return (x32.clamp(-FP16_MAX, FP16_MAX) if dtype == F16 else x32).to(dtype)


def _same_bits_or_nan(a: torch.Tensor, b: torch.Tensor) -> bool:
    nan = torch.isnan(a)
    return torch.equal(nan, torch.isnan(b)) and torch.equal(a[~nan], b[~nan])


def _padded(rows, cols, dtype, left=8, right=8, fill=SENTINEL):
    """A [rows, cols] view starting `left` columns into rows of left + cols + right (leading dimension > cols)."""
    buf = torch.full((rows, left + cols + right), fill, device=DEV, dtype=dtype)
    return buf, buf[:, left:left + cols]


def _untouched(buf, left, cols) -> bool:
    return bool((buf[:, :left] == SENTINEL).all()) and bool((buf[:, left + cols:] == SENTINEL).all())


# ------------------------------------------------------------------------------------------------
# ln_mod_residual: out = residual[(row / res_div) % res_mod] + LN(y) * scale + shift + add_rows[row % add_mod]
# ------------------------------------------------------------------------------------------------
LN_WIDTHS = [8, 24, 200, 256, 264, 512, 520, 1000, 1024, 1032, 2048]  # every CH bucket, with non-powers of two
LN_PAIRS = [("fp16", "fp16"), ("fp16", "bf16"), ("bf16", "fp16"), ("bf16", "bf16")]


def _ln_reference(y, scale, shift, residual, add_rows, res_div, res_mod, eps):
    """float64 LayerNorm + modulation + residual, and the absolute error bound of the kernel's fp32 evaluation.

    The kernel takes a two-pass mean / variance in fp32: lanes sum dim / 32 values each, then a 5-level butterfly, so
    the mean is off by at most (dim / 32 + 8) * 2^-24 * max|y| (the conditioning of a row whose mean is large against
    its spread), scaled by rstd * |scale| in the output.  rsqrtf, the products and the adds of shift / residual /
    add_rows cost a few fp32 roundings of the terms summed: 2^-21 of their magnitudes."""
    x = y.double()
    rows, dim = x.shape
    mu = x.mean(1, keepdim=True)
    rstd = (((x - mu) ** 2).mean(1, keepdim=True) + eps).rsqrt()
    n = (x - mu) * rstd
    s = scale.double() if scale is not None else torch.ones(dim, device=DEV, dtype=torch.float64)
    ref = n * s
    mag = ref.abs()
    if shift is not None:
        ref = ref + shift.double()
        mag = mag + shift.double().abs()
    if residual is not None:
        r = torch.arange(rows, device=DEV)
        rr = residual.double()[(r // res_div) % res_mod] if res_mod else residual.double()
        ref = ref + rr
        mag = mag + rr.abs()
    if add_rows is not None:
        ar = add_rows.double()[torch.arange(rows, device=DEV) % add_rows.shape[0]]
        ref = ref + ar
        mag = mag + ar.abs()
    cond = x.abs().amax(1, keepdim=True) * rstd
    atol = (dim // 32 + 8) * 2.0**-24 * cond * s.abs() + 2.0**-21 * torch.nan_to_num(mag, nan=0.0, posinf=0.0)
    return ref, torch.nan_to_num(atol, nan=0.0)


def _ln_run(y, din, dout, *, scale=None, shift=None, residual=None, add_rows=None, res_div=1, res_mod=0, eps=1e-5,
            want_f32=True, what=""):
    """Run the kernel on `y` (fp32 values, stored as `din` in a wider buffer) with both outputs in wider buffers; check
    both against the float64 reference, the 16-bit output against the rounding of the fp32 one, and the padding."""
    from aurora_b200 import cabi

    rows, dim = y.shape
    ybuf, y16 = _padded(rows, dim, DTYPES[din], left=16)
    y16.copy_(y)
    b32, o32 = _padded(rows, dim, F32)
    b16, o16 = _padded(rows, dim, DTYPES[dout])
    cabi.ln_mod_residual(y16, scale=scale, shift=shift, residual=residual, add_rows=add_rows, res_div=res_div,
                         res_mod=res_mod, out_f32=o32 if want_f32 else None, out_bf16=o16, eps=eps)
    torch.cuda.synchronize()
    ref, atol = _ln_reference(y16, scale, shift, residual, add_rows, res_div, res_mod, eps)
    assert _untouched(b16, 8, dim), f"{what}: 16-bit store outside [0, dim)"
    _check16(o16, ref, floor=atol, what=f"{what} 16-bit")
    if want_f32:
        assert _untouched(b32, 8, dim), f"{what}: fp32 store outside [0, dim)"
        _check32(o32, ref, atol, what=f"{what} fp32")
        assert _same_bits_or_nan(o16, _round16(o32, o16.dtype)), f"{what}: 16-bit output is not the rounding of fp32"
    else:
        assert bool((b32 == SENTINEL).all())
    return o32, o16, ref


@pytest.mark.parametrize("dim", LN_WIDTHS)
@pytest.mark.parametrize("din,dout", LN_PAIRS)
def test_ln_mod_residual_widths_and_dtypes(dim, din, dout):
    g = torch.Generator(device=DEV).manual_seed(dim)
    rows = 77  # not a multiple of the 8 rows of a CTA
    y = torch.randn(rows, dim, device=DEV, generator=g) * 3 + 1
    scale = torch.randn(dim, device=DEV, generator=g)
    shift = torch.randn(dim, device=DEV, generator=g)
    res_buf, res = _padded(rows, dim, F32, left=4, right=4, fill=0.0)  # ld_res > dim as well
    res.copy_(torch.randn(rows, dim, device=DEV, generator=g) * 2)
    _ln_run(y, din, dout, scale=scale, shift=shift, residual=res, what=f"dim={dim} {din}->{dout}")


@pytest.mark.parametrize("din,dout", LN_PAIRS)
def test_ln_mod_residual_broadcast_add_rows_and_absent_affine(din, dout):
    """Perceiver latents: residual row (row / nloc) % lq, add_rows row % nloc; scale / shift absent; 16-bit only."""
    g = torch.Generator(device=DEV).manual_seed(11)
    nloc, lq, dim = 37, 3, 520
    rows = lq * nloc
    y = torch.randn(rows, dim, device=DEV, generator=g)
    lat = torch.randn(lq, dim, device=DEV, generator=g)
    add = torch.randn(nloc, dim, device=DEV, generator=g)
    _ln_run(y, din, dout, residual=lat, res_div=nloc, res_mod=lq, add_rows=add, what="broadcast")
    _ln_run(y, din, dout, shift=torch.randn(dim, device=DEV, generator=g), what="shift only")
    _ln_run(y, din, dout, scale=torch.randn(dim, device=DEV, generator=g), want_f32=False, what="scale only, 16-bit")


@pytest.mark.parametrize("dim", [200, 1000, 2048])
@pytest.mark.parametrize("din,dout", LN_PAIRS)
def test_ln_mod_residual_large_mean_small_spread(dim, din, dout):
    """300 + N(0, 1): the mean is 300 times the spread, so a one-pass variance (E[y^2] - mean^2) loses ~1e-2."""
    g = torch.Generator(device=DEV).manual_seed(dim + 1)
    y = 300 + torch.randn(45, dim, device=DEV, generator=g)
    _ln_run(y, din, dout, scale=torch.randn(dim, device=DEV, generator=g) * 2,
            shift=torch.randn(dim, device=DEV, generator=g) * 0.1, what="mean 300")


@pytest.mark.parametrize("din,dout", LN_PAIRS)
def test_ln_mod_residual_overflow_saturates_only_fp16(din, dout):
    """Outputs beyond +-65504 (and +-inf from the residual): fp16 stores +-65504; bf16 and fp32 keep the value."""
    g = torch.Generator(device=DEV).manual_seed(5)
    rows, dim = 21, 264
    y = torch.randn(rows, dim, device=DEV, generator=g)
    res = torch.randn(rows, dim, device=DEV, generator=g)
    res[:, 3], res[:, 100], res[:, 263] = 1e5, -7e4, 65520.0  # 65520 would round to inf in an unsaturated fp16 store
    res[2, 7], res[5, 8] = INF, -INF
    o32, o16, _ = _ln_run(y, din, dout, residual=res, what="overflow")
    if dout == "fp16":
        assert bool((o16[:, 3] == FP16_MAX).all()) and bool((o16[:, 100] == -FP16_MAX).all())
        assert o16[2, 7].item() == FP16_MAX and o16[5, 8].item() == -FP16_MAX
    else:
        assert bool((o16[:, 3].float() > 9e4).all()) and math.isinf(o16[2, 7].item())


@pytest.mark.parametrize("din,dout", LN_PAIRS)
def test_ln_mod_residual_nan_row(din, dout):
    """One NaN element makes its row NaN in every output; the other rows are untouched by it."""
    g = torch.Generator(device=DEV).manual_seed(6)
    rows, dim = 19, 1032
    y = torch.randn(rows, dim, device=DEV, generator=g)
    y[4, 517] = NAN
    o32, o16, _ = _ln_run(y, din, dout, scale=torch.randn(dim, device=DEV, generator=g),
                          shift=torch.randn(dim, device=DEV, generator=g), what="NaN row")
    assert bool(torch.isnan(o16[4].float()).all()) and bool(torch.isnan(o32[4]).all())
    assert not bool(torch.isnan(o16[torch.arange(rows, device=DEV) != 4].float()).any())


# ------------------------------------------------------------------------------------------------
# Perceiver attention: softmax(q k^T / sqrt(dh)) v per (location, head)
# ------------------------------------------------------------------------------------------------
# (lq, lk, heads, head_dim, nloc); the kernel is chosen by the shape (ab_perceiver_attention): few-keys when lk <= 4,
# lq > lk and D % 256 == 0 (E = 16 when D % 512 == 0, else 8), the general kernel with E = D / 32 otherwise.
PERC_GENERAL = {
    "E4_D128": (3, 13, 4, 32, 333),
    "E8_D256_small_encoder": (3, 13, 8, 32, 1),
    "E16_D512_1p3B_encoder": (3, 13, 16, 32, 37),
    "E32_D1024_dh32": (3, 13, 32, 32, 37),
    "E32_D1024_dh64": (3, 13, 16, 64, 5),
    "E4_lk1": (2, 1, 4, 32, 33),
    "E8_lk4_lq3": (3, 4, 8, 32, 11),
}
PERC_FEWKEYS = {
    "fk_E8_D256_dh32": (13, 3, 8, 32, 333),
    "fk_E8_D256_dh64": (13, 3, 4, 64, 1),
    "fk_E16_D512_small_decoder": (13, 3, 8, 64, 37),
    "fk_E16_D1024_1p3B_decoder": (13, 3, 16, 64, 37),
    "fk_E16_lk1": (13, 1, 16, 32, 5),
    "fk_E8_lk4": (13, 4, 8, 32, 7),
    "fk_E16_lk4_nloc1": (5, 4, 32, 32, 1),
}
PERC_CASES = {**PERC_GENERAL, **PERC_FEWKEYS}


def _perc_inputs(lq, lk, heads, dh, nloc, logits, g):
    """q [lq, D] fp32 and K | V [lk * nloc, 2D] fp32 values.  logits = "random": O(1) scores;
    "ascending" / "descending": for query 0 the scores of the keys run from -60 to +60 (largest last: every key raises
    the running maximum, so the online softmax rescales at every step) or from +60 to -60 (largest first)."""
    d = heads * dh
    q = torch.randn(lq, d, device=DEV, generator=g)
    k = torch.randn(lk, nloc, heads, dh, device=DEV, generator=g)
    v = torch.randn(lk, nloc, heads, dh, device=DEV, generator=g) * 2
    if logits != "random":
        t = torch.linspace(-60.0, 60.0, lk, device=DEV) if lk > 1 else torch.tensor([60.0], device=DEV)
        if logits == "descending":
            t = t.flip(0)
        q0 = q[0].view(heads, dh)
        dirn = q0 * math.sqrt(dh) / (q0 * q0).sum(-1, keepdim=True)  # q0 . dirn / sqrt(dh) = 1 per head
        k = t.view(lk, 1, 1, 1) * dirn.view(1, 1, heads, dh) + 0.05 * k
    kv = torch.cat((k.reshape(lk * nloc, d), v.reshape(lk * nloc, d)), 1)
    return q, kv


def _perc_reference(q, kv, lq, lk, heads, dh, nloc):
    """float64 attention of the decoded K / V, and the floor for cancelling P.V sums: 8 * 2^-20 * max|V| of the
    (location, head).  The kernel's __expf is accurate to ~2^-21 relative for the score differences used here and the
    weighted sum adds a few fp32 roundings of terms bounded by max|V|."""
    d = heads * dh
    kd = kv[:, :d].double().view(lk, nloc, heads, dh).permute(1, 2, 0, 3)        # (nloc, heads, lk, dh)
    vd = kv[:, d:].double().view(lk, nloc, heads, dh).permute(1, 2, 0, 3)
    qh = q.double().view(lq, heads, dh).permute(1, 0, 2)[None]                   # (1, heads, lq, dh)
    o = torch.softmax(qh @ kd.transpose(-1, -2) / math.sqrt(dh), -1) @ vd        # (nloc, heads, lq, dh)
    ref = o.permute(2, 0, 1, 3).reshape(lq * nloc, d)
    vmax = vd.abs().amax(dim=(2, 3))                                              # (nloc, heads)
    floor = (8 * 2.0**-20 * vmax)[None, :, :, None].expand(lq, nloc, heads, dh).reshape(lq * nloc, d)
    return ref, floor


@pytest.mark.parametrize("logits", ["random", "ascending", "descending"])
@pytest.mark.parametrize("case", sorted(PERC_CASES))
@pytest.mark.parametrize("dt", ["fp16", "bf16"])
def test_perceiver_attention(case, dt, logits):
    """K | V and the output are column slices of wider buffers (ld_kv > 2D, ld_out > D)."""
    from aurora_b200 import cabi

    lq, lk, heads, dh, nloc = PERC_CASES[case]
    d = heads * dh
    g = torch.Generator(device=DEV).manual_seed(lq * 1000 + lk * 100 + heads + dh + nloc)
    q, kv32 = _perc_inputs(lq, lk, heads, dh, nloc, logits, g)
    kv_buf, kv = _padded(lk * nloc, 2 * d, DTYPES[dt], left=8, right=16)
    kv.copy_(kv32)
    out_buf, out = _padded(lq * nloc, d, DTYPES[dt])
    cabi.perceiver_attention(q, kv, out, nloc=nloc, num_heads=heads, head_dim=dh)
    torch.cuda.synchronize()
    ref, floor = _perc_reference(q, kv, lq, lk, heads, dh, nloc)
    assert _untouched(out_buf, 8, d), "store outside the output view"
    _check16(out, ref, floor=floor, what=f"{case} {dt} {logits}")


# ------------------------------------------------------------------------------------------------
# patchify: fields -> normalised, transformed, im2col'ed 16-bit A operand
# ------------------------------------------------------------------------------------------------
PLAIN, CLAMP, LOGC, NAN0, DENS, SIN, COS = 0, 1, 2, 3, 4, 5, 6
PATCH_PATHS = {  # (p, h, w, offset of the field pointer in floats)
    "p4_vector": (4, 8, 16, 0),
    "p4_unaligned_scalar": (4, 8, 16, 1),
    "p3_scalar": (3, 9, 12, 0),
    "p10_scalar": (10, 20, 30, 0),
}
SPECIALS = [NAN, INF, -INF, 7e4, -7e4, 65520.0, 0.0, -0.0, 1e-5, 1e-4, 2.4, 2.6, -1.0, 1e-6]


def _nan_to_num_f32(v):  # torch.nan_to_num(v, nan=0) on a float32 tensor: +-inf -> +-FLT_MAX
    return torch.nan_to_num(v, nan=0.0, posinf=FLT_MAX, neginf=-FLT_MAX)


def _transform_reference(x, loc, scale, transform, w0, w1, wb):
    """float64 restatement of Batch.normalise and the encoder hooks (positive clamp, AirPollution log combiner, the wave
    model's nan_to_num / density / sin / cos), with NaN kept by every clamp as torch.clamp keeps it."""
    v = (x.double() - loc) / scale
    if transform == NAN0:
        return _nan_to_num_f32(v)
    if transform == DENS:
        return (~torch.isnan(v)).double()
    if transform in (SIN, COS):
        f = torch.sin if transform == SIN else torch.cos
        return _nan_to_num_f32(f(v * (math.pi / 180.0)))
    if transform >= CLAMP:
        v = v.clamp(min=0.0)
    if transform == LOGC:
        eps = float(np.float32(1e-4))
        v = w0 * v.clamp(0.0, 2.5) + w1 * ((torch.log(v.clamp(min=eps)) - math.log(eps)) / -math.log(eps)) + wb
    return v


@pytest.mark.parametrize("path", sorted(PATCH_PATHS))
@pytest.mark.parametrize("dt", ["fp16", "bf16"])
def test_patchify_transforms_and_layout(path, dt):
    """One field per transform plus two constant fields; every field carries NaN, +-inf and values beyond 65504.  The K
    padding past the last field keeps what the buffer held."""
    from aurora_b200 import cabi

    p, h, w, off = PATCH_PATHS[path]
    t = 2
    g = torch.Generator(device=DEV).manual_seed(p * 100 + off)
    transforms = [PLAIN, CLAMP, LOGC, NAN0, DENS, SIN, COS]
    params = [(0.0, 1.0), (1.5, 2.0), (0.0, 1.0), (-3.0, 0.5), (2.0, 3.0), (10.0, 1.0), (0.0, 2.0)]
    storage, planes, descs = [], [], []
    for i, (tr, (loc, scale)) in enumerate(zip(transforms, params)):
        x = torch.randn(t * h * w, device=DEV, generator=g) * 3
        if tr in (SIN, COS):
            x = x * 120  # degrees
        x[: len(SPECIALS)] = torch.tensor(SPECIALS, device=DEV)
        x = x[torch.randperm(t * h * w, device=DEV, generator=g)]
        buf = torch.empty(t * h * w + 4, device=DEV)  # 16-byte aligned; `off` floats in when testing the scalar path
        buf[off:off + t * h * w] = x
        field = buf[off:off + t * h * w].view(t, h, w)
        storage.append(buf)
        d = cabi.AbFieldIn()
        d.ptr, d.stride_t, d.loc, d.scale, d.transform = field.data_ptr(), h * w, loc, scale, tr
        d.w0, d.w1, d.wb = 0.4, 0.6, 0.05
        descs.append(d)
        planes.append(_transform_reference(field, loc, scale, tr, float(np.float32(0.4)), float(np.float32(0.6)),
                                           float(np.float32(0.05))))
    static = storage[0][off:off + h * w].view(h, w)  # a static field: stride_t = 0
    d = cabi.AbFieldIn()
    d.ptr, d.stride_t, d.loc, d.scale = static.data_ptr(), 0, 0.5, 2.0
    descs.append(d)
    planes.append(((static.double() - 0.5) / 2.0)[None].expand(t, h, w))
    for cval in (1e5, -3.25):  # constant fields (no pointer)
        c = cabi.AbFieldIn()
        c.ptr, c.const_value, c.scale = None, cval, 1.0
        descs.append(c)
        planes.append(torch.full((t, h, w), cval, device=DEV, dtype=torch.float64))
    nv = len(descs)
    k = nv * t * p * p
    kpad = (k + 63) // 64 * 64 + 64
    out = torch.full(((h // p) * (w // p), kpad), SENTINEL, device=DEV, dtype=DTYPES[dt])
    cabi.patchify(descs, t, h, w, p, out)
    torch.cuda.synchronize()
    x = torch.stack(planes, 0)  # (V, T, H, W)
    ref = x.view(nv, t, h // p, p, w // p, p).permute(2, 4, 0, 1, 3, 5).reshape((h // p) * (w // p), k)
    # The kernel forms the radian argument of sin / cos in fp32 (v * 0.0174532925f): that product's rounding moves the
    # result by up to 2^-24 |argument|, plus sinf's own ~2^-22.  Every other transform is exact to far below one ulp.
    floor = torch.zeros(nv, t, h, w, device=DEV, dtype=torch.float64)
    for i, tr in enumerate(transforms):
        if tr in (SIN, COS):
            loc, scale = params[i]
            arg = ((storage[i][off:off + t * h * w].view(t, h, w).double() - loc) / scale * (math.pi / 180)).abs()
            floor[i] = 2.0**-22 * (1 + torch.nan_to_num(arg, nan=0.0, posinf=0.0))
    floor = floor.view(nv, t, h // p, p, w // p, p).permute(2, 4, 0, 1, 3, 5).reshape((h // p) * (w // p), k)
    _check16(out[:, :k], ref, floor=floor, what=f"{path} {dt}")
    assert bool((out[:, k:] == SENTINEL).all()), "a store landed in the K padding"


@pytest.mark.parametrize("path", ["p4_vector", "p3_scalar"])
@pytest.mark.parametrize("transform", [PLAIN, CLAMP, LOGC])
@pytest.mark.parametrize("dt", ["fp16", "bf16"])
def test_patchify_keeps_nan(path, transform, dt):
    """A NaN in a field with no transform, the positive clamp or the log combiner comes out as NaN (torch.clamp keeps
    it), not as a clamp bound or a saturated value."""
    from aurora_b200 import cabi

    p, h, w, _ = PATCH_PATHS[path]
    x = torch.rand(1, h, w, device=DEV) + 0.5
    x[0, 1, 2] = NAN
    d = cabi.AbFieldIn()
    d.ptr, d.stride_t, d.loc, d.scale, d.transform = x.data_ptr(), h * w, 0.0, 1.0, transform
    d.w0, d.w1, d.wb = 0.4, 0.6, 0.05
    out = torch.zeros((h // p) * (w // p), 64, device=DEV, dtype=DTYPES[dt])
    cabi.patchify([d], 1, h, w, p, out)
    torch.cuda.synchronize()
    nan = torch.isnan(out[:, : p * p].float())
    assert int(nan.sum()) == 1 and bool(nan[0, p + 2]), out[0, : p * p].tolist()


# ------------------------------------------------------------------------------------------------
# unpatchify: head output [L, V * P * P] fp32 -> per-variable planes in physical units
# ------------------------------------------------------------------------------------------------
def _unpatch(y, col, h, w, p):
    """float64 plane [h, w] of the p * p columns starting at `col` of the head output."""
    return y[:, col:col + p * p].double().reshape(h // p, w // p, p, p).permute(0, 2, 1, 3).reshape(h, w)


def _unpatch32(y, col, h, w, p):
    return y[:, col:col + p * p].reshape(h // p, w // p, p, p).permute(0, 2, 1, 3).reshape(h, w)


def test_unpatchify_angle_remainder_matches_float32_torch():
    """rad2deg(atan2(sin, cos)) % 360 with torch's floored remainder, in float32 as the reference model computes it: at
    0, -0, the axes and tiny negative angles (where -1e-6 + 360 rounds to 360.0 in float32, not to 359.999999)."""
    from aurora_b200 import cabi

    p, h, w = 4, 8, 16
    g = torch.Generator(device=DEV).manual_seed(7)
    y = torch.randn(h * w // (p * p), 2 * p * p + 8, device=DEV, generator=g)
    pairs = [(0.0, 1.0), (-0.0, 1.0), (0.0, -1.0), (-0.0, -1.0), (1.0, 0.0), (-1.0, 0.0), (0.0, 0.0), (-0.0, -0.0),
             (-1e-7, 1.0), (-1e-30, 1.0), (-1e-4, 1.0), (1e-7, 1.0), (-1e-7, -1.0), (-3.0, 4.0), (-2.0, -5.0),
             (-1e-6, 1e3), (-1e-20, 1e-3), (5.0, -1e-7)]
    sn, cs = torch.tensor(pairs, device=DEV).T
    for col, vals in ((0, sn), (p * p, cs)):  # the first entries of the sine / cosine columns
        block = y[:, col:col + p * p].clone()
        block.view(-1)[: len(pairs)] = vals
        y[:, col:col + p * p] = block
    out = torch.full((h, w), NAN, device=DEV)
    d = cabi.AbFieldOut()
    d.ptr, d.loc, d.scale, d.col, d.cos_col = out.data_ptr(), 0.0, 1.0, 0, p * p
    cabi.unpatchify([d], y, h, w, p)
    torch.cuda.synchronize()
    s32, c32 = _unpatch32(y, 0, h, w, p).cpu(), _unpatch32(y, p * p, h, w, p).cpu()
    deg = torch.rad2deg(torch.atan2(s32, c32))
    ref = torch.remainder(deg, 360.0)
    assert ref.dtype == F32 and float(ref.max()) <= 360.0
    # atan2f and the float32 degree conversion are within 2 ulp of torch's float32 result; the remainder's + 360 adds one
    # rounding at the result.
    tol = 4 * _ulp(deg, F32) + _ulp(ref, F32)
    o = out.cpu().double()
    _report((o - ref.double()).abs(), tol, torch.ones_like(o, dtype=torch.bool), "angle")
    assert bool((o >= 0).all() & (o <= 360).all())
    assert bool((o[ref == 360.0] == 360.0).all()) and int((ref == 360.0).sum()) >= 2


def test_unpatchify_density_mask_and_nan_placement():
    """density = sigmoid(logit) * (mask > mask_min); the value is NaN where density < 0.5 (exactly 0.5 is kept), else
    value * mask-bit in physical units."""
    from aurora_b200 import cabi

    p, h, w = 4, 8, 16
    l = h * w // (p * p)
    g = torch.Generator(device=DEV).manual_seed(8)
    y = torch.randn(l, 2 * p * p, device=DEV, generator=g) * 2
    logit = torch.randn(l, p * p, device=DEV, generator=g) * 3
    logit = torch.where(logit.abs() < 1e-3, torch.full_like(logit, 1e-3), logit)  # fp32 and fp64 agree on the side
    specials = torch.tensor([0.0, 0.0, 0.0, -1e-3, 1e-3, 60.0, -60.0, 100.0, -100.0, 0.0, 1e-6, -1e-6], device=DEV)
    logit.view(-1)[: len(specials)] = specials
    y[:, p * p:] = logit
    y[0, 2] = NAN  # a NaN value at pixel (0, 2), where the density keeps it (logit 0, mask just above mask_min)
    mask = (torch.rand(h, w, device=DEV, generator=g) > 0.3).float()
    mask[0, :4] = torch.tensor([1.0, 0.5, 0.50000006, NAN], device=DEV)  # with mask_min = 0.5: kept, masked, kept, masked
    mask[1, :3] = 1.0
    out = torch.full((h, w), SENTINEL, device=DEV)
    d = cabi.AbFieldOut()
    d.ptr, d.loc, d.scale, d.col, d.dens_col, d.mask, d.mask_min = out.data_ptr(), 1.5, 2.0, 0, p * p, mask.data_ptr(), 0.5
    cabi.unpatchify([d], y, h, w, p)
    torch.cuda.synchronize()
    val, lg = _unpatch(y, 0, h, w, p), _unpatch(y, p * p, h, w, p)
    m = (mask.double() > 0.5).double()
    dens = m * torch.sigmoid(lg)
    ref = torch.where(dens < 0.5, torch.full_like(val, NAN), val * m) * 2.0 + 1.5
    _check32(out, ref, 2.0**-21 * (val.abs() * 2.0 + 1.5), what="density")
    assert not math.isnan(out[0, 0].item())          # logit 0, mask 1: density exactly 0.5 keeps the value
    assert math.isnan(out[0, 1].item()) and math.isnan(out[0, 2].item())  # mask == mask_min is masked; NaN value kept
    assert torch.isnan(out).sum() > 0 and (~torch.isnan(out)).sum() > 0


def test_unpatchify_modulation_and_clamps_keep_nan():
    """pred = model + (1 + mod) * prev (normalised), then clamp_max1 / clamp_min0, then physical units; a NaN model
    output or previous state stays NaN through the clamps (torch.clamp keeps it); columns past the fields' untouched."""
    from aurora_b200 import cabi

    p, h, w = 3, 9, 12
    l = h * w // (p * p)
    g = torch.Generator(device=DEV).manual_seed(9)
    y = torch.randn(l, 4 * p * p + 5, device=DEV, generator=g) * 2
    y[0, 0], y[1, p * p + 4], y[2, 3 * p * p + 1] = NAN, NAN, NAN  # in field 0, field 1 and field 2's value columns
    y[3, 0], y[3, p * p] = 1e30, -1e30
    prev = torch.randn(h, w, device=DEV, generator=g) * 3 + 2
    prev[5, 7] = NAN
    outs = [torch.full((h, w), SENTINEL, device=DEV) for _ in range(3)]
    descs = []
    for i, (loc, scale) in enumerate([(1.0, 3.0), (-2.0, 0.5), (0.25, 4.0)]):
        d = cabi.AbFieldOut()
        d.ptr, d.loc, d.scale, d.col = outs[i].data_ptr(), loc, scale, i * p * p
        descs.append(d)
    descs[0].mod_col, descs[0].prev, descs[0].clamp_max1 = 2 * p * p, prev.data_ptr(), 1
    descs[1].mod_col, descs[1].prev, descs[1].clamp_min0 = 2 * p * p, prev.data_ptr(), 1
    descs[2].col, descs[2].clamp_min0, descs[2].clamp_max1 = 3 * p * p, 1, 1
    cabi.unpatchify(descs, y, h, w, p)
    torch.cuda.synchronize()
    mod = _unpatch(y, 2 * p * p, h, w, p)
    for i, d in enumerate(descs):
        val = _unpatch(y, d.col, h, w, p)
        loc, scale = float(d.loc), float(d.scale)
        mag = val.abs() * scale
        if d.mod_col >= 0:
            prev_n = (prev.double() - loc) / scale
            val = val + (1 + mod) * prev_n
            mag = mag + (1 + mod).abs() * (prev.double().abs() + abs(loc))
        if d.clamp_max1:
            val = val.clamp(max=1.0)
        if d.clamp_min0:
            val = val.clamp(min=0.0)
        ref = val * scale + loc
        _check32(outs[i], ref, 2.0**-20 * (torch.nan_to_num(mag, nan=0.0) + abs(loc)), what=f"field {i}")
    # NaN model outputs at pixels (0, 0), (1, 4), (0, 7) of fields 0, 1, 2; the NaN previous state at (5, 7)
    assert [int(torch.isnan(o).sum()) for o in outs] == [2, 2, 1]
    assert math.isnan(outs[0][0, 0].item()) and math.isnan(outs[1][1, 4].item()) and math.isnan(outs[2][0, 7].item())
    assert outs[0][0, 9].item() == 4.0 and outs[1][0, 9].item() == -2.0  # +-1e30 clamped to 1 / 0, in physical units


# ------------------------------------------------------------------------------------------------
# GEMM epilogues with 16-bit (fp16 / bf16) outputs
# ------------------------------------------------------------------------------------------------
GEMM_CASES = {  # (m, n, k, epilogue)
    "tma_coop256_k256": (300, 264, 256, "tma"),    # N > 128: 128 x 256 tiles, 8 live columns in the second
    "tma_coop256": (300, 264, 1088, "tma"),        # 128 x 256, K tail past 1024
    "tma_coop128": (200, 96, 128, "tma"),          # N <= 128: 128 x 128
    "direct_dual": (300, 131, 256, "dual"),        # fp32 + 16-bit outputs, residual: direct epilogue (odd N: to16 tail)
    "direct_dual_coop256": (257, 520, 512, "dual"),  # direct epilogue on 128 x 256 tiles, 8 live columns in the third
    "direct_unaligned": (200, 200, 128, "unaligned"),  # 16-bit output 2 bytes off 16-byte alignment: scalar stores
}


def _gemm_inputs(m, n, k, dt, g):
    """A / W with a NaN in one A row and one W row, and a block of products beyond 65504 in both signs."""
    a = torch.randn(m, k, device=DEV, generator=g)
    w = torch.randn(n, k, device=DEV, generator=g) / k**0.5
    a[7, k // 3] = NAN
    w[n - 2, k - 1] = NAN
    a[m - 3] = 100.0
    w[5], w[6] = 100.0, -100.0  # rows m - 3 x columns 5 / 6: +-1e4 * K, beyond fp16
    return a.to(DTYPES[dt]), w.to(DTYPES[dt])


def _gemm_reference(a, w, bias=None, residual=None):
    """float64 product of the decoded operands on the CPU, and the floor for cancelling sums: the wgmma accumulates in
    fp32, k-step by k-step, so its error is a few times 2^-24 * sum_k |a_k w_k| for the K used here: 2^-18 of that sum
    bounds it with room for the accumulator's rounding order."""
    ad, wd = a.double().cpu(), w.double().cpu()
    ref = ad @ wd.T
    absum = torch.nan_to_num(ad.abs() @ wd.abs().T, nan=0.0)
    floor = 2.0**-18 * absum
    if bias is not None:
        ref = ref + bias.double().cpu()
        floor = floor + 2.0**-22 * bias.double().cpu().abs()
    if residual is not None:
        ref = ref + residual.double().cpu()
        floor = floor + 2.0**-22 * residual.double().cpu().abs()
    return ref.to(DEV), floor.to(DEV)


@pytest.mark.parametrize("case", sorted(GEMM_CASES))
@pytest.mark.parametrize("dt", ["fp16", "bf16"])
def test_gemm_16bit_epilogues_nan_and_saturation(case, dt):
    from aurora_b200 import cabi

    m, n, k, epi = GEMM_CASES[case]
    g = torch.Generator(device=DEV).manual_seed(m + n + k)
    a, w = _gemm_inputs(m, n, k, dt, g)
    bias = torch.randn(n, device=DEV, generator=g)
    residual = torch.randn(m, n, device=DEV, generator=g) if epi == "dual" else None
    left = 1 if epi == "unaligned" else 8
    b16, o16 = _padded(m, n, DTYPES[dt], left=left)
    o32 = torch.full((m, n), SENTINEL, device=DEV) if epi == "dual" else None
    cabi.gemm(a, w, bias=bias, residual=residual, out_f32=o32, out_bf16=o16)
    torch.cuda.synchronize()
    ref, floor = _gemm_reference(a, w, bias, residual)
    assert _untouched(b16, left, n), "store outside the output view"
    _check16(o16, ref, floor=floor, what=f"{case} {dt}")
    if o32 is not None:
        _check32(o32, ref, floor, what=f"{case} fp32")
        assert _same_bits_or_nan(o16, _round16(o32, o16.dtype)), "16-bit output is not the rounding of the fp32 one"
    nan = torch.isnan(o16.float())
    assert bool(nan[7].all()) and bool(nan[:, n - 2].all()) and int(nan.sum()) == m + n - 1
    big = o16[m - 3, 5:7].float()
    if dt == "fp16":
        assert big.tolist() == [FP16_MAX, -FP16_MAX]
    else:
        assert float(big[0]) > 1e6 and float(big[1]) < -1e6


@pytest.mark.parametrize("n", [512, 1024])
@pytest.mark.parametrize("dt", ["fp16", "bf16"])
def test_gemm_ln_residual_nan_and_saturation(n, dt):
    """residual + LN(a @ w.T + bias) * scale + shift: a NaN in an A row makes that row NaN in both outputs, a NaN in a W
    row reaches every row through the row statistics; outputs beyond +-65504 saturate in fp16 only."""
    from aurora_b200 import cabi

    assert cabi.gemm_ln_supported(n)
    m, k = 200, 256
    g = torch.Generator(device=DEV).manual_seed(n)
    a = torch.randn(m, k, device=DEV, generator=g)
    w = torch.randn(n, k, device=DEV, generator=g) / k**0.5
    a[9, 17] = NAN
    a, w = a.to(DTYPES[dt]), w.to(DTYPES[dt])
    bias, scale, shift = (torch.randn(n, device=DEV, generator=g) for _ in range(3))
    res = torch.randn(m, n, device=DEV, generator=g) * 3
    res[:, 4], res[:, 300], res[11, 5] = 1e5, -7e4, INF
    o32 = torch.full((m, n), SENTINEL, device=DEV)
    b16, o16 = _padded(m, n, DTYPES[dt])
    cabi.gemm_ln_residual(a, w, bias=bias, scale=scale, shift=shift, residual=res, out_f32=o32, out_bf16=o16)
    torch.cuda.synchronize()
    ad, wd = a.double().cpu(), w.double().cpu()
    y = (ad @ wd.T + bias.double().cpu()).to(DEV)
    gemm_err = (2.0**-18 * torch.nan_to_num(ad.abs() @ wd.abs().T, nan=0.0)).to(DEV).amax(1, keepdim=True)
    mu = y.mean(1, keepdim=True)
    rstd = ((y - mu).pow(2).mean(1, keepdim=True) + 1e-5).rsqrt()
    nrm = (y - mu) * rstd * scale.double()
    ref = nrm + shift.double() + res.double()
    # the GEMM's error and the one-pass statistics' rounding (2^-20 of max|y| per row) pass through rstd * |scale|;
    # the modulation and residual add a few fp32 roundings of their terms
    cond = (gemm_err + 2.0**-20 * y.abs().amax(1, keepdim=True)) * rstd
    mag = nrm.abs() + shift.double().abs() + res.double().abs()
    atol = torch.nan_to_num(cond * scale.double().abs() + 2.0**-21 * mag, nan=0.0, posinf=0.0)
    assert _untouched(b16, 8, n)
    _check32(o32, ref, atol, what=f"gemm_ln n={n} fp32")
    _check16(o16, ref, floor=atol, what=f"gemm_ln n={n} {dt}")
    assert _same_bits_or_nan(o16, _round16(o32, o16.dtype))
    assert bool(torch.isnan(o16[9].float()).all()) and int(torch.isnan(o16.float()).sum()) == n
    if dt == "fp16":
        others = torch.arange(m, device=DEV) != 9
        assert bool((o16[others, 4] == FP16_MAX).all()) and bool((o16[others, 300] == -FP16_MAX).all())
        assert o16[11, 5].item() == FP16_MAX
    # a NaN in one W row: that column is NaN in every row, and so is every row's mean
    w[n - 1, 3] = NAN
    cabi.gemm_ln_residual(a, w, bias=bias, scale=scale, shift=shift, residual=res, out_f32=o32, out_bf16=o16)
    torch.cuda.synchronize()
    assert bool(torch.isnan(o32).all()) and bool(torch.isnan(o16.float()).all())


# ------------------------------------------------------------------------------------------------
# whole model
# ------------------------------------------------------------------------------------------------
def test_whole_model_keeps_a_planted_nan():
    """One NaN in a surface field (a variable without a NaN-to-zero transform) of the tiny model, run with the default
    fp16 encoder / decoder: every output variable is NaN on the planted pixel's patch, as in the reference, which
    computes in fp32.  The CPU oracle of the reference algorithm is checked on the same batch."""
    import aurora_b200 as ab
    from oracle import aurora_oracle as O
    from tests import fixtures as fx

    cfg = fx.CONFIGS["tiny"]
    sd = fx.make_state_dict(cfg, seed=4)
    model = ab.Aurora(**fx.our_kwargs(cfg))
    model.load_state_dict(sd, strict=True)
    model = model.to(DEV).eval()
    model.encoding_device = "cpu"
    batch = fx.make_batch(cfg, 32, 64, levels=fx.LEVELS4, seed=4)
    r, c, p = 9, 21, cfg.patch_size
    batch.surf_vars["2t"][0, -1, r, c] = NAN
    pred = model.forward(batch)
    torch.cuda.synchronize()
    assert model._get_engine().ed == torch.float16
    rows, cols = slice(r // p * p, r // p * p + p), slice(c // p * p, c // p * p + p)
    with torch.inference_mode():
        ref = O.forward(cfg, sd, batch, dtype=torch.float32)
    for got in (pred, ref):
        for grp, d in (("surf", got.surf_vars), ("atmos", got.atmos_vars)):
            for name, v in d.items():
                patch = v[..., rows, cols]
                assert bool(torch.isnan(patch).all()), (grp, name, int(torch.isnan(patch).sum()), patch.numel())
