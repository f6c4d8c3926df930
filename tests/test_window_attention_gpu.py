"""Window attention (`ab_window_attention`) against a float64 reference of the same operation, on every kernel and
gather path: the wgmma kernel for full 144-token windows with its TMA row-box gather at every box size the host picks
and with its cp.async gather, and the generic mma.sync kernel on clamped windows, with a dense bias, and (forced) on
full windows.

Reference.  The bf16 `qkv`, `pad_qkv` and fp32 `bias` the kernel reads are decoded to float64; tokens are routed
through the oracle's gather map and group ids (`oracle.windows`, pinned to the reference model), cross-group logits get
-100, and softmax(q k^T / 8 + bias + mask) V is evaluated in float64, window chunk by window chunk and head by head.

Per-element bound, with u = 2^-8 (bf16 unit roundoff), A the exact softmax and (A|V|)_i = sum_j A_ij |V_j|:
* P is rounded to bf16 before P V while the normaliser is the fp32 sum of the unrounded p, so the rounding of P moves
  output i by at most u (A|V|)_i; the bf16 store of the output adds u |ref_i|.
* The logits carry an absolute error e_i per query row: the fp32 tensor-core accumulation of q.k over 64 products,
  GAMMA_QK max_j sum_k |q_ik k_jk| / 8 (products of bf16 values are exact in fp32; the accumulation is taken to lose
  up to 2^-23 relative per addition, as a truncating adder does), plus a few fp32 roundings of the largest logit
  magnitude of the row (bias and mask additions, the exp2-domain scale, the max subtraction).  Logit errors of at
  most e move every softmax weight by a factor within exp(+-2e), so the output by at most expm1(2 e_i) (A|V|)_i.
* ex2.approx (2 ulp, taken as 2^-21) in numerator and normaliser, the fp32 sums over <= 144 keys of P V and of p,
  and the final scaling: SMALL (A|V|)_i, about 3e-5 relative.  No absolute floor is needed: every term scales with
  (A|V|)_i or |ref_i|, and a subnormal p flushed to zero by ex2.approx.ftz moves the output by < 2^-126 |V|.
NaN must come out exactly where float64 torch puts it: a NaN logit poisons its whole row (masked or not), and
0 * NaN in P V is NaN.

Measured on an H100 80GB HBM3 at a 700 W power limit, the largest error was 0.84 of the bound on the wgmma kernel
(TMA and cp.async gathers alike: their outputs are bit-identical), 0.75 on the generic kernel on clamped windows, 0.81
on the generic kernel forced onto full windows and 0.73 with a bias."""

import hashlib
import math
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import windows as W

pytestmark = pytest.mark.gpu
DEV = "cuda"
WS0 = (2, 6, 12)
SHIFT = (1, 3, 6)
BF16 = torch.bfloat16
U = 2.0 ** -8
U32 = 2.0 ** -24
GAMMA_QK = 64 * 2.0 ** -23
SMALL = 2 * 2.0 ** -21 + 144 * 2.0 ** -23 + 144 * U32 + 8 * U32 + U * U
ROOT = Path(__file__).resolve().parent.parent


# ------------------------------------------------------------------------------------------------
# cases: name -> (res, heads, batch, shifted, warped, inputs, bias)
# ------------------------------------------------------------------------------------------------
def _case(res, heads, batch, mode="plain", inputs="randn", bias=False):
    return {"res": tuple(res), "heads": heads, "batch": batch, "shifted": mode != "plain",
            "warped": mode != "unwarped", "inputs": inputs, "bias": bias}


def _shift(case):
    return SHIFT if case["shifted"] else (0, 0, 0)


def box_rows(res, shift):
    """The host's TMA box height for a full-window grid (None: not full windows, the generic kernel runs): the largest
    run R such that every run of R in-window tokens along W is all padding or contiguous in the token stream, i.e. the
    gcd of the window width and every in-window position where padding starts / ends or the cyclic shift wraps."""
    ws, ss = W.adjust_windows(WS0, shift, res)
    if ws != WS0:
        return None
    lo, hi = W.pad_lo_hi(res, ws)[2]
    r = ws[2]
    for kw in range((res[2] + lo + hi) // ws[2]):
        prev_valid, prev_src = None, 0
        for i in range(ws[2]):
            q = kw * ws[2] + i - lo
            valid = 0 <= q < res[2]
            src = (q + ss[2]) % res[2] if valid else -1
            if i > 0 and (valid != prev_valid or (valid and src != prev_src + 1)):
                r = math.gcd(r, i)
            prev_valid, prev_src = valid, src
    return r


# TMA row boxes: (res, heads, batch) -> box_rows (unshifted, shifted).  H = 8, 9, 15 and 7 are zero-padded up to a
# multiple of 6, C = 3 and 5 up to a multiple of 2.
BOX_GRIDS = {
    "w24": ((4, 12, 24), 2, 1, (12, 6)),
    "w48": ((2, 6, 48), 3, 2, (12, 6)),
    "w180": ((3, 12, 180), 1, 1, (12, 6)),
    "w360": ((5, 6, 360), 2, 1, (12, 6)),
    "w28": ((4, 8, 28), 2, 3, (4, 2)),
    "w40": ((2, 15, 40), 4, 1, (4, 2)),
    "w90": ((4, 6, 90), 2, 2, (3, 3)),
    "w30": ((3, 9, 30), 3, 1, (3, 3)),
    "w20": ((2, 6, 20), 2, 2, (2, 2)),
    "w26": ((4, 12, 26), 1, 2, (1, 1)),
    "w34": ((5, 7, 34), 2, 1, (1, 1)),
}
TC_CASES = {}
for _k, (_res, _heads, _batch, _boxes) in BOX_GRIDS.items():
    for _mode, _box in (("plain", _boxes[0]), ("shifted", _boxes[1]), ("unwarped", _boxes[1])):
        TC_CASES[f"tc_{_k}_box{_box}_{_mode}"] = _case(_res, _heads, _batch, _mode)
for _res, _heads in (((4, 180, 360), 8), ((4, 90, 180), 16), ((4, 45, 90), 32)):
    for _mode in ("plain", "shifted"):
        TC_CASES[f"tc_full_{'x'.join(map(str, _res))}_h{_heads}_{_mode}"] = _case(_res, _heads, 1, _mode)
for _mode in ("plain", "shifted"):
    TC_CASES[f"tc_ring_one_item_{_mode}"] = _case((2, 6, 12), 1, 1, _mode)
    TC_CASES[f"tc_ring_idle_loader_{_mode}"] = _case((4, 12, 24), 2, 1, _mode)  # 16 items: one per CTA
    TC_CASES[f"tc_ring_wraps_{_mode}"] = _case((4, 24, 48), 32, 1, _mode)       # 1024 items: ~8 per CTA
    TC_CASES[f"tc_big_logits_{_mode}"] = _case((4, 8, 28), 4, 1, _mode, "big")
    TC_CASES[f"tc_equal_keys_{_mode}"] = _case((4, 12, 24), 2, 1, _mode, "equal_keys")
    TC_CASES[f"tc_nan_inf_{_mode}"] = _case((4, 12, 26), 2, 2, _mode, "nan_inf")
for _res in ((4, 12, 24), (4, 45, 90)):
    TC_CASES[f"tc_masked_keys_60_above_{'x'.join(map(str, _res))}"] = _case(_res, 2, 1, "shifted", "groups60")

# Clamped windows (an axis no longer than the window): ntok = 4, 16, 64, 72, 96, 120, 132; 4, 72, 120 and 132 are
# ragged (not a multiple of 16), 120 and 132 take three key blocks of the online softmax.
CLAMPED = {4: (1, 2, 2), 16: (4, 2, 4), 64: (4, 4, 8), 72: (1, 12, 24), 96: (2, 4, 24), 120: (4, 5, 36),
           132: (4, 12, 11)}
GENERIC_CASES = {}
for _n, _res in CLAMPED.items():
    for _mode in ("plain", "shifted"):
        GENERIC_CASES[f"generic_n{_n}_{_mode}"] = _case(_res, 2, 2, _mode)
        GENERIC_CASES[f"generic_n{_n}_rising_logits_{_mode}"] = _case(_res, 2, 2, _mode, "ramp")
for _n in (72, 120):
    GENERIC_CASES[f"generic_n{_n}_big_logits"] = _case(CLAMPED[_n], 2, 1, "shifted", "big")
    GENERIC_CASES[f"generic_n{_n}_masked_keys_60_above"] = _case(CLAMPED[_n], 2, 1, "shifted", "groups60")
    GENERIC_CASES[f"generic_n{_n}_nan_inf"] = _case(CLAMPED[_n], 2, 2, "shifted", "nan_inf")
GENERIC_CASES["generic_n120_unwarped"] = _case(CLAMPED[120], 2, 1, "unwarped")
# A dense bias always runs the generic kernel, full windows included; N(0, 4^2) moves the row max.
BIAS_CASES = {
    "bias_full_shifted": _case((4, 12, 24), 2, 2, "shifted", bias=True),
    "bias_full_padded_shifted": _case((3, 8, 26), 2, 1, "shifted", bias=True),
    "bias_full_plain": _case((4, 12, 24), 3, 1, "plain", bias=True),
    "bias_n72_shifted": _case(CLAMPED[72], 2, 2, "shifted", bias=True),
    "bias_n120_shifted": _case(CLAMPED[120], 2, 1, "shifted", bias=True),
    "bias_n120_masked_keys_60_above": _case(CLAMPED[120], 2, 1, "shifted", "groups60", bias=True),
}
ALL_CASES = {**TC_CASES, **GENERIC_CASES, **BIAS_CASES}
LARGE_GRIDS = [k for k in TC_CASES if k.startswith(("tc_full_4x180x360", "tc_full_4x90x180"))]


def _geometry(case):
    res, shift = case["res"], _shift(case)
    idx = W.window_gather_map(res, WS0, shift)[0]
    grp = W.window_group_ids(res, WS0, shift, case["warped"])
    return idx, grp


# ------------------------------------------------------------------------------------------------
# inputs, kernel call, reference
# ------------------------------------------------------------------------------------------------
def _seed(name):
    return int.from_bytes(hashlib.sha256(name.encode()).digest()[:4], "little")


def _token_maps(case, idx, grp):
    """In-window position and group id of every source token (each token sits in exactly one window)."""
    l = math.prod(case["res"])
    valid = idx >= 0
    pos = np.zeros(l, np.int64)
    pos[idx[valid]] = np.broadcast_to(np.arange(idx.shape[1]), idx.shape)[valid]
    g = np.zeros(l, np.int64)
    if grp is not None:
        g[idx[valid]] = grp[valid]
    return torch.from_numpy(pos).to(DEV), torch.from_numpy(g).to(DEV)


def make_inputs(name):
    """Seeded inputs of case `name`: bf16 qkv [B L, 3 D], bf16 pad_qkv [3 D] (q, k, v parts all different) and the
    fp32 bias [heads, N, N] or None.  Deterministic, so a child process rebuilds the same inputs."""
    case = ALL_CASES[name]
    res, heads, batch = case["res"], case["heads"], case["batch"]
    l, d = math.prod(res), heads * 64
    gen = torch.Generator(device=DEV).manual_seed(_seed(name))

    def randn(*shape):
        return torch.randn(*shape, generator=gen, device=DEV, dtype=torch.float32)

    x = randn(batch, l, 3, heads, 64) * 1.5
    pad = randn(3, heads, 64)
    kind = case["inputs"]
    if kind in ("ramp", "groups60"):
        idx, grp = _geometry(case)
        pos, g = _token_maps(case, idx, grp)
        x[:, :, :2] *= 0.25  # small noise on q and k: the constructed logits dominate
        pad[:2] *= 0.25
        if kind == "ramp":
            # logits rise from -20 to -8 along the window: every key block raises the running max, and a phantom
            # key of logit 0 (a zero row past ntok) would outweigh all real keys
            x[:, :, 0, :, 0] = 8.0
            x[:, :, 1, :, 0] = (-20.0 + 12.0 * pos / (idx.shape[1] - 1))[None, :, None]
        else:
            # q_i = -480 e_g(i), k_j = e_g(j) on dims 0..27: same-group logits -60, other groups 0, i.e. 60 above the
            # visible keys; the -100 mask leaves them e^-40 of the weight.  Zero-padded tokens are group 27.
            x[:, :, :2, :, :32] = 0.0
            x[:, torch.arange(l, device=DEV), 0, :, g] = -480.0
            x[:, torch.arange(l, device=DEV), 1, :, g] = 1.0
            pad[:2, :, :32] = 0.0
            pad[0, :, W.PAD_GROUP] = -480.0
            pad[1, :, W.PAD_GROUP] = 1.0
    elif kind == "big":
        x[:, :, 0] *= 100.0 / 1.5  # q.k / 8 ~ N(0, 100^2): logits span about +-300
        x[:, :, 1] /= 1.5
        pad[0] *= 100.0
    elif kind == "equal_keys":
        x[:, :, 1] = pad[1]  # every key of every window is the same vector
    qkv = x.reshape(batch * l, 3 * d).to(BF16)
    if kind == "nan_inf":
        # batch element 0 only: a NaN in one K row and in one V row, +inf in one Q row, of head `heads - 1`
        c = (heads - 1) * 64
        qkv[l // 3, d + c + 5] = float("nan")
        qkv[(2 * l) // 3, 2 * d + c + 7] = float("nan")
        qkv[l - 1, c + 3] = float("inf")
    bias = randn(heads, *[math.prod(W.adjust_windows(WS0, _shift(case), res)[0])] * 2) * 4.0 if case["bias"] else None
    return qkv, pad.reshape(3 * d).to(BF16), bias


def run_kernel(name, qkv, pad, bias):
    from aurora_b200 import cabi

    case = ALL_CASES[name]
    res, heads, batch = case["res"], case["heads"], case["batch"]
    out = torch.full((qkv.shape[0], heads * 64), float("nan"), device=DEV, dtype=BF16)
    cabi.window_attention(qkv, out, batch=batch, res=res, window=WS0, shift=_shift(case), num_heads=heads,
                          pad_qkv=pad, bias=bias, warped=case["warped"])
    torch.cuda.synchronize()
    return out


def reference(name, qkv, pad, bias, chunk_bytes=1 << 29):
    """float64 output [B L, D] and its per-element error bound (see the module docstring)."""
    case = ALL_CASES[name]
    res, heads, batch = case["res"], case["heads"], case["batch"]
    l, d = math.prod(res), heads * 64
    idx_np, grp_np = _geometry(case)
    idx = torch.from_numpy(idx_np).to(DEV)
    nw, n = idx.shape
    valid = idx >= 0
    src = idx.clamp(min=0)
    grp = torch.from_numpy(grp_np.astype(np.int64)).to(DEV) if grp_np is not None else None
    x = qkv.view(batch, l, 3, heads, 64)
    p = pad.view(3, heads, 64).double()
    ref = torch.empty(batch, l, heads, 64, device=DEV, dtype=torch.float64)
    tol = torch.empty_like(ref)
    step = max(1, chunk_bytes // (n * n * 8))  # windows per chunk: one [chunk, N, N] float64 logit tensor
    for b in range(batch):
        for h in range(heads):
            xh = x[b, :, :, h].double()  # [L, 3, 64]
            for w0 in range(0, nw, step):
                w1 = min(nw, w0 + step)
                xw = xh[src[w0:w1]]
                xw[~valid[w0:w1]] = p[:, h]
                q, k, v = xw.unbind(2)
                s = q @ k.transpose(-1, -2) / 8.0
                if bias is not None:
                    s += bias[h].double()
                if grp is not None:
                    g = grp[w0:w1]
                    s -= 100.0 * (g[:, :, None] != g[:, None, :])
                a = torch.softmax(s, -1)
                o = a @ v
                av = a @ v.abs()
                e = GAMMA_QK * (q.abs() @ k.abs().transpose(-1, -2)).amax(-1) / 8.0 + 8 * U32 * s.abs().amax(-1)
                t = U * o.abs() + (U + torch.expm1(2 * e)[..., None] + SMALL) * av
                ok = valid[w0:w1]
                ref[b, idx[w0:w1][ok], h] = o[ok]
                tol[b, idx[w0:w1][ok], h] = t[ok]
    return ref.view(batch * l, d), tol.view(batch * l, d)


def check(name, out, ref, tol):
    """NaN exactly where the reference has NaN; elsewhere |out - ref| <= tol.  Returns the worst error / bound."""
    o = out.double()
    nan_o, nan_r = torch.isnan(o), torch.isnan(ref)
    assert torch.equal(nan_o, nan_r), (f"{name}: NaN placement differs at {int((nan_o != nan_r).sum())} elements, "
                                       f"first (row, col) {torch.nonzero(nan_o != nan_r)[:4].tolist()}")
    fin = ~nan_r
    err = torch.where(fin, (o - ref).abs(), torch.zeros_like(o))
    ratio = torch.where(fin, err / tol, torch.zeros_like(o))
    worst = float(ratio.max())
    if not worst <= 1.0:
        i = int(torch.argmax(torch.nan_to_num(ratio, nan=math.inf)))
        r, c = divmod(i, out.shape[1])
        raise AssertionError(f"{name}: out[{r}, {c}] = {float(o.flatten()[i]):.6g}, reference "
                             f"{float(ref.flatten()[i]):.6g}, error {float(err.flatten()[i]):.3e} > bound "
                             f"{float(tol.flatten()[i]):.3e} (worst error / bound {worst:.2f}, "
                             f"{int((ratio > 1).sum())} elements over)")
    print(f"[window attention] {name}: worst error / bound {worst:.3f}")
    return worst


def _check_case(name):
    qkv, pad, bias = make_inputs(name)
    out = run_kernel(name, qkv, pad, bias)
    ref, tol = reference(name, qkv, pad, bias)
    return check(name, out, ref, tol)


# ------------------------------------------------------------------------------------------------
# the default paths: wgmma kernel with the TMA gather, generic kernel on clamped windows, bias
# ------------------------------------------------------------------------------------------------
def test_case_labels_match_the_host_rules():
    for name, case in TC_CASES.items():
        box = box_rows(case["res"], _shift(case))
        assert box is not None, name
        if "_box" in name:
            assert f"_box{box}_" in name, (name, box)
        assert case["bias"] is False
    for name, case in GENERIC_CASES.items():
        ws = W.adjust_windows(WS0, _shift(case), case["res"])[0]
        assert ws != WS0 and f"_n{math.prod(ws)}_" in name, name
    assert {box_rows(c["res"], _shift(c)) for c in TC_CASES.values()} == {1, 2, 3, 4, 6, 12}


@pytest.mark.parametrize("name", list(TC_CASES))
def test_tc_kernel_tma_gather(name):
    _check_case(name)


@pytest.mark.parametrize("name", list(GENERIC_CASES))
def test_generic_kernel_clamped_windows(name):
    _check_case(name)


@pytest.mark.parametrize("name", list(BIAS_CASES))
def test_bias_path(name):
    _check_case(name)


@pytest.mark.parametrize("name", [k for k in ALL_CASES if k.endswith("nan_inf") or "_nan_inf_" in k])
def test_nan_inf_poisons_exactly_the_rows_and_columns_float64_does(name):
    """Pin the NaN pattern down explicitly: a NaN in a K row poisons every query row of its window (that head's 64
    columns), a NaN in a V row poisons one column of every row of its window, +inf in a Q row poisons that row."""
    case = ALL_CASES[name]
    qkv, pad, bias = make_inputs(name)
    out = run_kernel(name, qkv, pad, bias)
    l, heads = math.prod(case["res"]), case["heads"]
    c = (heads - 1) * 64
    idx, _ = _geometry(case)
    win_of = {int(t): w for w, row in enumerate(idx) for t in row if t >= 0}
    members = lambda tok: torch.from_numpy(idx[win_of[tok]][idx[win_of[tok]] >= 0]).to(DEV)  # noqa: E731
    want = torch.zeros_like(out, dtype=torch.bool)
    want[members(l // 3), c:c + 64] = True
    want[members((2 * l) // 3), c + 7] = True
    want[l - 1, c:c + 64] = True
    assert torch.equal(torch.isnan(out), want)


# ------------------------------------------------------------------------------------------------
# forced paths, in child processes: AB_ATTN_NO_TMA / AB_ATTN_NO_TC are read once per process
# ------------------------------------------------------------------------------------------------
def dump_outputs(names, path, keep_below=None):
    """Run `names` and write {name: [sha256 of the output bits, the output on the CPU, or None if it has
    `keep_below` elements or more]}."""
    res = {}
    for name in names:
        out = run_kernel(name, *make_inputs(name)).cpu()
        digest = hashlib.sha256(out.view(torch.int16).numpy().tobytes()).hexdigest()
        res[name] = [digest, out if keep_below is None or out.numel() < keep_below else None]
    torch.save(res, path)


def _in_child(env, names, path, keep_below=None):
    code = ("from tests.test_window_attention_gpu import dump_outputs; "
            f"dump_outputs({list(names)!r}, {str(path)!r}, {keep_below!r})")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", code], cwd=ROOT, env={**os.environ, env: "1"},
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return torch.load(path, weights_only=False)


def test_tc_cp_async_gather_is_bit_identical_to_tma(tmp_path):
    """Both gathers fill the same swizzled stage layout and the math is the same: outputs must agree bit for bit."""
    got = _in_child("AB_ATTN_NO_TMA", TC_CASES, tmp_path / "no_tma.pt", keep_below=1 << 24)
    for name in TC_CASES:
        out = run_kernel(name, *make_inputs(name)).cpu()
        digest = hashlib.sha256(out.view(torch.int16).numpy().tobytes()).hexdigest()
        if digest != got[name][0]:
            other = got[name][1]
            diff = "" if other is None else f": {int((other.view(torch.int16) != out.view(torch.int16)).sum())} differ"
            raise AssertionError(f"{name}: cp.async and TMA gathers give different bits{diff}")


def test_generic_kernel_on_full_windows(tmp_path):
    """`AB_ATTN_NO_TC` runs every full-window case on the generic kernel (three key blocks of 48): same bound.  The two
    largest grids are left out to keep the child's output file small; (4, 45, 90) x 32 heads stays."""
    names = [k for k in TC_CASES if k not in LARGE_GRIDS]
    got = _in_child("AB_ATTN_NO_TC", names, tmp_path / "no_tc.pt")
    worst = 0.0
    for name in names:
        qkv, pad, bias = make_inputs(name)
        ref, tol = reference(name, qkv, pad, bias)
        worst = max(worst, check(f"{name} (generic kernel)", got[name][1].to(DEV), ref, tol))
    print(f"[window attention] generic kernel on full windows: worst error / bound {worst:.3f}")


# ------------------------------------------------------------------------------------------------
# identities: bit for bit on both kernels
# ------------------------------------------------------------------------------------------------
IDENTITY_CASES = ["tc_w28_box2_shifted", "tc_ring_wraps_plain", "generic_n120_shifted", "generic_n72_plain",
                  "bias_full_shifted"]


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


@pytest.mark.parametrize("name", IDENTITY_CASES)
def test_repeated_calls_are_bit_identical(name):
    qkv, pad, bias = make_inputs(name)
    first = run_kernel(name, qkv, pad, bias)
    for _ in range(2):
        assert _bits_equal(run_kernel(name, qkv, pad, bias), first)


@pytest.mark.parametrize("name", ["tc_w28_box4_plain", "tc_w28_box2_shifted", "tc_nan_inf_shifted",
                                  "generic_n72_shifted", "generic_n120_plain", "generic_n4_plain"])
def test_batch_elements_equal_single_calls(name):
    from aurora_b200 import cabi

    case = ALL_CASES[name]
    assert case["batch"] > 1
    res, heads = case["res"], case["heads"]
    l = math.prod(res)
    qkv, pad, bias = make_inputs(name)
    full = run_kernel(name, qkv, pad, bias)
    for b in range(case["batch"]):
        one = torch.empty(l, heads * 64, device=DEV, dtype=BF16)
        cabi.window_attention(qkv[b * l:(b + 1) * l].contiguous(), one, batch=1, res=res, window=WS0,
                              shift=_shift(case), num_heads=heads, pad_qkv=pad, bias=bias, warped=case["warped"])
        torch.cuda.synchronize()
        assert _bits_equal(one, full[b * l:(b + 1) * l]), (name, b)


@pytest.mark.parametrize("name,roll", [("tc_w24_box12_plain", 12), ("tc_w48_box12_plain", 36),
                                       ("tc_ring_wraps_plain", 24), ("generic_n72_plain", 12)])
def test_roll_along_w_rolls_the_output(name, roll):
    """Unpadded, unshifted grid: rolling the input by a multiple of the window along W permutes whole windows (and keeps
    box_rows), so the output rolls the same way, bit for bit."""
    case = ALL_CASES[name]
    res, heads, batch = case["res"], case["heads"], case["batch"]
    assert not case["shifted"] and all(r % w == 0 or r < w for r, w in zip(res, WS0))
    assert box_rows(res, (0, 0, 0)) in (None, 12)
    qkv, pad, bias = make_inputs(name)
    out = run_kernel(name, qkv, pad, bias)
    rolled_in = qkv.view(batch, *res, -1).roll(roll, dims=3).reshape(qkv.shape).contiguous()
    rolled_out = run_kernel(name, rolled_in, pad, bias)
    assert _bits_equal(rolled_out, out.view(batch, *res, -1).roll(roll, dims=3).reshape(out.shape))
