"""wgmma GEMM (ab_gemm_bf16) against a plain PyTorch fp32 reference of the same op."""

import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(a, w, bias, residual, act):
    y = a.float() @ w.float().t()
    if bias is not None:
        y = y + bias
    if act:
        y = torch.nn.functional.gelu(y)
    if residual is not None:
        y = y + residual
    return y


SHAPES = [
    # (M, N, K)
    (128, 256, 64),
    (128, 256, 512),
    (256, 512, 128),
    (300, 256, 192),     # M tail
    (1000, 1536, 512),   # qkv-like
    (777, 80, 1024),     # decoder heads: N tail inside a 128-wide tile
    (64, 64, 256),       # tiny
    (129, 520, 72),      # M, N and K tails (K % 64 != 0)
    (4096, 2048, 512),   # fc1 stage-1-like, many tiles per CTA
    (2048, 512, 2048),   # fc2-like, long K
    (5, 16, 8),          # minimum sizes
    # many tiles, N = 256 blocks
    (1300, 520, 192),    # M tail inside the second warpgroup's rows, N tail, 3 k-blocks
    (2049, 256, 72),     # one row into a new tile (second warpgroup fully out of bounds), K tail
    (5000, 1536, 512),   # qkv-like, many tiles per cluster
    (1024, 300, 64),     # N tail in the only N block
]


@pytest.mark.parametrize("m,n,k", SHAPES)
@pytest.mark.parametrize("mode", ["plain_bf16", "bias_gelu_bf16", "bias_res_f32_dual"])
def test_gemm_matches_fp32_reference(m, n, k, mode):
    from aurora_b200 import cabi

    torch.manual_seed(m * 31 + n * 7 + k)
    dev = "cuda"
    a = torch.randn(m, k, device=dev).to(torch.bfloat16)
    w = (torch.randn(n, k, device=dev) / k**0.5).to(torch.bfloat16)
    bias = torch.randn(n, device=dev) if mode != "plain_bf16" else None
    residual = torch.randn(m, n, device=dev) if mode == "bias_res_f32_dual" else None
    act = cabi.AB_ACT_GELU_ERF if mode == "bias_gelu_bf16" else cabi.AB_ACT_NONE
    out_bf16 = torch.full((m, n), float("nan"), device=dev, dtype=torch.bfloat16)
    out_f32 = torch.full((m, n), float("nan"), device=dev) if mode == "bias_res_f32_dual" else None

    cabi.gemm(a, w, bias=bias, residual=residual, out_f32=out_f32, out_bf16=out_bf16, act=act)
    torch.cuda.synchronize()

    ref = _ref(a, w, bias, residual, act)
    # fp32 accumulation of bf16 products: only the output rounding differs from the fp32 reference.
    if out_f32 is not None:
        torch.testing.assert_close(out_f32, ref, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(out_bf16.float(), ref, rtol=1e-2, atol=1e-2)


LONG_K_SHAPES = [
    (1024, 256, 1024),    # eight full 128-row tiles
    (1500, 520, 1024),    # M tail inside the second warpgroup's rows, N tail (8 live columns in the last block)
    (2049, 256, 1088),    # one row into a new tile (all but one 16-row box fully out of bounds), odd k-block count
    (20000, 1536, 1024),  # several tiles per CTA: the accumulator registers are reused between tiles
    (4096, 512, 4096),    # long K
]


@pytest.mark.parametrize("m,n,k", LONG_K_SHAPES)
@pytest.mark.parametrize("mode", ["plain_bf16", "bias_gelu_bf16", "bias_res_f32_dual"])
def test_long_k_matches_reference_and_repeats_bit_identically(m, n, k, mode):
    """Large shapes with K >= 1024 (long main loops, many tiles per CTA): fp32 reference tolerance, and two launches on
    the same operands are bit-identical (the persistent schedule fixes the fp32 accumulation order over K)."""
    from aurora_b200 import cabi

    torch.manual_seed(m + n + k)
    dev = "cuda"
    a = torch.randn(m, k, device=dev).to(torch.bfloat16)
    w = (torch.randn(n, k, device=dev) / k**0.5).to(torch.bfloat16)
    bias = torch.randn(n, device=dev) if mode != "plain_bf16" else None
    residual = torch.randn(m, n, device=dev) if mode == "bias_res_f32_dual" else None
    act = cabi.AB_ACT_GELU_ERF if mode == "bias_gelu_bf16" else cabi.AB_ACT_NONE
    outs = []
    for _ in range(2):
        out_bf16 = torch.full((m, n), float("nan"), device=dev, dtype=torch.bfloat16)
        out_f32 = torch.full((m, n), float("nan"), device=dev) if mode == "bias_res_f32_dual" else None
        cabi.gemm(a, w, bias=bias, residual=residual, out_f32=out_f32, out_bf16=out_bf16, act=act)
        torch.cuda.synchronize()
        outs.append((out_bf16, out_f32))
    ref = _ref(a, w, bias, residual, act)
    (out_bf16, out_f32), (again_bf16, again_f32) = outs
    if out_f32 is not None:
        torch.testing.assert_close(out_f32, ref, rtol=1e-4, atol=1e-4)
        assert torch.equal(out_f32, again_f32)
    torch.testing.assert_close(out_bf16.float(), ref, rtol=1e-2, atol=1e-2)
    assert torch.equal(out_bf16, again_bf16)


def test_gemm_strided_views():
    """Leading dimensions larger than the logical width (writes into a slice of a wider buffer)."""
    from aurora_b200 import cabi

    torch.manual_seed(0)
    m, n, k = 384, 256, 128
    a_full = torch.randn(m, 2 * k, device="cuda").to(torch.bfloat16)
    a = a_full[:, k:]
    w = (torch.randn(n, k, device="cuda") / k**0.5).to(torch.bfloat16)
    out_full = torch.zeros(m, 2 * n, device="cuda", dtype=torch.bfloat16)
    out = out_full[:, n:]
    cabi.gemm(a, w, out_bf16=out)
    torch.cuda.synchronize()
    ref = a.float() @ w.float().t()
    torch.testing.assert_close(out.float(), ref, rtol=1e-2, atol=1e-2)
    assert out_full[:, :n].abs().max().item() == 0.0


def test_gemm_rejects_bad_arguments():
    from aurora_b200 import cabi

    a = torch.zeros(16, 12, device="cuda", dtype=torch.bfloat16)  # K % 8 != 0
    w = torch.zeros(16, 12, device="cuda", dtype=torch.bfloat16)
    out = torch.zeros(16, 16, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(cabi.AbError):
        cabi.gemm(a, w, out_bf16=out)


# ------------------------------------------------------------------------------------------------------------
# projection with adaLN + residual fused into the epilogue (csrc/gemm_ln.cu)
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m,n,k", [
    (1000, 512, 512),     # proj-like, M tail inside the last tile
    (5000, 512, 2048),    # fc2-like, many tiles per cluster, long K
    (37, 512, 128),       # fewer rows than one CTA holds
    (785, 1024, 1024),    # four CTAs per cluster: row statistics meet through distributed shared memory
    (20000, 1024, 4096),  # stage-2 fc2-like
    (300, 1024, 72),      # K tail (K % 64 != 0), cluster of 4
])
@pytest.mark.parametrize("mode", ["inplace_bf16", "f16_wide_ld", "no_residual_f32_only"])
def test_gemm_ln_residual_matches_fp32_reference(m, n, k, mode):
    """out = residual + LN(a @ w.T + bias) * scale + shift against plain fp32 PyTorch on the same 16-bit operands.
    Tolerance: the kernel takes the statistics on the fp32 accumulator, so only summation order differs: 2e-3 abs / rel
    on the fp32 stream (values are O(1..10)), one 16-bit ulp on the 16-bit copy."""
    from aurora_b200 import cabi

    torch.manual_seed(m + n + k)
    dev = "cuda"
    dt = torch.float16 if mode == "f16_wide_ld" else torch.bfloat16
    a = torch.randn(m, k, device=dev).to(dt)
    w = (torch.randn(n, k, device=dev) / k**0.5).to(dt)
    bias = torch.randn(n, device=dev)
    scale = torch.randn(n, device=dev)
    shift = torch.randn(n, device=dev)
    residual = None if mode == "no_residual_f32_only" else torch.randn(m, n, device=dev) * 3
    y = a.float() @ w.float().t() + bias
    ref = torch.nn.functional.layer_norm(y, (n,), eps=1e-5) * scale + shift
    if residual is not None:
        ref = ref + residual
    if mode == "inplace_bf16":
        out_f32 = residual.clone()              # the fp32 stream is updated IN PLACE (output aliases the residual)
        out16 = torch.full((m, n), float("nan"), device=dev, dtype=dt)
        cabi.gemm_ln_residual(a, w, bias=bias, scale=scale, shift=shift, residual=out_f32, out_f32=out_f32, out_bf16=out16)
    elif mode == "f16_wide_ld":
        wide = torch.full((m, 2 * n), float("nan"), device=dev, dtype=dt)   # one half of a concatenation buffer
        out16 = wide[:, n:]
        out_f32 = torch.full((m, n), float("nan"), device=dev)
        cabi.gemm_ln_residual(a, w, bias=bias, scale=scale, shift=shift, residual=residual, out_f32=out_f32, out_bf16=out16)
        assert torch.isnan(wide[:, :n]).all()   # the other half is untouched
    else:
        out16 = None
        out_f32 = torch.full((m, n), float("nan"), device=dev)
        cabi.gemm_ln_residual(a, w, bias=bias, scale=scale, shift=shift, out_f32=out_f32)
    torch.cuda.synchronize()
    torch.testing.assert_close(out_f32, ref, rtol=2e-3, atol=2e-3)
    if out16 is not None:
        torch.testing.assert_close(out16.float(), ref, rtol=1e-2, atol=2e-2)
        assert torch.equal(out16, out_f32.to(dt))  # the 16-bit copy is the rounding of the fp32 result


def test_gemm_ln_residual_rejects_other_widths():
    from aurora_b200 import cabi

    a = torch.zeros(256, 64, device="cuda", dtype=torch.bfloat16)
    w = torch.zeros(2048, 64, device="cuda", dtype=torch.bfloat16)
    out = torch.zeros(256, 2048, device="cuda")
    assert not cabi.gemm_ln_supported(2048) and cabi.gemm_ln_supported(512) and cabi.gemm_ln_supported(1024)
    with pytest.raises(cabi.AbError, match="not supported"):
        cabi.gemm_ln_residual(a, w, out_f32=out)


# ------------------------------------------------------------------------------------------------------------
# fused compute + exchange: the epilogue also stores boundary rows into (peer) halo slots (AbGemm.peer_push)
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,w", [(5, 12), (10, 36), (30, 144)])
@pytest.mark.parametrize("to_above,to_below", [(3, 2), (0, 5), (1, 0)])
def test_gemm_epilogue_pushes_boundary_rows_into_halo_slots(rows, w, to_above, to_below):
    """The QKV projection of a latitude band [C, rows, W, 3D] with `peer_push`: columns [D, 3D) of the first `to_above`
    and last `to_below` rows of every level land in the halo slots (here: in this GPU's own memory) exactly as
    `ab_halo_push` would place them, the round is published in both flags once, the completion counter is back at zero,
    and the regular output is untouched by the extra stores.  M = 240, 1440 and 17280: 6 and 36 tiles of 128 x 256,
    fewer than SMs, and 405 tiles, several per CTA."""
    from aurora_b200 import cabi

    c, d, k, slot_rows = 4, 256, 1024, 5
    m, n = c * rows * w, 3 * d
    torch.manual_seed(c + rows + w + to_above)
    dev = "cuda"
    a = torch.randn(m, k, device=dev).to(torch.bfloat16)
    wt = (torch.randn(n, k, device=dev) / k**0.5).to(torch.bfloat16)
    bias = torch.randn(n, device=dev)
    ref_out = torch.empty(m, n, device=dev, dtype=torch.bfloat16)
    cabi.gemm(a, wt, bias=bias, out_bf16=ref_out)
    out = torch.full((m, n), float("nan"), device=dev, dtype=torch.bfloat16)
    slots = torch.full((2, c, slot_rows, w, 2 * d), float("nan"), device=dev, dtype=torch.bfloat16)
    ctrl = torch.zeros(64, device=dev, dtype=torch.int32)
    ctrl[2] = 41  # the previous round
    hp = cabi.AbHaloPush()
    hp.above_slot, hp.below_slot = slots[1].data_ptr(), slots[0].data_ptr()   # side 1 of the rank above, side 0 of the rank below
    hp.above_flag, hp.below_flag, hp.ctrl = ctrl.data_ptr() + 4, ctrl.data_ptr(), ctrl.data_ptr()
    hp.c, hp.rows, hp.w, hp.slot_rows = c, rows, w, slot_rows
    hp.rows_to_above, hp.rows_to_below = to_above, to_below
    hp.src_tok_bytes, hp.tok_off_bytes, hp.tok_bytes = 3 * d * 2, d * 2, 2 * d * 2
    cabi.gemm(a, wt, bias=bias, out_bf16=out, peer_push=hp)
    torch.cuda.synchronize()
    assert torch.equal(out, ref_out)
    assert ctrl[:4].tolist() == [42, 42, 42, 0]
    o4 = ref_out.view(c, rows, w, n)[..., d:]
    assert torch.equal(slots[1][:, :to_above], o4[:, :to_above])                                 # my first rows -> above
    assert torch.isnan(slots[1][:, to_above:].float()).all()
    assert torch.equal(slots[0][:, slot_rows - to_below:], o4[:, rows - to_below:])             # my last rows -> below
    assert torch.isnan(slots[0][:, : slot_rows - to_below].float()).all()
