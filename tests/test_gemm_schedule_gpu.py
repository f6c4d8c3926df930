"""Tile schedule of the wgmma GEMM (ab_gemm_bf16).  Each CTA takes a persistent sequence of 128 x BN tiles (BN = 256
for N > 128, 128 / 64 for narrower outputs), and both of its math warpgroups work on every tile, 64 rows each.  Tile
counts around multiples of the grid, last row blocks with no live row for the second warpgroup, tails in every
dimension, fewer k-blocks than pipeline stages, both operand types, every epilogue mode and every GEMM shape of a
full-size forecast step are checked against an fp32 PyTorch reference of the same op, and the cases with many tiles
per CTA or few k-blocks also for bit-identical repeat launches."""

import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}


@pytest.fixture(autouse=True)
def _no_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = saved


def _gemm(m, n, k, dtype, bias, gelu, out_f32, out16, residual, seed):
    """Runs the kernel on seeded operands; returns (16-bit output or None, fp32 output or None, fp32 reference)."""
    from aurora_b200 import cabi

    g = torch.Generator(device="cuda").manual_seed(seed)
    dt = DTYPES[dtype]
    a = torch.randn(m, k, device="cuda", generator=g).to(dt)
    w = (torch.randn(n, k, device="cuda", generator=g) / k**0.5).to(dt)
    b = torch.randn(n, device="cuda", generator=g) if bias else None
    r = torch.randn(m, n, device="cuda", generator=g) if residual else None
    o16 = torch.full((m, n), float("nan"), device="cuda", dtype=DTYPES[out16]) if out16 else None
    o32 = torch.full((m, n), float("nan"), device="cuda") if out_f32 else None
    cabi.gemm(a, w, bias=b, residual=r, out_f32=o32, out_bf16=o16,
              act=cabi.AB_ACT_GELU_ERF if gelu else cabi.AB_ACT_NONE)
    torch.cuda.synchronize()
    y = a.float() @ w.float().t()
    del a, w
    if b is not None:
        y += b
    if gelu:
        y = torch.nn.functional.gelu(y)
    if r is not None:
        y += r
    return o16, o32, y


def _check(*shape_and_mode, seed=0):
    o16, o32, y = _gemm(*shape_and_mode, seed=seed)
    if o32 is not None:
        torch.testing.assert_close(o32, y, rtol=1e-4, atol=1e-4)
    if o16 is not None:
        # fp32 accumulation of 16-bit products: only the output rounding differs from the fp32 reference
        torch.testing.assert_close(o16.float(), y, rtol=1e-2, atol=1e-2)
    return o16, o32


def _check_twice(m, n, k, dtype, mode, seed):
    """_check on outputs that start as NaN, then a second launch on the same operands, bit-identical to the first."""
    first = _check(m, n, k, dtype, *_mode(mode, dtype), seed=seed)
    second = _gemm(m, n, k, dtype, *_mode(mode, dtype), seed=seed)[:2]
    for a, b in zip(first, second):
        assert a is None or torch.equal(a, b)


MODES = {  # bias, gelu, out_f32, residual
    "plain": (False, False, False, False),
    "bias": (True, False, False, False),
    "bias_gelu": (True, True, False, False),
    "bias_res_f32_dual": (True, False, True, True),
}


def _mode(name, out16):
    bias, gelu, f32, res = MODES[name]
    return bias, gelu, f32, out16, res


@pytest.mark.parametrize("tiles", ["2", "sms", "sms+2", "2sms+2", "3sms+2"])
@pytest.mark.parametrize("mode", ["bias_gelu", "bias_res_f32_dual", "plain"])
def test_tile_counts_around_the_grid(tiles, mode):
    """N = 256, K = 320: one 128 x 256 tile per 128 rows; the last row block has a 40-row tail, no live row for the
    second warpgroup.  `tiles` counts 128 x 128 blocks, so the kernel runs (tiles + 1) // 2 tiles: 2: one tile on one
    CTA; sms: half the SMs busy; sms + 2: one more tile; 2 sms + 2: one CTA with two tiles; 3 sms + 2: about half the
    CTAs with two tiles."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    t = {"2": 2, "sms": sms, "sms+2": sms + 2, "2sms+2": 2 * sms + 2, "3sms+2": 3 * sms + 2}[tiles]
    m = 128 * ((t + 1) // 2 - 1) + 40
    _check(m, 256, 320, "bf16", *_mode(mode, "bf16"), seed=t)


@pytest.mark.parametrize("m,n,k", [
    (257, 200, 136),    # one 128 x 256 tile per row block with 200 live columns, K tail
    (517, 136, 1024),   # 128 x 256: 136 live columns, 16 k-blocks
    (131, 520, 72),     # 128 x 256: 8 live columns in the third tile, inside one 64-column epilogue box; K tail
    (3000, 1032, 520),  # 128 x 256: 120 tiles, 8 live columns in the last of each row block; K tail
    (1000, 300, 1096),  # 128 x 256: 44 live columns in the second tile, K tail past 1024
    (1000, 80, 72),     # decoder-head width (128 x 128), K tail
    (300, 64, 200),     # the 64-wide tile, M and K tails
])
@pytest.mark.parametrize("mode", ["bias_gelu", "bias_res_f32_dual", "plain"])
@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
def test_tails_modes_and_operand_types(m, n, k, mode, dtype):
    """fp16 operands (encoder / decoder) write fp16, bf16 operands write bf16."""
    _check(m, n, k, dtype, *_mode(mode, dtype), seed=m + n + k)


# Every distinct GEMM of one step of the 1.3 B model at 0.25 degrees (721 x 1440, 13 levels), full size:
# (M, N, K, operand dtype, bias, GELU, fp32 output, 16-bit output dtype, residual)
PRODUCTION_SHAPES = [
    (259200, 1536, 512, "bf16", True, False, False, "bf16", False),    # Swin stage 1: qkv, proj, fc1, fc2
    (259200, 512, 512, "bf16", True, False, False, "bf16", False),
    (259200, 2048, 512, "bf16", True, True, False, "bf16", False),
    (259200, 512, 2048, "bf16", True, False, False, "bf16", False),
    (64800, 3072, 1024, "bf16", True, False, False, "bf16", False),    # stage 2
    (64800, 1024, 1024, "bf16", True, False, False, "bf16", False),
    (64800, 4096, 1024, "bf16", True, True, False, "bf16", False),
    (64800, 1024, 4096, "bf16", True, False, False, "bf16", False),
    (16200, 6144, 2048, "bf16", True, False, False, "bf16", False),    # stage 3
    (16200, 2048, 2048, "bf16", True, False, False, "bf16", False),
    (16200, 8192, 2048, "bf16", True, True, False, "bf16", False),
    (16200, 2048, 8192, "bf16", True, False, False, "bf16", False),
    (64800, 1024, 2048, "bf16", False, False, True, "bf16", False),    # patch merges and splits
    (16200, 2048, 4096, "bf16", False, False, True, "bf16", False),
    (16200, 4096, 2048, "bf16", False, False, False, "bf16", False),
    (64800, 2048, 1024, "bf16", False, False, False, "bf16", False),
    (64800, 1024, 1024, "bf16", False, False, True, "bf16", False),
    (259200, 512, 512, "bf16", False, False, True, "bf16", True),
    (842400, 2048, 1024, "fp16", True, True, False, "fp16", False),    # encoder and decoder (Perceiver)
    (842400, 1024, 2048, "fp16", True, False, False, "fp16", False),
    (842400, 1024, 1024, "fp16", False, False, False, "fp16", False),
    (842400, 1024, 512, "fp16", False, False, False, "fp16", False),
    (194400, 2048, 1024, "fp16", False, False, False, "fp16", False),
    (194400, 2048, 512, "fp16", True, True, False, "fp16", False),
    (194400, 512, 2048, "fp16", True, False, False, "fp16", False),
    (194400, 512, 512, "fp16", False, False, False, "fp16", False),
    (64800, 512, 192, "fp16", True, False, False, "fp16", False),
    (64800, 2048, 512, "fp16", True, True, False, "fp16", False),
    (64800, 512, 2048, "fp16", True, False, False, "fp16", False),
    (64800, 512, 256, "fp16", True, False, True, "fp16", False),
    (842400, 80, 1024, "fp16", True, False, True, None, False),        # output heads
    (64800, 64, 1024, "fp16", True, False, True, None, False),
]


@pytest.mark.parametrize("shape", PRODUCTION_SHAPES, ids=lambda s: "x".join(map(str, s[:3])) + "-" + "-".join(
    f for f, on in zip(("bias", "gelu", "f32", "res"), (s[4], s[5], s[6], s[8])) if on))
def test_production_shapes_full_size(shape):
    _check(*shape, seed=sum(shape[:3]))
    torch.cuda.empty_cache()


@pytest.mark.parametrize("mode", ["bias_gelu", "bias_res_f32_dual"])
@pytest.mark.parametrize("k", [1024, 2048])
def test_two_launches_are_bit_identical(mode, k):
    """The accumulation order over K is fixed by the kernel, not by which CTA takes a tile (128 x 256 tiles, about
    12 per CTA)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    args = (2 * 128 * sms + 77, 1536, k, "bf16", *_mode(mode, "bf16"))
    first = _gemm(*args, seed=5)
    second = _gemm(*args, seed=5)
    assert torch.equal(first[0], second[0])
    if first[1] is not None:
        assert torch.equal(first[1], second[1])


# N = 768: three 128 x 256 tiles per 128 rows, K = 320.  M = 128 (blocks - 1) + 40, so the last row block has no live
# row for the second warpgroup.  Row blocks from the SM count: 3 tiles, about sms, sms + 3 (some CTAs with two tiles)
# and about 2 sms + 3 (an odd count on most CTAs).
ROW_BLOCKS = {
    "3": lambda sms: 1,
    "sms": lambda sms: math.ceil(sms / 3),
    "sms+3": lambda sms: math.ceil(sms / 3) + 1,
    "2sms+3": lambda sms: math.ceil(2 * sms / 3) + 1,
}


@pytest.mark.parametrize("tiles", list(ROW_BLOCKS))
@pytest.mark.parametrize("mode", ["plain", "bias_gelu"])
def test_last_row_block_without_rows_for_the_second_warpgroup(tiles, mode):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    m, n, k = 128 * (ROW_BLOCKS[tiles](sms) - 1) + 40, 768, 320
    _check_twice(m, n, k, "bf16", mode, seed=m * 7 + n * 3 + k)


@pytest.mark.parametrize("m,n,k", [
    (131, 520, 64),     # one k-block; 8 live columns in the third tile, inside one 64-column box
    (257, 200, 72),     # two k-blocks, the second 8 deep; one 256-column tile with 200 live columns
    (300, 1032, 136),   # three k-blocks; N tail of 8 columns, M tail of 44 rows
    (517, 264, 1024),   # sixteen k-blocks; 8 live columns in the second tile
    (1000, 300, 1096),  # a K tail past 1024
])
@pytest.mark.parametrize("mode", ["plain", "bias", "bias_gelu", "bias_res_f32_dual"])
@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
def test_few_k_blocks_and_tails_twice(m, n, k, mode, dtype):
    """Fewer k-blocks than the 4 pipeline stages of the 128 x 256 tile, and tails in every dimension."""
    _check_twice(m, n, k, dtype, mode, seed=m * 7 + n * 3 + k)


def test_many_tiles_per_cta_twice():
    """The stage-2 width, about 12 tiles per CTA."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    m, n, k = 2 * 128 * sms + 77, 1536, 1024
    _check_twice(m, n, k, "bf16", "bias_gelu", seed=m * 7 + n * 3 + k)
