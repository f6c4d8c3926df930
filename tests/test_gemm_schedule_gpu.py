"""Tile schedules of the wgmma GEMM (ab_gemm_bf16).  For K <= 1024 and N > 128 the two math warpgroups of a CTA take
alternate 128 x 128 tiles of its persistent tile sequence ("ping-pong"); otherwise both work on every tile.  Tile
counts around multiples of the grid, tails in every dimension, both operand types, every epilogue mode and every GEMM
shape of a full-size forecast step are checked against an fp32 PyTorch reference of the same op."""

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


MODES = {  # bias, gelu, out_f32, residual
    "plain": (False, False, False, False),
    "bias_gelu": (True, True, False, False),
    "bias_res_f32_dual": (True, False, True, True),
}


def _mode(name, out16):
    bias, gelu, f32, res = MODES[name]
    return bias, gelu, f32, out16, res


@pytest.mark.parametrize("tiles", ["2", "sms", "sms+2", "2sms+2", "3sms+2"])
@pytest.mark.parametrize("mode", sorted(MODES))
def test_tile_counts_around_the_grid(tiles, mode):
    """N = 256, K = 320: ping-pong, two 128-column tiles per 128 rows (so tile counts are even); the last row block
    has a 40-row tail.  2: one tile per CTA on two CTAs, the second warpgroup idle; sms: one tile per CTA; sms + 2: two
    CTAs with one tile per warpgroup; 2 sms + 2: two CTAs with an odd count; 3 sms + 2: most CTAs with one tile more
    on the first warpgroup than on the second."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    t = {"2": 2, "sms": sms, "sms+2": sms + 2, "2sms+2": 2 * sms + 2, "3sms+2": 3 * sms + 2}[tiles]
    m = 128 * ((t + 1) // 2 - 1) + 40
    _check(m, 256, 320, "bf16", *_mode(mode, "bf16"), seed=t)


@pytest.mark.parametrize("m,n,k", [
    (257, 200, 136),    # ping-pong: two 128-column blocks, the second with 72 live columns
    (517, 136, 1024),   # ping-pong: 8 live columns in the second block, longest K of the schedule
    (131, 520, 72),     # ping-pong: N tail inside a 64-column epilogue box, K tail
    (3000, 1032, 520),  # ping-pong: many tiles per CTA, K tail
    (1000, 300, 1096),  # cooperative 128 x 256 tile (K > 1024), K tail
    (1000, 80, 72),     # decoder-head width (cooperative 128 x 128), K tail
    (300, 64, 200),     # the 64-wide tile, M and K tails
])
@pytest.mark.parametrize("mode", sorted(MODES))
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
    """The accumulation order over K is fixed by the kernel, not by which warpgroup or CTA takes a tile (K = 1024:
    ping-pong, K = 2048: cooperative)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    args = (2 * 128 * sms + 77, 1536, k, "bf16", *_mode(mode, "bf16"))
    first = _gemm(*args, seed=5)
    second = _gemm(*args, seed=5)
    assert torch.equal(first[0], second[0])
    if first[1] is not None:
        assert torch.equal(first[1], second[1])
