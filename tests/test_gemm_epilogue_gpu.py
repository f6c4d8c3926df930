"""The 16-bit-only epilogue of the wgmma GEMM (ab_gemm_bf16 with a bf16 / fp16 output, no fp32 output, no residual):
the tile's bias copied into shared memory when the tile starts, bias / GELU / rounding on the registers, stmatrix into
the staging boxes and TMA stores.  Checked against an fp32 PyTorch reference: N tails that are not multiples of 8, 64
or the tile width (no write may land past the 16-byte chunk holding column N - 1), M tails, many tiles per CTA (the bias
copy is refilled every tile), both output types with and without GELU, no bias, and repeat launches."""

import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}
SENTINEL = -1000.0  # exactly representable in bf16 and fp16


@pytest.fixture(autouse=True)
def _no_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = saved


def _run(m, n, k, dtype, gelu, bias=True, pad=0, seed=0):
    """16-bit output of the kernel (a view of width n into rows of n + pad columns, pre-filled with SENTINEL), the
    whole padded buffer, and the fp32 reference."""
    from aurora_b200 import cabi

    g = torch.Generator(device="cuda").manual_seed(seed)
    dt = DTYPES[dtype]
    a = torch.randn(m, k, device="cuda", generator=g).to(dt)
    w = (torch.randn(n, k, device="cuda", generator=g) / k**0.5).to(dt)
    b = 4.0 * torch.randn(n, device="cuda", generator=g) if bias else None  # large enough to show a misplaced column
    buf = torch.full((m, n + pad), SENTINEL, device="cuda", dtype=dt)
    out = buf[:, :n]
    cabi.gemm(a, w, bias=b, out_bf16=out, act=cabi.AB_ACT_GELU_ERF if gelu else cabi.AB_ACT_NONE)
    torch.cuda.synchronize()
    y = a.float() @ w.float().t()
    if b is not None:
        y += b
    if gelu:
        y = torch.nn.functional.gelu(y)
    return out, buf, y


def _check(m, n, k, dtype, gelu, bias=True, pad=0, seed=0):
    out, buf, y = _run(m, n, k, dtype, gelu, bias=bias, pad=pad, seed=seed)
    torch.testing.assert_close(out.float(), y, rtol=1e-2, atol=1e-2)
    if pad:  # the TMA store writes the 16-byte chunk that holds column N - 1 whole, nothing after it
        assert bool((buf[:, -(-n // 8) * 8:] == SENTINEL).all()), "a store landed past the row's last 16-byte chunk"


@pytest.mark.parametrize("m,n,k", [
    (300, 131, 256),    # 128 x 256: 3 live columns in the third 64-column box
    (1000, 1029, 512),  # 128 x 256: 5 live columns in the last tile
    (257, 190, 1024),   # 128 x 256: N tail inside the third 64-column box, 62 = 7 groups of 8 + 6
    (500, 303, 1088),   # 128 x 256, K tail past 1024: 47 live columns in the second tile
    (333, 83, 136),     # 128 x 128: 19 live columns in the second 64-column box
    (141, 61, 64),      # the 64-wide tile: 61 of 64 columns
])
@pytest.mark.parametrize("gelu", [False, True], ids=["bias", "bias_gelu"])
@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
def test_n_and_m_tails(m, n, k, dtype, gelu):
    """Rows padded to a multiple of 8 columns plus 8: the last 8 must keep their sentinel."""
    _check(m, n, k, dtype, gelu, pad=(-n) % 8 + 8, seed=m + n)


@pytest.mark.parametrize("n,k,gelu", [(1536, 512, False), (520, 1024, True), (700, 2048, False), (200, 256, True)])
@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
def test_many_tiles_per_cta(n, k, gelu, dtype):
    """Dozens of tiles per CTA, with N-blocks of different bias values following each other on the same warps."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    m = 128 * sms * 6 // max(1, n // 256) + 45
    _check(m, n, k, dtype, gelu, seed=n + k)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
def test_without_bias(dtype):
    _check(777, 333, 320, dtype, gelu=True, bias=False, pad=3, seed=3)


@pytest.mark.parametrize("n,k", [(1029, 1024), (303, 2048)])
def test_two_launches_are_bit_identical(n, k):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    args = (2 * 128 * sms + 77, n, k, "bf16", True)
    first = _run(*args, pad=(-n) % 8, seed=9)[1]
    second = _run(*args, pad=(-n) % 8, seed=9)[1]
    assert torch.equal(first, second)
