"""The fp16 GEMM is persistent: each CTA walks a strided list of tiles while its producer warp runs ahead through the
shared-memory ring into the next tile.  With a full grid and the small shapes of the other GEMM tests most CTAs run one
or two tiles, so the hand-over from one tile to the next is barely exercised.  These tests cap the grid at a few CTAs,
so that each one runs 8 or more tiles back-to-back, on M and N that are ragged against the 128-row tile and the
256-column edge, and check every epilogue form of the fp16 data path against fp64 torch and bit-for-bit against the
uncapped grid (the tile order must not change a bit)."""
import os

import pytest
import torch

import enhancing_transformers_b200 as etb

pytestmark = pytest.mark.gpu
ops = etb.ops
H = torch.float16
CAPPED_CTAS = 2


def relerr(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


def hrand(*shape, scale=1.0):
    return (torch.randn(*shape, device="cuda") * scale).to(H)


@pytest.fixture(autouse=True)
def _restore_sm_limit():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    torch.manual_seed(0)
    yield
    ops.set_sm_limit(int(os.environ.get("B200VQ_SM_LIMIT", "0") or 0))


def full_and_capped(fn):
    """fn() on the full grid and on CAPPED_CTAS CTAs"""
    ops.set_sm_limit(0)
    full = fn()
    ops.set_sm_limit(CAPPED_CTAS)
    capped = fn()
    ops.set_sm_limit(0)
    torch.cuda.synchronize()
    return full, capped


def tiles(M, N, splits=1):
    """a lower bound on the tile count: the kernel's tiles are 128 rows by at most 256 columns"""
    return -(-M // 128) * -(-N // 256) * splits


# the last row block is 104 rows; N = 648 is not a multiple of 64, 128 or 256
M, N, K = 1000, 648, 320


def test_enough_tiles_per_cta():
    assert min(tiles(M, N), tiles(M, 640), tiles(640, 576, 3)) >= 8 * CAPPED_CTAS


def test_fp32_out_bias_and_residual():
    a, b = hrand(M, K), hrand(N, K)
    bias, res = torch.randn(N, device="cuda"), torch.randn(M, N, device="cuda")
    full, capped = full_and_capped(lambda: ops.gemm(a, b, M, N, K, bias=bias, res=res))
    assert torch.equal(full, capped)
    assert relerr(capped, a.double() @ b.double().t() + bias.double() + res.double()) < 1e-5


def test_fp16_out_bias_and_tanh():
    a, b = hrand(M, K), hrand(N, K, scale=0.1)
    bias = torch.randn(N, device="cuda")
    full, capped = full_and_capped(lambda: ops.gemm(a, b, M, N, K, bias=bias, act=1, out_half=True))
    assert full.dtype == H and torch.equal(full, capped)
    assert relerr(capped, torch.tanh(a.double() @ b.double().t() + bias.double())) < 1e-3   # 2^-11 rounding + fast tanh


def test_fp16_out_tanh_backward_input_and_column_sums():
    # the dgrad form of fc1's backward: B MN-major (N in whole 64-column atoms: 640 = 256 + 256 + 128), aux = the
    # forward's fp16 tanh output
    N = 640
    a, bs = hrand(M, K), hrand(K, N)
    aux = torch.tanh(torch.randn(M, N, device="cuda")).to(H)
    full, capped = full_and_capped(lambda: ops.gemm(a, bs, M, N, K, b_major=1, aux=aux, out_half=True, want_colsum=True))
    assert torch.equal(full[0], capped[0]) and torch.equal(full[1], capped[1])
    d, cs = capped
    assert relerr(d, (a.double() @ bs.double()) * (1 - aux.double() ** 2)) < 1e-3
    assert relerr(cs, d.double().sum(0)) < 1e-5                            # column sums of the *stored* fp16 values


def test_fp16_out_alpha():
    a, b = hrand(M, K), hrand(N, K)
    alpha = torch.tensor([0.25], device="cuda")
    full, capped = full_and_capped(lambda: ops.gemm(a, b, M, N, K, alpha=alpha, out_half=True))
    assert torch.equal(full, capped)
    assert relerr(capped, 0.25 * (a.double() @ b.double().t())) < 1e-3


def test_split_k_wgrad():
    # MN-major operands need M and N in whole 64-element atoms; 576 = 256 + 256 + 64
    rows, cols, tokens, splits = 640, 576, 3 * 384, 3
    dy, x = hrand(tokens, rows), hrand(tokens, cols)
    full, capped = full_and_capped(lambda: ops.gemm(dy, x, rows, cols, tokens // splits, a_major=1, b_major=1, splits=splits))
    assert full.shape == (splits, rows, cols) and torch.equal(full, capped)
    ref = dy.double().view(splits, tokens // splits, rows).transpose(1, 2) @ x.double().view(splits, tokens // splits, cols)
    assert relerr(capped, ref) < 2e-5
