"""GPU tests of the wgmma fp16 attention core (ops.attention_f16_fwd / ops.attention_f16_bwd): tiles that run past N
stay inside their own image and head, repeated calls are bit-identical, and the benchmark's shape matches fp64."""
import pytest
import torch

import enhancing_transformers_b200 as etb

pytestmark = pytest.mark.gpu
ops = etb.ops
H = torch.float16
DH = 64


def relerr(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


@pytest.fixture(autouse=True)
def _need_cuda():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    torch.manual_seed(0)


def run(qkv, dout, B, N, heads):
    o, lse = ops.attention_f16_fwd(qkv, B, N, heads, DH, DH ** -0.5)
    dqkv = ops.attention_f16_bwd(qkv, o, lse, dout, B, N, heads, DH, DH ** -0.5)
    return o, lse, dqkv


@pytest.mark.parametrize("N", [200, 130])
def test_images_and_heads_do_not_leak(N):
    """every other image and head scaled by 100: the image and head under test do not change, bit for bit"""
    B, heads, b0, h0 = 3, 3, 1, 1
    inner = heads * DH
    qkv = torch.randn(B * N, 3 * inner, device="cuda").to(H)
    dout = (torch.randn(B * N, inner, device="cuda") * 1e-2).to(H)
    o, lse, dqkv = run(qkv, dout, B, N, heads)

    def others_x100(x, parts):
        y = x.view(B, N, parts, heads, DH).clone()
        keep = y[b0, :, :, h0].clone()
        y *= 100
        y[b0, :, :, h0] = keep
        return y.view(B * N, parts * inner)

    o2, lse2, dqkv2 = run(others_x100(qkv, 3), others_x100(dout, 1), B, N, heads)
    sel = lambda x, parts: x.view(B, N, parts, heads, DH)[b0, :, :, h0]
    assert torch.equal(sel(o, 1), sel(o2, 1))
    assert torch.equal(lse.view(B, heads, N)[b0, h0], lse2.view(B, heads, N)[b0, h0])
    assert torch.equal(sel(dqkv, 3), sel(dqkv2, 3))


def test_repeated_calls_are_bit_identical():
    B, N, heads = 16, 1024, 12
    inner = heads * DH
    qkv = torch.randn(B * N, 3 * inner, device="cuda").to(H)
    dout = (torch.randn(B * N, inner, device="cuda") * 1e-2).to(H)
    first, second = run(qkv, dout, B, N, heads), run(qkv, dout, B, N, heads)
    for a, b in zip(first, second):
        assert torch.equal(a, b)


@pytest.mark.parametrize("do_scale", [1.0, 1e-7])
def test_bench_shape_matches_fp64(do_scale):
    """B = 8 images of the base config's attention (1024 tokens, 12 x 64 heads); dO of unit size and of the size a
    per-image loss gradient has, carried in fp16 by the power-of-two gradient scale as the backward does"""
    B, N, heads = 8, 1024, 12
    inner = heads * DH
    scale = DH ** -0.5
    qkv = torch.randn(B * N, 3 * inner, device="cuda").to(H)
    do = torch.randn(B * N, inner, device="cuda") * do_scale
    sc = ops.grad_scale(do)
    dout = ops.to_half(do, sc[0:1])
    o, lse, dqkv = run(qkv, dout, B, N, heads)
    dqkv = dqkv.double() * sc[1].double()
    q, k, v = (t.reshape(B, N, heads, DH).permute(0, 2, 1, 3).double().requires_grad_(True) for t in qkv.split(inner, dim=-1))
    s = (q @ k.transpose(-1, -2)) * scale
    oref = (torch.softmax(s, -1) @ v).permute(0, 2, 1, 3).reshape(B * N, inner)
    assert relerr(o, oref.detach()) < 1.5e-3
    assert relerr(lse, torch.logsumexp(s, -1).reshape(-1).detach()) < 1e-5
    oref.backward(dout.double() * sc[1].double())
    for i, t in enumerate((q, k, v)):
        ref = t.grad.permute(0, 2, 1, 3).reshape(B * N, inner)
        assert relerr(dqkv[:, i * inner:(i + 1) * inner], ref) < 3e-3, "qkv"[i]
