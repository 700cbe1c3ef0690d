"""GPU parity tests of the round-2 kernels (pytest -m gpu, through the C ABI): the fp16-operand GEMM
(f16 tensor cores) and its fp16 epilogue, the error-compensated 3xTF32 GEMM, the 3xTF32 attention core, the fp16
outputs of LayerNorm / attention, the device-side gradient scale, the un-normalised quantiser and the
contention-proof codebook scatter.  Floating-point references are fp64 torch on identical (pre-rounded)
inputs; the tolerance is written at each assert."""
import numpy as np
import pytest
import torch

import enhancing_transformers_b200 as etb
from oracle import vitvq_oracle as O

pytestmark = pytest.mark.gpu
ops = etb.ops
H = torch.float16


def relerr(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


@pytest.fixture(autouse=True)
def _need_cuda():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    torch.manual_seed(0)


def hrand(*shape, scale=1.0):
    return (torch.randn(*shape, device="cuda") * scale).to(H)


# ------------------------------------------------------------------------------- fp16-operand GEMM
@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("M,N,K,bn", [(256, 64, 64, 64), (256, 256, 128, 256), (512, 768, 768, 0), (384, 192, 192, 192),
                                      (256, 96, 160, 64), (1024, 2304, 768, 0), (256, 128, 3072, 128), (32, 288, 64, 0)])
def test_gemm_f16_nt_matches_fp64(cg, M, N, K, bn):
    a, b = hrand(M, K), hrand(N, K)
    c = ops.gemm(a, b, M, N, K, cta_group=cg, bn=bn)
    assert c.dtype == torch.float32
    assert relerr(c, a.double() @ b.double().t()) < 2e-5      # exact products, fp32 accumulation order only


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("M,N,K", [(256, 256, 64), (512, 768, 3072), (256, 128, 192), (1024, 192, 768), (64, 64, 320)])
def test_gemm_f16_nn_dgrad_form(cg, M, N, K):
    a, bs = hrand(M, K), hrand(K, N)
    assert relerr(ops.gemm(a, bs, M, N, K, b_major=1, cta_group=cg), a.double() @ bs.double()) < 2e-5


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("M,N,K,splits", [(256, 256, 128, 1), (768, 768, 4096, 4), (256, 128, 2048, 2), (3072, 768, 2048, 2),
                                          (320, 64, 64, 1), (768, 192, 1024, 2)])
def test_gemm_f16_tn_wgrad_form_with_split_k_and_alpha(cg, M, N, K, splits):
    As, Bs = hrand(K, M), hrand(K, N)
    alpha = torch.tensor([0.125], device="cuda")
    if splits > 1:
        part = ops.gemm(As, Bs, M, N, K // splits, a_major=1, b_major=1, splits=splits, cta_group=cg)
        c = ops.splitk_reduce(part, alpha=alpha)
    else:
        c = ops.gemm(As, Bs, M, N, K, a_major=1, b_major=1, cta_group=cg, alpha=alpha)
    assert relerr(c, 0.125 * (As.double().t() @ Bs.double())) < 2e-5


@pytest.mark.parametrize("cg", [1, 2])
def test_gemm_f16_epilogues(cg):
    M, N, K = 512, 768, 256
    a, b = hrand(M, K), hrand(N, K)
    bias, res = torch.randn(N, device="cuda"), torch.randn(M, N, device="cuda")
    aux = torch.tanh(torch.randn(M, N, device="cuda")).to(H)
    base = a.double() @ b.double().t()
    alpha = torch.tensor([0.5], device="cuda")
    assert relerr(ops.gemm(a, b, M, N, K, bias=bias, res=res, cta_group=cg), base + bias.double() + res.double()) < 1e-5
    assert relerr(ops.gemm(a, b, M, N, K, alpha=alpha, cta_group=cg), 0.5 * base) < 1e-5
    c = ops.gemm(a, b, M, N, K, round_out=True, cta_group=cg)
    assert int((c.view(torch.int32) & 0x1fff).abs().max()) == 0          # tf32-rounded fp32 (feeds the attention core)
    # fp16 output: exactly the fp16 rounding of the fp32-epilogue value
    t = ops.gemm(a, b, M, N, K, bias=bias, act=1, out_half=True, cta_group=cg)
    assert t.dtype == H
    assert relerr(t, torch.tanh(base + bias.double())) < 1e-3             # 2^-11 rounding + fast tanh
    d = ops.gemm(a, b, M, N, K, aux=aux, out_half=True, cta_group=cg)
    assert relerr(d, base * (1 - aux.double() ** 2)) < 1e-3
    d2, cs = ops.gemm(a, b, M, N, K, aux=aux, out_half=True, cta_group=cg, want_colsum=True)
    assert torch.equal(d, d2)
    assert relerr(cs, d.double().sum(0)) < 1e-5                           # column sums of the *stored* fp16 values
    # saturation instead of inf
    big = ops.gemm(a, b, M, N, K, alpha=torch.tensor([1e6], device="cuda"), out_half=True, cta_group=cg)
    assert torch.isfinite(big.float()).all() and big.float().abs().max() == 65504.0


def test_gemm_f16_ragged_edges_and_large_k():
    for (M, N, K) in [(1000, 320, 192), (40, 64, 64), (130, 200, 72)]:
        a, b = hrand(M, K), hrand(N, K)
        assert relerr(ops.gemm(a, b, M, N, K, cta_group=2), a.double() @ b.double().t()) < 2e-5
        t = ops.gemm(a, b, M, N, K, out_half=True, cta_group=2)
        assert relerr(t, a.double() @ b.double().t()) < 1e-3


# ------------------------------------------------------------------------------------- 3xTF32 GEMM
@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("M,N,K", [(256, 256, 256), (512, 768, 768), (1024, 32, 768), (512, 768, 32), (256, 128, 3072)])
def test_gemm_3xtf32_is_fp32_grade(cg, M, N, K):
    a, b = torch.randn(M, K, device="cuda"), torch.randn(N, K, device="cuda")      # NOT pre-rounded
    ref = a.double() @ b.double().t()
    c3 = ops.gemm(a, b, M, N, K, a_lo=ops.split_tf32_lo(a), b_lo=ops.split_tf32_lo(b), cta_group=cg)
    c1 = ops.gemm(a, b, M, N, K, cta_group=cg)
    e3, e1 = relerr(c3, ref), relerr(c1, ref)
    assert e3 < 2e-6 * max(1.0, (K / 256) ** 0.5), e3      # fp32 sgemm-level (grows like sqrt(K): fp32 accumulation)
    assert e1 > 20 * e3                                      # and far better than the single truncating pass


def test_gemm_3xtf32_dgrad_and_wgrad_forms():
    M, N, K = 512, 256, 384
    a, bs = torch.randn(M, K, device="cuda"), torch.randn(K, N, device="cuda")
    c = ops.gemm(a, bs, M, N, K, b_major=1, a_lo=ops.split_tf32_lo(a), b_lo=ops.split_tf32_lo(bs), cta_group=2)
    assert relerr(c, a.double() @ bs.double()) < 3e-6
    As, Bs = torch.randn(2048, 256, device="cuda"), torch.randn(2048, 128, device="cuda")
    part = ops.gemm(As, Bs, 256, 128, 1024, a_major=1, b_major=1, splits=2, a_lo=ops.split_tf32_lo(As),
                    b_lo=ops.split_tf32_lo(Bs), cta_group=2)
    assert relerr(ops.splitk_reduce(part), As.double().t() @ Bs.double()) < 3e-6


def test_split_tf32_lo_is_exact():
    x = torch.randn(4096, device="cuda") * torch.logspace(-6, 6, 4096, device="cuda")
    lo = ops.split_tf32_lo(x)
    hi = (x.view(torch.int32) & ~0x1fff).view(torch.float32)
    assert torch.equal(hi + lo, x)
    assert (lo.abs() <= hi.abs() * 2.0 ** -10 + 1e-45).all()


# ------------------------------------------------------------------------- exact (3xTF32) attention
@pytest.mark.parametrize("B,N,heads,dh", [(2, 16, 2, 32), (1, 24, 3, 64), (2, 200, 2, 64), (1, 1024, 2, 64), (1, 130, 1, 32)])
def test_attention_exact_fwd_bwd(B, N, heads, dh):
    inner = heads * dh
    qkv = torch.randn(B * N, 3 * inner, device="cuda")                    # unrounded fp32
    scale = dh ** -0.5
    o, lse = ops.attention_exact_fwd(qkv, B, N, heads, dh, scale)
    q, k, v = (t.reshape(B, N, heads, dh).permute(0, 2, 1, 3).double() for t in qkv.split(inner, dim=-1))
    q.requires_grad_(True); k.requires_grad_(True); v.requires_grad_(True)
    s = (q @ k.transpose(-1, -2)) * scale
    oref = (torch.softmax(s, -1) @ v).permute(0, 2, 1, 3).reshape(B * N, inner)
    assert relerr(o, oref.detach()) < 3e-5                   # exp2f (2 ulp) on scores up to ~|15|: fp32-grade, not tf32-grade (1e-4)
    assert relerr(lse, torch.logsumexp(s, -1).reshape(-1).detach()) < 2e-6
    do = torch.randn(B * N, inner, device="cuda")
    oref.backward(do.double())
    dqkv = ops.attention_exact_bwd(qkv, o, lse, do, B, N, heads, dh, scale)
    dref = torch.cat([t.grad.permute(0, 2, 1, 3).reshape(B * N, inner) for t in (q, k, v)], dim=-1)
    for i, nm in enumerate("qkv"):
        assert relerr(dqkv[:, i * inner:(i + 1) * inner], dref[:, i * inner:(i + 1) * inner]) < 2e-5, nm


# ----------------------------------------------------------------- fp16 outputs of the producer kernels
@pytest.mark.parametrize("M,D", [(64, 64), (1000, 192), (4096, 768), (512, 1280)])
def test_layernorm_fp16_outputs(M, D):
    x = torch.randn(M, D, device="cuda") * 3 + 1
    g, b = torch.randn(D, device="cuda"), torch.randn(D, device="cuda")
    y32, mean, rstd = ops.layernorm_fwd(x, g, b, False)
    y16, mean2, rstd2 = ops.layernorm_fwd(x, g, b, False, out_half=True)
    assert y16.dtype == H and torch.equal(y16, y32.to(H)) and torch.equal(mean, mean2) and torch.equal(rstd, rstd2)
    dy, dres = torch.randn(M, D, device="cuda") * 1e-6, torch.randn(M, D, device="cuda") * 1e-6
    sc = ops.grad_scale(dres)
    dx, dg, db, dxs = ops.layernorm_bwd(dy, x, mean, rstd, g, dres, want_colsum=True)
    dx2, dg2, db2, dxs2, dxh = ops.layernorm_bwd(dy, x, mean, rstd, g, dres, want_colsum=True, half_scale=sc[0:1])
    assert torch.equal(dx, dx2) and torch.equal(dg, dg2)
    assert torch.equal(dxh, (dx * sc[0]).to(H))
    # fp16 dy carrying the gradient scale (what an fp16 dgrad GEMM hands over): the kernel multiplies by 1/S as it reads,
    # so the result is bit-identical to the fp32 path fed with the same (fp16-representable) values
    dyh = ops.to_half(dy, sc[0:1])
    dy_rt = dyh.float() * sc[1]
    dx3, dg3, db3, dxs3 = ops.layernorm_bwd(dy_rt, x, mean, rstd, g, dres, want_colsum=True)
    dx4, dg4, db4, dxs4 = ops.layernorm_bwd(dyh, x, mean, rstd, g, dres, want_colsum=True, dy_scale=sc[1:2])
    assert torch.equal(dx3, dx4) and torch.equal(dg3, dg4) and torch.equal(db3, db4) and torch.equal(dxs3, dxs4)


def test_grad_scale_and_to_half():
    g = torch.randn(1 << 20, device="cuda") * 3e-8
    sc = ops.grad_scale(g).cpu()
    amax = g.abs().max().item()
    assert sc[0] * sc[1] == 1.0 and float(np.log2(sc[0].item())).is_integer()
    assert 2.0 ** 5 <= amax * sc[0].item() <= 2.0 ** 6                      # max|g| * S in (2^5, 2^6]
    gh = ops.to_half(g, ops.grad_scale(g)[0:1])
    assert torch.equal(gh, (g * sc[0].item()).to(H))
    assert torch.equal(ops.grad_scale(torch.zeros(64, device="cuda")).cpu(), torch.tensor([1.0, 1.0]))
    h = ops.to_half(torch.tensor([1e9, -1e9, 1.0, float("nan")], device="cuda"))
    assert h[0] == 65504 and h[1] == -65504 and h[2] == 1


@pytest.mark.parametrize("B,N,heads,dh", [(2, 200, 2, 64), (1, 130, 2, 32), (2, 1024, 3, 64)])
def test_attention_fp16_io_matches_fp32_io(B, N, heads, dh):
    inner = heads * dh
    i = torch.randn(B * N, 3 * inner, device="cuda").view(torch.int32)
    qkv = ((i + 0x1000) & ~0x1fff).view(torch.float32)
    scale = dh ** -0.5
    o32, lse = ops.attention_fwd(qkv, B, N, heads, dh, scale, False)
    o16, lse2 = ops.attention_fwd(qkv, B, N, heads, dh, scale, False, out_half=True)
    assert torch.equal(o16, o32.to(H)) and torch.equal(lse, lse2)
    do = torch.randn(B * N, inner, device="cuda") * 1e-5
    sc = ops.grad_scale(do)
    d32 = ops.attention_bwd(qkv, o32, lse, do, B, N, heads, dh, scale, False)
    d16 = ops.attention_bwd(qkv, o32, lse, do, B, N, heads, dh, scale, False, half_scale=sc[0:1])
    assert d16.dtype == H
    assert relerr(d16.float() * sc[1], d32) < 1e-3                        # fp16 rounding of the same accumulators
    # delta from the fp16 copy of O: a 2^-11 perturbation of O
    d16b = ops.attention_bwd(qkv, o16, lse, do, B, N, heads, dh, scale, False, half_scale=sc[0:1])
    assert relerr(d16b.float() * sc[1], d32) < 3e-3


# ------------------------------------------------------------------------------------- quantiser
def test_vq_without_normalisation_matches_torch_reference():
    """use_norm=False (reference quantizers.py:24: norm is the identity)"""
    z = torch.randn(2048, 32, device="cuda", requires_grad=True)
    E = torch.randn(512, 32, device="cuda", requires_grad=True)
    out, loss, idx = ops.vq_fwd(z.detach(), E.detach(), 1, 0.25, use_norm=False)
    d = (z.detach() ** 2).sum(1, keepdim=True) + (E.detach() ** 2).sum(1) - 2 * z.detach() @ E.detach().t()
    ref_idx = d.argmin(1)
    mism = (idx.view(-1) != ref_idx).nonzero().view(-1)
    if mism.numel():      # cuBLAS-ordered fp32 distances vs sequential FMA: only exact near-ties may differ
        d64 = ((z.detach()[mism].double()[:, None] - E.detach().double()[None]) ** 2).sum(-1)
        top2 = d64.topk(2, largest=False).values
        assert ((top2[:, 1] - top2[:, 0]) < 1e-4).all()
    zq = E[idx.view(-1)]
    lref = 0.25 * ((zq.detach() - z) ** 2).mean() + ((zq - z.detach()) ** 2).mean()
    assert abs(loss.item() - lref.item()) < 1e-5 * abs(lref.item())
    assert torch.allclose(out, z.detach() + (zq.detach() - z.detach()), atol=1e-6)
    g_out = torch.randn(2048, 32, device="cuda")
    gz, gE = ops.vq_bwd(z.detach(), E.detach(), idx, g_out, torch.tensor(1.0, device="cuda"), False, 0.25, use_norm=False)
    (lref + (z * g_out).sum()).backward()
    assert torch.allclose(gz, z.grad, atol=1e-6) and torch.allclose(gE, E.grad, atol=1e-6)


@pytest.mark.parametrize("depth", [1, 4])
def test_vq_bwd_clustered_codes_scatter(depth):
    """all tokens on a handful of codes (what an encoder produces at initialisation): the shared-memory
    accumulation must give the same codebook gradient as the oracle's dense scatter"""
    torch.manual_seed(1)
    E = torch.randn(8192, 32)
    base = E[torch.randint(0, 5, (16384,))]
    z = (base + 0.01 * torch.randn(16384, 32)).contiguous()
    out, loss, idx = ops.vq_fwd(z.cuda(), E.cuda(), depth, 0.25)
    assert idx[:, 0].unique().numel() <= 5
    g_out = torch.randn(16384, 32)
    gz, gE = ops.vq_bwd(z.cuda(), E.cuda(), idx, g_out.cuda(), torch.tensor(1.0, device="cuda"), depth > 1, 0.25)
    gz_ref, gE_ref = O.vq_backward_np(z.numpy(), E.numpy(), idx.cpu().numpy(), g_out.numpy(), 1.0, 0.25, depth > 1)
    np.testing.assert_allclose(gz.cpu().numpy(), gz_ref, rtol=1e-4, atol=1e-9)
    np.testing.assert_allclose(gE.cpu().numpy(), gE_ref, rtol=2e-3, atol=1e-7)


def test_vq_ffma2_codes_bit_exact_large():
    """the packed-FMA distance loop must keep the reference's indices on 32k x 8192 (numpy oracle, fp32 FMA order)"""
    torch.manual_seed(3)
    z, E = torch.randn(32768, 32), torch.randn(8192, 32)
    _, _, idx = ops.vq_fwd(z.cuda(), E.cuda(), 1, 0.25)
    ref = O.vq_lookup_np(z.numpy(), E.numpy())
    mism = np.nonzero(idx.cpu().numpy().reshape(-1) != ref)[0]
    if mism.size:
        gaps = O.vq_top2_gap_f64(z.numpy()[mism], E.numpy())
        assert (gaps < 1e-6).all(), (mism.size, gaps.max())
    assert mism.size <= 4


# --------------------------------------------------------------------------- fp16-operand attention core
@pytest.mark.parametrize("B,N,heads", [(1, 24, 3), (2, 200, 2), (2, 1024, 4), (1, 130, 1), (3, 64, 2), (1, 1024, 12)])
def test_attention_f16_fwd_bwd(B, N, heads):
    dh, inner = 64, heads * 64
    qkv = torch.randn(B * N, 3 * inner, device="cuda").to(H)
    scale = dh ** -0.5
    o, lse = ops.attention_f16_fwd(qkv, B, N, heads, dh, scale)
    assert o.dtype == H
    q, k, v = (t.reshape(B, N, heads, dh).permute(0, 2, 1, 3).double() for t in qkv.split(inner, dim=-1))
    q.requires_grad_(True); k.requires_grad_(True); v.requires_grad_(True)
    s = (q @ k.transpose(-1, -2)) * scale
    oref = (torch.softmax(s, -1) @ v).permute(0, 2, 1, 3).reshape(B * N, inner)
    assert relerr(o, oref.detach()) < 1.5e-3                      # fp16 P (2^-11) + fp16 output rounding
    assert relerr(lse, torch.logsumexp(s, -1).reshape(-1).detach()) < 1e-5
    # backward: dout carries a gradient scale; dqkv comes back with the same scale
    do = torch.randn(B * N, inner, device="cuda") * 1e-6
    sc = ops.grad_scale(do)
    doh = ops.to_half(do, sc[0:1])
    oref.backward(doh.double() * sc[1].double())
    dqkv = ops.attention_f16_bwd(qkv, o, lse, doh, B, N, heads, dh, scale).double() * sc[1].double()
    dref = torch.cat([t.grad.permute(0, 2, 1, 3).reshape(B * N, inner) for t in (q, k, v)], dim=-1)
    for i, nm in enumerate("qkv"):
        assert relerr(dqkv[:, i * inner:(i + 1) * inner], dref[:, i * inner:(i + 1) * inner]) < 3e-3, nm


def test_attention_f16_matches_tf32_core():
    """same inputs through the tf32 core (fp16 values are exactly representable in tf32): outputs agree to
    fp16 rounding, i.e. the fp16 core loses nothing against the tf32 one"""
    B, N, heads, dh = 2, 512, 3, 64
    inner = heads * dh
    qkv = torch.randn(B * N, 3 * inner, device="cuda").to(H)
    o16, lse16 = ops.attention_f16_fwd(qkv, B, N, heads, dh, 0.125)
    o32, lse32 = ops.attention_fwd(qkv.float(), B, N, heads, dh, 0.125, False)
    assert relerr(o16, o32) < 1.5e-3 and relerr(lse16, lse32) < 1e-5
