"""GPU parity tests of the individual C-ABI kernels (run on an H100: pytest -m gpu).
References: exact integer/index parity against the oracle and the golden fixtures; floating
point against fp64 torch on the same (tf32-pre-rounded, where the tensor cores consume them)
inputs with the tolerance written at each assert."""
import os

import numpy as np
import pytest
import torch

import enhancing_transformers_b200 as etb
from oracle import vitvq_oracle as O

pytestmark = pytest.mark.gpu
ops = etb.ops


def tf32_rn(t):
    i = t.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1fff).view(torch.float32)


def relerr(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


@pytest.fixture(autouse=True)
def _need_cuda():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    torch.manual_seed(0)


# ------------------------------------------------------------------------------------------ GEMM
@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("M,N,K,bn", [(256, 64, 32, 64), (256, 256, 64, 256), (512, 768, 768, 0), (384, 192, 96, 192),
                                      (256, 96, 160, 64), (1024, 2304, 768, 0), (256, 128, 3072, 128), (32, 288, 64, 0)])
def test_gemm_nt_matches_fp64(cg, M, N, K, bn):
    a, b = tf32_rn(torch.randn(M, K, device="cuda")), tf32_rn(torch.randn(N, K, device="cuda"))
    c = ops.gemm(a, b, M, N, K, cta_group=cg, bn=bn)
    assert relerr(c, a.double() @ b.double().t()) < 2e-5      # fp32 accumulation order only


@pytest.mark.parametrize("cg", [1, 2])
def test_gemm_epilogues(cg):
    M, N, K = 512, 768, 256
    a, b = tf32_rn(torch.randn(M, K, device="cuda")), tf32_rn(torch.randn(N, K, device="cuda"))
    bias, res = torch.randn(N, device="cuda"), torch.randn(M, N, device="cuda")
    aux, pos = torch.tanh(torch.randn(M, N, device="cuda")), torch.randn(128, N, device="cuda")
    base = a.double() @ b.double().t()
    assert relerr(ops.gemm(a, b, M, N, K, bias=bias, cta_group=cg), base + bias.double()) < 1e-5
    assert relerr(ops.gemm(a, b, M, N, K, bias=bias, act=1, cta_group=cg), torch.tanh(base + bias.double())) < 1e-4
    assert relerr(ops.gemm(a, b, M, N, K, bias=bias, res=res, cta_group=cg), base + bias.double() + res.double()) < 1e-5
    assert relerr(ops.gemm(a, b, M, N, K, res=pos, res_row_mod=128, cta_group=cg), base + pos.double().repeat(4, 1)) < 1e-5
    assert relerr(ops.gemm(a, b, M, N, K, aux=aux, cta_group=cg), base * (1 - aux.double() ** 2)) < 1e-5
    c = ops.gemm(a, b, M, N, K, round_out=True, cta_group=cg)
    assert int((c.view(torch.int32) & 0x1fff).abs().max()) == 0          # stored values are tf32
    assert torch.equal(c, tf32_rn(ops.gemm(a, b, M, N, K, cta_group=cg)))


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("M,N,K", [(512, 768, 256), (1000, 320, 96), (40, 64, 64), (4096, 3072, 128)])
def test_gemm_epilogue_column_sums(cg, M, N, K):
    """the epilogue's per-16-row partial column sums reduce to colsum of the *stored* C (ragged M and N included)"""
    a, bs = tf32_rn(torch.randn(M, K, device="cuda")), tf32_rn(torch.randn(K, N, device="cuda"))
    aux, bias = torch.tanh(torch.randn(M, N, device="cuda")), torch.randn(N, device="cuda")
    c, cs = ops.gemm(a, bs, M, N, K, b_major=1, aux=aux, bias=bias, round_out=True, cta_group=cg, want_colsum=True)
    assert torch.equal(c, ops.gemm(a, bs, M, N, K, b_major=1, aux=aux, bias=bias, round_out=True, cta_group=cg))
    assert relerr(cs, c.double().sum(0)) < 1e-5


def test_gemm_epilogue_input_refill_is_race_free():
    """Regression: the epilogue's TMA refill of the tanh'/residual input box used to be ordered only against the
    *issue* of the shared-memory loads of the previous box; with a short K loop (tensor cores saturating shared
    memory) and a busier epilogue (column sums) ~10% of launches of this shape stored one stale 16-byte group."""
    M, N, K = 4096, 3072, 128
    for it in range(40):
        a, bs = tf32_rn(torch.randn(M, K, device="cuda")), tf32_rn(torch.randn(K, N, device="cuda"))
        aux, bias = torch.tanh(torch.randn(M, N, device="cuda")), torch.randn(N, device="cuda")
        kw = dict(b_major=1, aux=aux, bias=bias, round_out=True, cta_group=2)
        c1, _ = ops.gemm(a, bs, M, N, K, want_colsum=True, **kw)
        c2 = ops.gemm(a, bs, M, N, K, **kw)
        assert torch.equal(c1, c2), f"iteration {it}: {(c1 != c2).sum().item()} elements differ"
    ref = ((a.double() @ bs.double()) + bias.double()) * (1 - aux.double() ** 2)
    assert relerr(c1, ref) < 1e-3          # tf32-rounded output


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("M,N,K", [(256, 256, 64), (512, 768, 3072), (256, 96, 160), (1024, 192, 768), (32, 64, 288)])
def test_gemm_nn_dgrad_form(cg, M, N, K):
    a, bs = tf32_rn(torch.randn(M, K, device="cuda")), tf32_rn(torch.randn(K, N, device="cuda"))
    c = ops.gemm(a, bs, M, N, K, b_major=1, cta_group=cg)
    assert relerr(c, a.double() @ bs.double()) < 2e-5


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("M,N,K,splits", [(256, 256, 128, 1), (768, 768, 4096, 4), (256, 96, 2048, 2), (3072, 768, 2048, 2),
                                          (288, 64, 32, 1)])
def test_gemm_tn_wgrad_form_with_split_k(cg, M, N, K, splits):
    As, Bs = tf32_rn(torch.randn(K, M, device="cuda")), tf32_rn(torch.randn(K, N, device="cuda"))
    part = ops.gemm(As, Bs, M, N, K // splits, a_major=1, b_major=1, splits=splits, cta_group=cg)
    c = ops.splitk_reduce(part) if splits > 1 else part
    assert relerr(c, As.double().t() @ Bs.double()) < 2e-5


def test_gemm_hardware_truncates_unrounded_operands():
    """documents why operands are pre-rounded: a tf32 MMA drops the low 13 mantissa bits"""
    a, b = torch.randn(256, 256, device="cuda"), torch.randn(256, 256, device="cuda")
    c = ops.gemm(a, b, 256, 256, 256)
    trunc = lambda t: (t.view(torch.int32) & ~0x1fff).view(torch.float32)
    assert relerr(c, trunc(a).double() @ trunc(b).double().t()) < 1e-5


def test_gemm_rejects_bad_arguments():
    a = torch.randn(64, 30, device="cuda")
    with pytest.raises(RuntimeError, match="lda/ldb"):
        ops.gemm(a, a, 64, 64, 30)
    with pytest.raises(RuntimeError, match="no CPU path"):
        ops.gemm(torch.randn(64, 32), torch.randn(64, 32), 64, 64, 32)


# ------------------------------------------------------------------------------------- row-wise
@pytest.mark.parametrize("M,D", [(64, 64), (1000, 96), (4096, 768), (512, 1280), (256, 512), (8, 2048)])
def test_layernorm_fwd_bwd(M, D):
    x = torch.randn(M, D, device="cuda") * 2 + 0.5
    g, b = torch.randn(D, device="cuda"), torch.randn(D, device="cuda")
    y, mean, rstd = ops.layernorm_fwd(x, g, b, False)
    xr, gr, br = x.double().requires_grad_(True), g.double().requires_grad_(True), b.double().requires_grad_(True)
    yr = torch.nn.functional.layer_norm(xr, (D,), gr, br, 1e-5)
    dy, dres = torch.randn(M, D, device="cuda"), torch.randn(M, D, device="cuda")
    yr.backward(dy.double())
    dx, dg, db = ops.layernorm_bwd(dy, x, mean, rstd, g, dres)
    assert relerr(y, yr.detach()) < 1e-6
    assert relerr(dx, xr.grad + dres.double()) < 1e-6
    assert relerr(dg, gr.grad) < 1e-5 and relerr(db, br.grad) < 1e-5
    yt, _, _ = ops.layernorm_fwd(x, g, b, True)
    assert torch.equal(yt, tf32_rn(y))
    # the same kernel can hand back the column sums of its output (the bias gradient of the Linear upstream)
    dx2, dg2, db2, dxs = ops.layernorm_bwd(dy, x, mean, rstd, g, dres, want_colsum=True)
    assert torch.equal(dx2, dx) and torch.equal(dg2, dg) and torch.equal(db2, db)
    assert relerr(dxs, dx.double().sum(0)) < 1e-5


def test_layout_and_reduction_kernels():
    img = torch.rand(3, 3, 64, 32, device="cuda")
    p = ops.patchify(img, 8, False)
    assert torch.equal(p.cpu(), O.patchify(img.cpu(), 8).reshape(p.shape))
    bias = torch.randn(3, device="cuda")
    assert torch.equal(ops.unpatchify(p, bias, 3, 3, 64, 32, 8), img + bias.view(1, 3, 1, 1))
    x = torch.randn(5000, 768, device="cuda")
    assert relerr(ops.colsum(x), x.double().sum(0)) < 1e-5
    v = torch.randn(4096, device="cuda")
    assert torch.equal(ops.round_tf32(v), tf32_rn(v))
    t = torch.randn(16, 64, device="cuda")
    assert torch.equal(ops.add_rows_mod(x[:64, :64].contiguous(), t), x[:64, :64] + t.repeat(4, 1))
    part = torch.randn(4, 96, 64, device="cuda")
    assert relerr(ops.splitk_reduce(part), part.double().sum(0)) < 1e-6


# ------------------------------------------------------------------------------------ attention
@pytest.mark.parametrize("B,N,heads,dh", [(2, 16, 2, 32), (1, 24, 3, 64), (2, 200, 2, 64), (2, 1024, 4, 64), (1, 130, 1, 32)])
def test_attention_fwd_bwd(B, N, heads, dh):
    inner = heads * dh
    qkv = tf32_rn(torch.randn(B * N, 3 * inner, device="cuda"))
    scale = dh ** -0.5
    o, lse = ops.attention_fwd(qkv, B, N, heads, dh, scale, False)
    q, k, v = (t.reshape(B, N, heads, dh).permute(0, 2, 1, 3).double() for t in qkv.split(inner, dim=-1))
    for t in (q, k, v):
        t.requires_grad_(True)
    s = (q @ k.transpose(-1, -2)) * scale
    oref = (torch.softmax(s, -1) @ v).permute(0, 2, 1, 3).reshape(B * N, inner)
    do = tf32_rn(torch.randn(B * N, inner, device="cuda"))
    oref.backward(do.double())
    dqkv = ops.attention_bwd(qkv, o, lse, do, B, N, heads, dh, scale, False)
    dref = torch.cat([t.grad.permute(0, 2, 1, 3).reshape(B * N, inner) for t in (q, k, v)], dim=-1)
    # P and dS re-enter the tensor cores rounded to tf32 (2^-11): tolerance 2e-3 of the tensor scale
    assert relerr(o, oref.detach()) < 2e-3
    assert relerr(lse, torch.logsumexp(s, -1).reshape(-1).detach()) < 1e-5
    assert relerr(dqkv, dref) < 3e-3


# ------------------------------------------------------------------------------------ quantiser
@pytest.mark.parametrize("tag,depth", [("plain", 1), ("res4", 4), ("res2", 2), ("clustered", 1)])
def test_vq_matches_reference_golden(golden_dir, tag, depth):
    g = np.load(os.path.join(golden_dir, "vq_cases.npz"))
    z, E = torch.from_numpy(g[f"{tag}.z"]).cuda(), torch.from_numpy(g[f"{tag}.E"]).cuda()
    out, loss, idx = ops.vq_fwd(z, E, depth, 0.25)
    np.testing.assert_array_equal(idx.cpu().numpy().reshape(g[f"{tag}.idx"].shape), g[f"{tag}.idx"])   # bit-exact codes
    np.testing.assert_allclose(out.cpu().numpy(), g[f"{tag}.zq"], rtol=0, atol=3e-7)
    np.testing.assert_allclose(loss.item(), float(g[f"{tag}.loss"]), rtol=1e-5)
    g_out = torch.from_numpy(g[f"{tag}.g_out"]).cuda() if f"{tag}.g_out" in g.files else torch.zeros_like(z)
    gl = float(g[f"{tag}.g_loss"]) if f"{tag}.g_loss" in g.files else 1.0
    gz, gE = ops.vq_bwd(z, E, idx, g_out, torch.tensor(gl, device="cuda"), depth > 1, 0.25)
    assert relerr(gz.cpu(), torch.from_numpy(g[f"{tag}.gz"])) < 1e-5
    assert relerr(gE.cpu(), torch.from_numpy(g[f"{tag}.gE"])) < 1e-5


def test_vq_indices_bit_exact_vs_oracle_with_near_tie_audit():
    M, K = 16384, 8192
    z, E = torch.randn(M, 32), torch.randn(K, 32)
    ref = O.vq_lookup_np(z.numpy(), E.numpy())
    _, _, idx = ops.vq_fwd(z.cuda(), E.cuda(), 1, 0.25)
    mism = np.nonzero(idx.cpu().numpy()[:, 0] != ref)[0]
    if len(mism):   # only fp32 near-ties may differ (SURVEY.md section 7): audit in float64
        assert len(mism) <= 2 and (O.vq_top2_gap_f64(z.numpy()[mism], E.numpy()) < 1e-6).all()


def test_vq_full_size_properties():
    """config-2 size (M = 128*1024 tokens, 8192 codes): size-independent properties"""
    M, K = 131072, 8192
    z, E = torch.randn(M, 32, device="cuda"), torch.randn(K, 32, device="cuda")
    out, loss, idx = ops.vq_fwd(z, E, 1, 0.25)
    assert idx.min() >= 0 and idx.max() < K and idx.dtype == torch.int64
    q = torch.nn.functional.normalize(E[idx[:, 0]], dim=-1)
    assert (out - q).abs().max() < 1e-6                                    # out == z + (q - z)
    zn = torch.nn.functional.normalize(z, dim=-1)
    np.testing.assert_allclose(loss.item(), 1.25 * ((q - zn) ** 2).mean().item(), rtol=1e-5)
    # the chosen code is at least as close as 64 random other codes (argmin property)
    rnd = torch.randint(0, K, (M, 64), device="cuda")
    en = torch.nn.functional.normalize(E, dim=-1)
    d_best = ((zn - en[idx[:, 0]]) ** 2).sum(-1)
    d_rnd = ((zn[:, None, :] - en[rnd]) ** 2).sum(-1).min(dim=1).values
    assert (d_best <= d_rnd + 1e-6).all()
    # idempotence: quantising the selected (normalised) codes returns the same codes
    _, _, idx2 = ops.vq_fwd(q.contiguous(), E, 1, 0.25)
    assert (idx2 == idx).float().mean().item() > 0.9999
    # residual mode: depth-0 codes equal the plain codes, residual norms shrink
    _, _, idx4 = ops.vq_fwd(z, E, 4, 0.25)
    assert torch.equal(idx4[:, 0], idx[:, 0])
    # embed (decode_codes) equals the straight-through value
    np.testing.assert_allclose(ops.vq_embed(E, idx, 1).cpu().numpy(), out.cpu().numpy(), atol=1e-6)


def test_vq_edge_cases():
    E = torch.randn(64, 32, device="cuda")
    z = torch.zeros(4, 32, device="cuda")                 # zero rows: F.normalize gives 0; every distance is |e_n|^2 ~ 1
    out, loss, idx = ops.vq_fwd(z, E, 1, 0.25)            # (a 8192-way fp32 near-tie: any code within 1 ulp is correct)
    en = torch.nn.functional.normalize(E, dim=-1)
    d = (en ** 2).sum(-1)
    assert torch.isfinite(loss) and (idx[:, 0] == idx[0, 0]).all() and d[idx[0, 0]] <= d.min() + 2.4e-7
    E2 = E.clone(); E2[5] = E2[3]                         # duplicate code: lowest index wins (torch.argmin)
    z = (E2[5] * 3.0).repeat(4, 1).contiguous()
    _, _, idx = ops.vq_fwd(z, E2, 1, 0.25)
    assert (idx == 3).all()
    with pytest.raises(RuntimeError):
        ops.vq_fwd(torch.randn(4, 16, device="cuda"), torch.randn(64, 16, device="cuda"), 1, 0.25)   # embed_dim != 32
