"""GPU checks of the opt-in bit-reproducible backward (run on an H100: pytest -m gpu): ops.vq_bwd_deterministic and
ops.token_embed_bwd_deterministic give the same bits on every call and under any SM limit, match fp64 references computed
from the same ids, and leave every other output bit-identical to the atomic path; whole modules give bit-identical
gradients run after run.  fp64 references are computed outside torch.use_deterministic_algorithms (under it torch's
own index and matmul backward may raise)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import enhancing_transformers_b200 as etb
from enhancing_transformers_b200 import functional as Fn

pytestmark = pytest.mark.gpu
ops = etb.ops


def relerr(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


@pytest.fixture(autouse=True)
def _need_cuda():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    torch.manual_seed(0)


def ref_vq_grads(z, E, idx, g_out, g_loss, residual, beta, use_norm):
    """(gz, gE) of out * g_out + loss * g_loss in fp64, with the codes fixed to idx (quantizers.py:38-63,85-92)"""
    z = z.double().requires_grad_(True)
    E = E.double().requires_grad_(True)
    nrm = (lambda x: F.normalize(x, dim=-1, eps=1e-12)) if use_norm else (lambda x: x)
    if not residual:
        zn, qn = nrm(z), nrm(E[idx[:, 0]])
        loss = beta * ((qn.detach() - zn) ** 2).mean() + ((qn - zn.detach()) ** 2).mean()
        zq = qn
    else:
        r, zq, losses = z.detach().clone(), 0, []
        for t in range(idx.shape[1]):
            rn, qn = nrm(r), nrm(E[idx[:, t]])
            losses.append(beta * ((qn.detach() - rn) ** 2).mean() + ((qn - rn.detach()) ** 2).mean())
            r = r - qn
            zq = zq + qn
        loss = torch.stack(losses).mean()
    out = z + (zq - z).detach()
    total = (out * g_out.double()).sum() + loss * g_loss.double()
    return torch.autograd.grad(total, (z, E))


# ------------------------------------------------------------------------------------------------ VQ
@pytest.mark.parametrize("tag,depth", [("plain", 1), ("res2", 2), ("res4", 4), ("clustered", 1)])
def test_vq_deterministic_matches_golden_and_keeps_gz(golden_dir, tag, depth):
    g = np.load(os.path.join(golden_dir, "vq_cases.npz"))
    z, E = torch.from_numpy(g[f"{tag}.z"]).cuda(), torch.from_numpy(g[f"{tag}.E"]).cuda()
    _, _, idx = ops.vq_fwd(z, E, depth, 0.25)
    g_out = torch.from_numpy(g[f"{tag}.g_out"]).cuda() if f"{tag}.g_out" in g.files else torch.zeros_like(z)
    gl = torch.tensor(float(g[f"{tag}.g_loss"]) if f"{tag}.g_loss" in g.files else 1.0, device="cuda")
    gz, gE = ops.vq_bwd_deterministic(z, E, idx, g_out, gl, depth > 1, 0.25)
    assert relerr(gE.cpu(), torch.from_numpy(g[f"{tag}.gE"])) < 1e-5
    gz_atomic, _ = ops.vq_bwd(z, E, idx, g_out, gl, depth > 1, 0.25)
    assert torch.equal(gz, gz_atomic)


def _z(kind, E, M, gen):
    if kind == "uniform":
        return torch.randn(M, E.shape[1], device="cuda", generator=gen)
    rows = torch.randint(0, 45, (M,), device="cuda", generator=gen) if kind == "clustered" else torch.zeros(M, dtype=torch.int64, device="cuda")
    return (E[rows] + 0.01 * torch.randn(M, E.shape[1], device="cuda", generator=gen)).contiguous()


@pytest.mark.parametrize("use_norm", [True, False])
@pytest.mark.parametrize("kind", ["uniform", "clustered", "one_code"])
@pytest.mark.parametrize("depth", [1, 4])
def test_vq_deterministic_base_shape(depth, kind, use_norm):
    M, K, D = 131072, 8192, 32
    gen = torch.Generator(device="cuda").manual_seed(1)
    E = torch.randn(K, D, device="cuda", generator=gen)
    z = _z(kind, E, M, gen)
    _, _, idx = ops.vq_fwd(z, E, depth, 0.25, use_norm)
    if kind == "one_code":
        assert bool((idx[:, 0] == 0).all())
    g_out = torch.randn(M, D, device="cuda", generator=gen)
    g_loss = torch.tensor(1.0, device="cuda")
    args = (z, E, idx, g_out, g_loss, depth > 1, 0.25, use_norm)
    gz1, gE1 = ops.vq_bwd_deterministic(*args)
    gz2, gE2 = ops.vq_bwd_deterministic(*args)
    assert torch.equal(gz1, gz2) and torch.equal(gE1, gE2)
    ops.set_sm_limit(8)
    try:
        gz3, gE3 = ops.vq_bwd_deterministic(*args)
    finally:
        ops.set_sm_limit(0)
    assert torch.equal(gz1, gz3) and torch.equal(gE1, gE3)
    gz_a, gE_a = ops.vq_bwd(*args)
    assert torch.equal(gz1, gz_a)
    gz_ref, gE_ref = ref_vq_grads(*args)
    # Against fp64 the error is set by the fp32 per-token contributions both paths share, not by the reduction: with z a
    # code plus 0.01 noise every contribution J^T(q - z) carries the same rounding of the normalised code, and those
    # add up coherently over the code's thousands of tokens (1e-4 to 1e-3 with use_norm on).  So: no further from fp64
    # than the atomic path, and within 1e-5 of it.  (The reduction alone is checked against fp64 at 1e-5 in
    # test_token_embed_deterministic, whose rows are exact inputs.)
    err, err_atomic = relerr(gE1, gE_ref), relerr(gE_a, gE_ref)
    assert err <= max(1e-5, 1.1 * err_atomic), (err, err_atomic)
    assert relerr(gE1, gE_a) <= 1e-5
    assert relerr(gz1, gz_ref) <= 1e-5


def test_vq_deterministic_equals_atomic_when_every_code_is_hit_at_most_once():
    M, K, D = 4096, 8192, 32
    gen = torch.Generator(device="cuda").manual_seed(2)
    E = torch.randn(K, D, device="cuda", generator=gen)
    perm = torch.randperm(K, device="cuda", generator=gen)[:M]
    z = (E[perm] + 1e-3 * torch.randn(M, D, device="cuda", generator=gen)).contiguous()
    _, _, idx = ops.vq_fwd(z, E, 1, 0.25)
    assert idx.unique().numel() == M
    args = (z, E, idx, torch.randn(M, D, device="cuda", generator=gen), torch.tensor(0.5, device="cuda"), False, 0.25)
    gz, gE = ops.vq_bwd_deterministic(*args)
    gz_a, gE_a = ops.vq_bwd(*args)
    assert torch.equal(gz, gz_a) and torch.equal(gE, gE_a)


def test_vector_quantizer_under_the_torch_flag_is_reproducible():
    """the module switch: under torch.use_deterministic_algorithms the codebook gradient is the deterministic op's"""
    vq = etb.VectorQuantizer(embed_dim=32, n_embed=512, use_residual=True, num_quantizers=4).cuda()
    z = torch.randn(8, 1024, 32, device="cuda")
    grads = []
    for _ in range(2):
        vq.zero_grad(set_to_none=True)
        zz = z.clone().requires_grad_(True)
        torch.use_deterministic_algorithms(True)
        try:
            zq, loss, idx = vq(zz)
            (zq.sum() + loss).backward()
        finally:
            torch.use_deterministic_algorithms(False)
        grads.append(vq.embedding.weight.grad.clone())
    assert torch.equal(grads[0], grads[1])
    _, want = ops.vq_bwd_deterministic(z.view(-1, 32), vq.embedding.weight.detach(), idx.view(-1, 4), torch.ones(8 * 1024, 32, device="cuda"),
                                       torch.tensor(1.0, device="cuda"), True, 0.25)
    assert torch.equal(grads[0], want)


# ------------------------------------------------------------------------------------------ stage 2
@pytest.mark.parametrize("ids", ["random", "equal"])
def test_token_embed_deterministic(ids):
    B, Tc, Ti, C, Vc, Vi = 4, 1, 1024, 1024, 1000, 8192
    gen = torch.Generator(device="cuda").manual_seed(3)
    if ids == "random":
        conds = torch.randint(0, Vc, (B, Tc), device="cuda", generator=gen)
        codes = torch.randint(0, Vi, (B, Ti), device="cuda", generator=gen)
        codes[0, :3] = torch.tensor([-5, Vi, Vi + 7])            # clamped into the table, as the forward gathers them
    else:
        conds = torch.full((B, Tc), 7, dtype=torch.int64, device="cuda")
        codes = torch.full((B, Ti), 11, dtype=torch.int64, device="cuda")
    g = torch.randn(B * (Tc + Ti), C, device="cuda", generator=gen)
    out1 = ops.token_embed_bwd_deterministic(conds, codes, g, Vc, Vi)
    out2 = ops.token_embed_bwd_deterministic(conds, codes, g, Vc, Vi)
    assert all(torch.equal(a, b) for a, b in zip(out1, out2))
    ops.set_sm_limit(8)
    try:
        out3 = ops.token_embed_bwd_deterministic(conds, codes, g, Vc, Vi)
    finally:
        ops.set_sm_limit(0)
    assert all(torch.equal(a, b) for a, b in zip(out1, out3))
    gWc, gpc, gWi, gpi = out1
    _, gpc_a, _, gpi_a = ops.token_embed_bwd(conds, codes, g, Vc, Vi)
    assert torch.equal(gpc, gpc_a) and torch.equal(gpi, gpi_a)
    g3 = g.double().view(B, Tc + Ti, C)
    ref_c = torch.zeros(Vc, C, dtype=torch.float64, device="cuda").index_add_(0, conds.clamp(0, Vc - 1).reshape(-1), g3[:, :Tc].reshape(-1, C))
    ref_i = torch.zeros(Vi, C, dtype=torch.float64, device="cuda").index_add_(0, codes.clamp(0, Vi - 1).reshape(-1), g3[:, Tc:].reshape(-1, C))
    assert relerr(gWc, ref_c) <= 1e-5 and relerr(gWi, ref_i) <= 1e-5
    assert relerr(gpc, g3[:, :Tc].sum(0)) <= 1e-5 and relerr(gpi, g3[:, Tc:].sum(0)) <= 1e-5


# ---------------------------------------------------------------------------------------------- modules
def _grads_twice(build, step, monkeypatch):
    """every .grad of two forward + backward runs with the deterministic switch on"""
    monkeypatch.setattr(Fn, "DETERMINISTIC", True)
    torch.manual_seed(0)
    model = build()
    runs = []
    for _ in range(2):
        model.zero_grad(set_to_none=True)
        step(model).backward()
        runs.append({n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None})
    return runs


def test_vitvq_stack_gradients_are_bit_identical(monkeypatch):
    class Stack(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.encoder = etb.ViTEncoder(32, 8, dim=64, depth=1, heads=2, mlp_dim=128, dim_head=32)
            self.pre_quant = etb.QuantLinear(64, 32)
            self.quantizer = etb.VectorQuantizer(embed_dim=32, n_embed=128, use_residual=True, num_quantizers=4)
            self.post_quant = etb.QuantLinear(32, 64)
            self.decoder = etb.ViTDecoder(32, 8, dim=64, depth=1, heads=2, mlp_dim=128, dim_head=32)

        def forward(self, x):
            q, qloss, _ = self.quantizer(self.pre_quant(self.encoder(x)))
            return self.decoder(self.post_quant(q)), qloss

    x = torch.rand(16, 3, 32, 32, device="cuda")
    w = torch.randn(16, 3, 32, 32, device="cuda")

    def step(m):
        rec, qloss = m(x)
        return (rec * w).sum() + qloss
    runs = _grads_twice(lambda: Stack().cuda(), step, monkeypatch)
    assert "quantizer.embedding.weight" in runs[0] and runs[0].keys() == runs[1].keys()
    for n in runs[0]:
        assert torch.equal(runs[0][n], runs[1][n]), n


def test_gpt_gradients_are_bit_identical(monkeypatch):
    B = 8
    codes = torch.randint(0, 64, (B, 16), device="cuda")
    conds = torch.randint(0, 10, (B, 1), device="cuda")

    def step(m):
        logits = m(codes, conds)
        return (logits * torch.linspace(-1, 1, logits.numel(), device="cuda").view_as(logits)).sum()
    runs = _grads_twice(lambda: etb.GPT(vocab_cond_size=10, vocab_img_size=64, embed_dim=64, cond_num_tokens=1, img_num_tokens=16,
                                        n_heads=2, n_layers=2).cuda(), step, monkeypatch)
    assert runs[0].keys() == runs[1].keys() and len(runs[0]) > 10
    for n in runs[0]:
        assert torch.equal(runs[0][n], runs[1][n]), n
