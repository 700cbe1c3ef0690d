"""GPU checks of the EMA codebook kernels (vq_fwd_ema statistics, vq_ema_update) and of EMAVectorQuantizer on them, against
the fp64 oracle of oracle/ema_oracle.py and against the existing lookup / backward kernels."""
import os
import socket
import sys

import numpy as np
import pytest
import torch

import enhancing_transformers_b200 as etb
from enhancing_transformers_b200 import functional as Fn
from oracle import ema_oracle as EO

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda", 0)
M_BIG, K_BIG, D = 131072, 8192, 32
# relative L2 error of s against fp64: fp32 sums of unit vectors.  Measured on an H100: 6.7e-8 - 7.3e-6 over the cases
# below, except one code at depth 4: 3.0e-5 in both summation modes alike -- there every token carries the same fp32
# rounding of its residual chain (z minus three unit codes), which no sum averages out; it is not the summation.
S_TOL = 1e-5
S_TOL_ONE_CODE_DEEP = 1e-4


def _z(kind, M, E, seed=0):
    g = torch.Generator().manual_seed(seed)
    if kind == "uniform":
        return torch.randn(M, D, generator=g)
    if kind == "clustered":          # bench.py's VQ block: 45 codes + 0.01 noise
        return E[torch.randint(0, 45, (M,), generator=g)] + 0.01 * torch.randn(M, D, generator=g)
    return E[7].expand(M, D).clone()  # one code


def _stats(buf, K):
    return buf[K * D:].cpu().numpy(), buf[:K * D].view(K, D).cpu().double().numpy()


def _rel(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


@pytest.mark.parametrize("deterministic", [False, True], ids=["atomic", "deterministic"])
@pytest.mark.parametrize("kind", ["uniform", "clustered", "one_code"])
@pytest.mark.parametrize("use_norm", [True, False], ids=["norm", "raw"])
@pytest.mark.parametrize("depth", [1, 4])
def test_statistics_against_fp64(depth, use_norm, kind, deterministic):
    E = torch.randn(K_BIG, D, generator=torch.Generator().manual_seed(1))
    z = _z(kind, M_BIG, E)
    zd, Ed = z.to(DEV), E.to(DEV)
    out, loss, idx, buf = etb.ops.vq_fwd_ema(zd, Ed, depth, 0.25, use_norm, True, deterministic)
    out0, loss0, idx0 = etb.ops.vq_fwd(zd, Ed, depth, 0.25, use_norm)
    assert torch.equal(idx, idx0) and torch.equal(out, out0)          # the same lookup, bit for bit
    idx_np = idx.cpu().numpy()
    n, s = _stats(buf, K_BIG)
    n_ref, s_ref = EO.statistics(z.numpy(), E.numpy(), idx_np, use_norm)
    np.testing.assert_array_equal(n, n_ref.astype(np.float32))
    err = _rel(s, s_ref)
    print(f"s rel-L2 {err:.2e}")
    assert err < (S_TOL_ONE_CODE_DEEP if kind == "one_code" and depth > 1 else S_TOL), err
    want = EO.loss(z.numpy(), E.numpy(), idx_np, 0.25, use_norm)
    assert abs(loss.item() - want) <= 1e-5 * abs(want) + 1e-12, (loss.item(), want)


@pytest.mark.parametrize("deterministic", [False, True], ids=["atomic", "deterministic"])
def test_ragged_token_count_and_eval_mode(deterministic):
    M = M_BIG - 4 * 17                                 # not a multiple of the 128-token tile
    E = torch.randn(K_BIG, D, generator=torch.Generator().manual_seed(2))
    z = _z("clustered", M, E, seed=3)
    out, loss, idx, buf = etb.ops.vq_fwd_ema(z.to(DEV), E.to(DEV), 2, 0.25, True, True, deterministic)
    n, s = _stats(buf, K_BIG)
    n_ref, s_ref = EO.statistics(z.numpy(), E.numpy(), idx.cpu().numpy())
    np.testing.assert_array_equal(n, n_ref.astype(np.float32))
    assert n.sum() == 2 * M and _rel(s, s_ref) < S_TOL
    out2, loss2, idx2, none = etb.ops.vq_fwd_ema(z.to(DEV), E.to(DEV), 2, 0.25, True, False, deterministic)
    assert none is None and torch.equal(idx2, idx) and torch.equal(out2, out) and torch.equal(loss2, loss)


def test_update_kernel_against_fp64():
    K = K_BIG
    g = torch.Generator().manual_seed(4)
    E = torch.randn(K, D, generator=g)
    z = _z("clustered", M_BIG, E, seed=5)
    _, _, idx, buf = etb.ops.vq_fwd_ema(z.to(DEV), E.to(DEV), 1, 0.25)
    cs = torch.rand(K, generator=g) * 20
    ea = torch.randn(K, D, generator=g)
    n, s = _stats(buf, K)
    cs_ref, ea_ref, w_ref = EO.update(cs.numpy(), ea.numpy(), n, s, 0.99, 1e-5)
    csd, ead, wd = cs.to(DEV), ea.to(DEV), torch.empty(K, D, device=DEV)
    etb.ops.vq_ema_update(buf, csd, ead, wd, 0.99, 1e-5)
    assert _rel(csd.cpu().double().numpy(), cs_ref) < 1e-6
    assert _rel(ead.cpu().double().numpy(), ea_ref) < 1e-6
    assert np.abs(wd.cpu().double().numpy() - w_ref).max() / np.abs(w_ref).max() < 1e-5


@pytest.mark.parametrize("residual", [False, True])
def test_module_outputs_and_backward_use_the_looked_up_codebook(residual):
    torch.manual_seed(0)
    q = etb.EMAVectorQuantizer(32, 1024, use_residual=residual, num_quantizers=4 if residual else None).to(DEV)
    g = torch.Generator().manual_seed(6)
    for step in range(3):
        z = torch.randn(16, 256, 32, generator=g).to(DEV).requires_grad_(True)
        E = q.embedding.weight.detach().clone()
        zq, loss, idx = q(z)
        out0, _, idx0 = etb.ops.vq_fwd(z.detach().view(-1, 32), E, q.depth, 0.25)
        assert torch.equal(idx.view(-1, q.depth), idx0) and torch.equal(zq.view(-1, 32), out0)
        assert not torch.equal(E, q.embedding.weight)                     # the update happened
        want = EO.loss(z.detach().view(-1, 32).cpu().numpy(), E.cpu().numpy(), idx0.cpu().numpy())
        assert abs(loss.item() - want) <= 1e-5 * want
        g_out = torch.randn(zq.shape, generator=g).to(DEV)
        g_loss = torch.full((), 2.0, device=DEV)
        torch.autograd.backward([zq, loss], [g_out, g_loss])
        if residual:
            assert torch.equal(z.grad, g_out)
        else:
            gz0, _ = etb.ops.vq_bwd(z.detach().view(-1, 32), E, idx0, g_out.view(-1, 32), g_loss, False, 0.25)
            assert torch.equal(z.grad.view(-1, 32), gz0)                  # today's gz, on the pre-update codebook
        assert q.embedding.weight.grad is None


def _train(steps, seed=0):
    torch.manual_seed(seed)
    q = etb.EMAVectorQuantizer(32, 2048, use_residual=True, num_quantizers=2, decay=0.9).to(DEV)
    pre = torch.nn.Linear(64, 32).to(DEV)
    opt = torch.optim.SGD(pre.parameters(), lr=0.1)
    g = torch.Generator().manual_seed(seed + 1)
    for _ in range(steps):
        x = torch.randn(64, 256, 64, generator=g).to(DEV)
        opt.zero_grad()
        zq, loss, _ = q(pre(x))
        ((zq ** 2).mean() + loss).backward()
        opt.step()
    torch.cuda.synchronize()
    return [t.detach().cpu().clone() for t in (q.embedding.weight, q.cluster_size, q.embed_avg)]


def test_deterministic_training_is_bit_reproducible(monkeypatch):
    monkeypatch.setattr(Fn, "DETERMINISTIC", True)
    a, b = _train(4), _train(4)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_multi_step_replay_through_vitvq_matches_the_oracle():
    """a tiny ViTVQ stand-in with patch(ema=True): after each step the codebook matches an fp64 replay fed the kernels' own z;
    the next step's codes are the fp32 lookup's on the kernels' own updated codebook"""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_abi_and_boundary import _stand_in_vitvqgan
    mod = _stand_in_vitvqgan()
    etb.patch(mod, ema=True)
    torch.manual_seed(0)
    model = mod.ViTVQ(image_size=64, patch_size=8, encoder=dict(dim=64, depth=1, heads=2, mlp_dim=128),
                      decoder=dict(dim=64, depth=1, heads=2, mlp_dim=128),
                      quantizer=dict(embed_dim=32, n_embed=512, decay=0.9, eps=1e-5),
                      loss=lambda qloss, x, xrec, i: ((xrec - x) ** 2).mean() + qloss).to(DEV)
    q = model.quantizer
    seen = []
    q.register_forward_hook(lambda m, inp, out: seen.append((inp[0].detach().reshape(-1, 32).clone(), out[2].detach().clone())))
    opt = torch.optim.Adam([p for p in model.parameters() if p.requires_grad], lr=1e-3)
    cs, ea = q.cluster_size.double().cpu().numpy(), q.embed_avg.double().cpu().numpy()
    g = torch.Generator().manual_seed(1)
    for step in range(5):
        E = q.embedding.weight.detach().clone()
        imgs = torch.rand(8, 3, 64, 64, generator=g).to(DEV)
        opt.zero_grad()
        model.training_step(imgs, step, 0).backward()
        opt.step()
        z, idx = seen[-1]
        _, _, idx_fp32 = etb.ops.vq_fwd(z, E, 1, 0.25)                 # the fp32 lookup on the codebook of this step
        assert torch.equal(idx.view(-1, 1), idx_fp32)
        n, s = EO.statistics(z.double().cpu().numpy(), E.cpu().numpy(), idx.view(-1, 1).cpu().numpy())
        cs, ea, w = EO.update(cs, ea, n, s, 0.9, 1e-5)
        got = q.embedding.weight.detach().double().cpu().numpy()
        assert np.abs(got - w).max() / np.abs(w).max() < 1e-5, step


def _nccl_worker(rank, world, port, out):
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    import enhancing_transformers_b200 as etb_
    dev = torch.device("cuda", rank)
    torch.manual_seed(0)
    q = etb_.EMAVectorQuantizer(32, 1024, decay=0.9).to(dev)
    g = torch.Generator().manual_seed(10 + rank)                     # each replica sees different tokens
    worst = 0.0
    for _ in range(3):
        q(torch.randn(8192, 32, generator=g).to(dev))
        book = torch.cat([q.embedding.weight.reshape(-1), q.cluster_size, q.embed_avg.reshape(-1)])
        other = [torch.empty_like(book) for _ in range(world)]
        dist.all_gather(other, book)
        worst = max(worst, (other[0] - other[1]).abs().max().item())
    if rank == 0:
        out.put(worst)
    dist.barrier()
    dist.destroy_process_group()


def test_nccl_replicas_stay_identical():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_nccl_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    worst = q.get(timeout=300)
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    assert worst == 0.0
