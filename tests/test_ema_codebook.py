"""CPU checks of the EMA codebook (EMAVectorQuantizer): the fp64 oracle against a hand-worked case, the module surface,
patch(ema=True), and the host logic -- statistics, all-reduce, update, backward -- with the two new entry points replaced
by torch stand-ins written from include/b200vq.h (the kernels themselves are checked on the GPU, test_gpu_ema_codebook.py)."""
import inspect
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

import enhancing_transformers_b200 as etb
from oracle import ema_oracle as EO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- stand-ins for ops.vq_fwd_ema / ops.vq_ema_update (contract: include/b200vq.h) ---------------------------------------
def emu_vq_fwd_ema(z, E, depth, beta, use_norm=True, stats=True, deterministic=False):
    K, D = E.shape
    nrm = (lambda x: F.normalize(x, dim=-1)) if use_norm else (lambda x: x)
    en = nrm(E)
    r, acc = z.detach().clone(), torch.zeros_like(z)
    idxs, xs, losses = [], [], []
    for _ in range(depth):
        x = nrm(r)
        d = (x * x).sum(1, keepdim=True) + (en * en).sum(1) - 2 * x @ en.t()
        i = d.argmin(1)
        q = en[i]
        losses.append(beta * ((q - x) ** 2).mean())
        idxs.append(i)
        xs.append(x)
        r, acc = r - q, acc + q
    out = z.detach() + (acc - z.detach())
    idx = torch.stack(idxs, 1)
    buf = None
    if stats:
        buf = torch.zeros(K * (D + 1))
        buf[:K * D].view(K, D).index_add_(0, idx.reshape(-1), torch.stack(xs, 1).reshape(-1, D))
        buf[K * D:] = torch.bincount(idx.reshape(-1), minlength=K).float()
    return out, torch.stack(losses).mean(), idx, buf


def emu_vq_ema_update(stats, cluster_size, embed_avg, weight, decay, eps):
    K, D = weight.shape
    cluster_size.mul_(decay).add_(stats[K * D:], alpha=1 - decay)
    embed_avg.mul_(decay).add_(stats[:K * D].view(K, D), alpha=1 - decay)
    N = cluster_size.sum()
    weight.copy_(embed_avg / ((cluster_size + eps) / (N + K * eps) * N)[:, None])


class _Patcher:
    """monkeypatch's two methods, for spawned workers"""

    @staticmethod
    def setattr(obj, name, value):
        setattr(obj, name, value)

    @staticmethod
    def setitem(mapping, key, value):
        mapping[key] = value


def _install(mp_):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import emulated_ops
    emulated_ops.install(mp_)
    mp_.setattr(etb.ops, "vq_fwd_ema", emu_vq_fwd_ema)
    mp_.setattr(etb.ops, "vq_ema_update", emu_vq_ema_update)


# ---- oracle -------------------------------------------------------------------------------------------------------------
def test_oracle_against_a_hand_worked_case():
    """3 codes, 5 tokens, D 2, use_norm off, decay 0.5: every number below is worked out by hand"""
    E = np.array([[1.0, 0.5], [0.0, 1.0], [1.5, 1.5]])
    z = np.array([[1.0, 0.0], [0.0, 1.0], [1.0, 1.0], [2.0, 2.0], [1.5, 2.0]])
    idx = EO.lookup(z, E, 1, use_norm=False)
    np.testing.assert_array_equal(idx[:, 0], [0, 1, 0, 2, 2])
    n, s = EO.statistics(z, E, idx, use_norm=False)
    np.testing.assert_array_equal(n, [2, 1, 2])
    np.testing.assert_array_equal(s, [[2.0, 1.0], [0.0, 1.0], [3.5, 4.0]])
    # squared distances to the chosen codes: 0.25, 0, 0.25, 0.5, 0.25 -> mean over 10 elements 0.125
    assert EO.loss(z, E, idx, beta=0.25, use_norm=False) == pytest.approx(0.25 * 0.125, abs=1e-15)
    cs, ea, w = EO.update(np.array([1.0, 1.0, 0.0]), E, n, s, decay=0.5, eps=0.0)
    np.testing.assert_allclose(cs, [1.5, 1.0, 1.0], atol=1e-15)
    np.testing.assert_allclose(ea, [[1.5, 0.75], [0.0, 1.0], [2.5, 2.75]], atol=1e-15)
    np.testing.assert_allclose(w, [[1.0, 0.5], [0.0, 1.0], [2.5, 2.75]], atol=1e-15)    # eps 0: weight = ea / cs
    _, _, w = EO.update(np.array([1.0, 1.0, 0.0]), E, n, s, decay=0.5, eps=0.1)
    smoothed = np.array([1.6, 1.1, 1.1]) / 3.8 * 3.5                                    # (cs + eps) / (N + K eps) * N, N 3.5
    np.testing.assert_allclose(w, [[1.5 / smoothed[0], 0.75 / smoothed[0]], [0.0, 1.0 / smoothed[1]],
                                   [2.5 / smoothed[2], 2.75 / smoothed[2]]], rtol=1e-14)
    n2, s2 = EO.allreduce([EO.statistics(z[:2], E, idx[:2], False), EO.statistics(z[2:], E, idx[2:], False)])
    np.testing.assert_array_equal(n2, n)
    np.testing.assert_allclose(s2, s)
    g = EO.grad_z(z, E, idx, np.ones_like(z), 1.0, beta=0.25, use_norm=False)
    np.testing.assert_allclose(g, 1 + 0.25 * 2 / 10 * (z - E[idx[:, 0]]))


# ---- module surface -----------------------------------------------------------------------------------------------------
def test_constructor_keywords_and_defaults():
    sig = inspect.signature(etb.EMAVectorQuantizer.__init__)
    assert list(sig.parameters) == ["self", "embed_dim", "n_embed", "beta", "use_norm", "use_residual", "num_quantizers", "decay",
                                    "eps", "kwargs"]
    assert sig.parameters["decay"].default == 0.99 and sig.parameters["eps"].default == 1e-5
    q = etb.EMAVectorQuantizer(32, 64, beta=0.5, use_residual=True, num_quantizers=3, decay=0.9, eps=1e-3, unused=1)
    assert (q.beta, q.depth, q.decay, q.eps, q.process_group) == (0.5, 3, 0.9, 1e-3, None)
    assert isinstance(q, etb.VectorQuantizer)
    with pytest.raises(ValueError):
        etb.EMAVectorQuantizer(32, 64, use_residual=True)


def test_same_init_and_rng_stream_as_vector_quantizer():
    torch.manual_seed(0)
    a = etb.VectorQuantizer(32, 128)
    after_a = torch.rand(4)
    torch.manual_seed(0)
    b = etb.EMAVectorQuantizer(32, 128)
    after_b = torch.rand(4)
    assert torch.equal(a.embedding.weight, b.embedding.weight) and torch.equal(after_a, after_b)
    assert torch.equal(b.embed_avg, b.embedding.weight) and torch.equal(b.cluster_size, torch.zeros(128))
    assert b.embed_avg.data_ptr() != b.embedding.weight.data_ptr()


def test_state_dict_keys_and_frozen_codebook():
    a, b = etb.VectorQuantizer(32, 64), etb.EMAVectorQuantizer(32, 64)
    assert set(b.state_dict()) == set(a.state_dict()) | {"cluster_size", "embed_avg"}
    assert b.embedding.weight.requires_grad is False
    assert [n for n, p in b.named_parameters() if p.requires_grad] == []
    fg = etb.FlatGradients(b.parameters())
    assert fg.params == []


def test_missing_buffers_are_reseeded_from_the_loaded_weight():
    torch.manual_seed(1)
    grad_trained = etb.VectorQuantizer(32, 64)
    ema = etb.EMAVectorQuantizer(32, 64)
    ema.cluster_size.fill_(3.0)
    res = ema.load_state_dict(grad_trained.state_dict(), strict=False)      # init_from_ckpt's strict=False (vitvqgan.py:58)
    assert set(res.missing_keys) == {"cluster_size", "embed_avg"} and not res.unexpected_keys
    assert torch.equal(ema.embedding.weight, grad_trained.embedding.weight)
    assert torch.equal(ema.embed_avg, grad_trained.embedding.weight) and torch.equal(ema.cluster_size, torch.zeros(64))
    # a full EMA state dict keeps its buffers; nested under a prefix as well
    full = {k: v.clone() for k, v in ema.state_dict().items()}
    full["cluster_size"].fill_(2.0)
    full["embed_avg"].fill_(0.5)
    fresh = etb.EMAVectorQuantizer(32, 64)
    fresh.load_state_dict(full, strict=True)
    assert torch.equal(fresh.cluster_size, full["cluster_size"]) and torch.equal(fresh.embed_avg, full["embed_avg"])
    holder = torch.nn.ModuleDict({"quantizer": etb.EMAVectorQuantizer(32, 64)})
    holder.load_state_dict({"quantizer." + k: v for k, v in grad_trained.state_dict().items()}, strict=False)
    assert torch.equal(holder["quantizer"].embed_avg, grad_trained.embedding.weight)


def test_cpu_tensors_are_rejected_loudly():
    q = etb.EMAVectorQuantizer(32, 64)
    for training in (True, False):
        q.train(training)
        with pytest.raises(RuntimeError, match="no CPU path"):
            q(torch.randn(1, 4, 32))
    assert torch.equal(q.embed_avg, q.embedding.weight)        # nothing was updated


def test_patch_ema_binds_the_class_and_yaml_keywords_reach_it():
    from test_abi_and_boundary import _stand_in_vitvqgan
    mod = _stand_in_vitvqgan()
    kw = dict(image_size=32, patch_size=8, encoder=dict(dim=64, depth=1, heads=2, mlp_dim=64),
              decoder=dict(dim=64, depth=1, heads=2, mlp_dim=64), quantizer=dict(embed_dim=32, n_embed=128, decay=0.95, eps=1e-4))
    etb.patch(mod, ema=True)
    assert mod.VectorQuantizer is etb.EMAVectorQuantizer
    model = mod.ViTVQ(**kw)
    assert isinstance(model.quantizer, etb.EMAVectorQuantizer)
    assert (model.quantizer.decay, model.quantizer.eps) == (0.95, 1e-4)
    etb.patch(mod)
    assert mod.VectorQuantizer is etb.VectorQuantizer


# ---- host logic with stand-in kernels -----------------------------------------------------------------------------------
@pytest.mark.parametrize("residual", [False, True])
def test_training_steps_match_the_oracle_and_backward_sees_the_looked_up_codebook(monkeypatch, residual):
    _install(monkeypatch)
    torch.manual_seed(0)
    q = etb.EMAVectorQuantizer(32, 48, use_residual=residual, num_quantizers=3 if residual else None, decay=0.8, eps=1e-5)
    cs, ea = q.cluster_size.double().numpy().copy(), q.embed_avg.double().numpy().copy()
    g = torch.Generator().manual_seed(2)
    for step in range(4):
        z = torch.randn(2, 8, 32, generator=g).requires_grad_(True)
        E_before = q.embedding.weight.detach().clone()
        zq, loss, idx = q(z)
        # codes and loss are those of the codebook in effect at this forward
        idx2 = idx.reshape(-1, q.depth).numpy()
        np.testing.assert_array_equal(idx2, EO.lookup(z.detach().reshape(-1, 32).numpy(), E_before.numpy(), q.depth))
        assert loss.item() == pytest.approx(EO.loss(z.detach().reshape(-1, 32).numpy(), E_before.numpy(), idx2, 0.25), rel=1e-5)
        n, s = EO.statistics(z.detach().reshape(-1, 32).numpy(), E_before.numpy(), idx2)
        cs, ea, w = EO.update(cs, ea, n, s, 0.8, 1e-5)
        np.testing.assert_allclose(q.embedding.weight.numpy(), w, rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(q.cluster_size.numpy(), cs, rtol=1e-6)
        g_out = torch.randn(zq.shape, generator=g)
        (zq * g_out).sum().add(loss * 3.0).backward()
        want = EO.grad_z(z.detach().reshape(-1, 32).numpy(), E_before.numpy(), idx2, g_out.reshape(-1, 32).numpy(), 3.0,
                         residual=residual)
        np.testing.assert_allclose(z.grad.reshape(-1, 32).numpy(), want, rtol=1e-4, atol=1e-6)
        assert q.embedding.weight.grad is None
    # eval: same lookup, no statistics, no update
    q.eval()
    before = [t.clone() for t in (q.embedding.weight, q.cluster_size, q.embed_avg)]
    z = torch.randn(2, 8, 32, generator=g)
    _, _, idx = q(z)
    np.testing.assert_array_equal(idx.reshape(-1, q.depth).numpy(), EO.lookup(z.reshape(-1, 32).numpy(), before[0].numpy(), q.depth))
    assert all(torch.equal(a, b) for a, b in zip(before, (q.embedding.weight, q.cluster_size, q.embed_avg)))
    q.train()
    with torch.no_grad():                                   # grad mode does not decide: training mode does
        q(z)
    assert not torch.equal(before[0], q.embedding.weight)


def test_adamw_skips_the_frozen_codebook(monkeypatch):
    """the reference's configure_optimizers (vitvqgan.py:152-160) hands every parameter, the frozen codebook included, to
    AdamW: with no .grad it is left alone, weight decay included"""
    _install(monkeypatch)
    torch.manual_seed(0)
    pre, q = torch.nn.Linear(16, 32), etb.EMAVectorQuantizer(32, 24)
    opt = torch.optim.AdamW(list(pre.parameters()) + list(q.parameters()), lr=1e-2, weight_decay=0.5)
    zq, loss, _ = q(pre(torch.randn(3, 4, 16)))
    ((zq ** 2).mean() + loss).backward()
    w = q.embedding.weight.detach().clone()
    opt.step()
    assert torch.equal(q.embedding.weight, w) and q.embedding.weight.grad is None


def test_detach_discriminator_forward_updates_like_the_grad_enabled_forward(monkeypatch):
    """the ViTVQ training step runs the autoencoder twice (optimizer_idx 0 and 1); with detach_discriminator_forward the
    second runs under no_grad and must update the codebook exactly as the grad-enabled forward does"""
    _install(monkeypatch)
    from test_abi_and_boundary import _stand_in_vitvqgan
    kw = dict(image_size=32, patch_size=8, encoder=dict(dim=64, depth=1, heads=2, mlp_dim=64, dim_head=32),
              decoder=dict(dim=64, depth=1, heads=2, mlp_dim=64, dim_head=32), quantizer=dict(embed_dim=32, n_embed=64, decay=0.9))
    prev = etb.set_precision("parity")
    try:
        books = []
        for detach in (False, True):
            mod = _stand_in_vitvqgan()
            etb.patch(mod, ema=True)
            cls = type("ViTVQ", (mod.ViTVQ,), {})
            if detach:
                etb.detach_discriminator_forward(cls)
            torch.manual_seed(0)
            model = cls(**kw, loss=lambda qloss, x, xrec, i: ((xrec - x) ** 2).mean() + qloss)
            imgs = torch.rand(2, 3, 32, 32, generator=torch.Generator().manual_seed(3))
            for step in range(2):
                model.training_step(imgs, step, 0).backward()
                model.training_step(imgs, step, 1)
            books.append([t.clone() for t in (model.quantizer.embedding.weight, model.quantizer.cluster_size,
                                              model.quantizer.embed_avg)])
    finally:
        etb.set_precision(prev)
    assert all(torch.equal(a, b) for a, b in zip(*books))
    assert books[0][1].sum().item() == pytest.approx((1 - 0.9 ** 4) * 2 * 16)   # four updates of 2 images x 16 tokens


# ---- world size 2 over gloo ---------------------------------------------------------------------------------------------
class _Net(torch.nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(0)
        self.pre = torch.nn.Linear(16, 32)
        self.q = etb.EMAVectorQuantizer(32, 24, use_residual=True, num_quantizers=2, decay=0.8)

    def forward(self, x):
        zq, qloss, _ = self.q(self.pre(x))
        return (zq ** 2).mean() + qloss


def _gloo_worker(rank, world, port, out, kind):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    _install(_Patcher)
    solo = dist.new_group([0])
    full = torch.randn(3, 8, 4, 16, generator=torch.Generator().manual_seed(1))       # 3 steps x 8 images
    net = _Net()
    ddp = torch.nn.parallel.DistributedDataParallel(net) if kind == "ddp" else None
    fg = etb.FlatGradients(net.parameters()) if kind == "flat" else None
    opt = torch.optim.SGD(net.pre.parameters(), lr=0.5)
    single = _Net() if rank == 0 else None
    if single is not None:
        single.q.process_group = solo                           # a group of one: no all-reduce
        opt1 = torch.optim.SGD(single.pre.parameters(), lr=0.5)
    worst_cross, worst_single = 0.0, 0.0
    for step in range(3):
        shard = full[step, rank * 4:(rank + 1) * 4]
        if fg is not None:
            fg.zero_()
            net(shard).backward()
            fg.allreduce()
        else:
            opt.zero_grad()
            ddp(shard).backward()
        opt.step()
        book = torch.cat([net.q.embedding.weight.reshape(-1), net.q.cluster_size, net.q.embed_avg.reshape(-1)])
        gathered = [torch.empty_like(book) for _ in range(world)]
        dist.all_gather(gathered, book)
        worst_cross = max(worst_cross, (gathered[0] - gathered[1]).abs().max().item())
        if single is not None:
            opt1.zero_grad()
            single(full[step]).backward()
            opt1.step()
            ref = torch.cat([single.q.embedding.weight.reshape(-1), single.q.cluster_size, single.q.embed_avg.reshape(-1)])
            worst_single = max(worst_single, ((book - ref).abs().max() / ref.abs().max()).item())
    if rank == 0:
        out.put((worst_cross, worst_single, len(fg.params) if fg is not None else -1))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("kind", ["flat", "ddp"])
def test_replicas_apply_the_same_update_as_one_process(kind):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q, kind)) for r in range(2)]
    for p in procs:
        p.start()
    worst_cross, worst_single, nparams = q.get(timeout=240)
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    assert worst_cross == 0.0                         # the same all-reduced statistics, the same update: the same bits
    assert worst_single < 1e-5, worst_single          # the concatenated batch in one process, up to fp32 reordering
    if kind == "flat":
        assert nparams == 2                           # pre.weight, pre.bias: the frozen codebook has no gradient slot


def test_c_abi_rejects_bad_arguments_before_touching_the_device():
    lib = etb._lib.lib()

    def err():
        return lib.b200vq_last_error().decode()
    ws = lib.b200vq_vq_fwd_ema_workspace_bytes(128, 256, 32, 1, 0)
    assert ws > lib.b200vq_vq_workspace_bytes(128, 256, 1)
    assert lib.b200vq_vq_fwd_ema_workspace_bytes(128, 256, 32, 2, 1) > lib.b200vq_vq_fwd_ema_workspace_bytes(128, 256, 32, 2, 0)
    assert lib.b200vq_vq_fwd_ema_workspace_bytes(128, 256, 16, 1, 0) == 0
    p = 256                                                            # never dereferenced: validation comes first
    assert lib.b200vq_vq_fwd_ema(p, p, p, p, p, None, None, 128, 256, 16, 1, 0.25, 1, 0, p, ws, None) < 0 and "embed_dim" in err()
    assert lib.b200vq_vq_fwd_ema(p, p, p, p, p, None, None, 128, 256, 32, 9, 0.25, 1, 0, p, ws, None) < 0 and "num_quantizers" in err()
    assert lib.b200vq_vq_fwd_ema(p, p, p, p, p, p, None, 128, 256, 32, 1, 0.25, 1, 0, p, ws, None) < 0 and "both" in err()
    assert lib.b200vq_vq_fwd_ema(None, p, p, p, p, p, p, 128, 256, 32, 1, 0.25, 1, 0, p, ws, None) < 0 and "null" in err()
    assert lib.b200vq_vq_fwd_ema(p, p, p, p, p, p, p, 128, 256, 32, 1, 0.25, 1, 0, p, ws - 1, None) < 0 and "workspace" in err()
    assert lib.b200vq_vq_fwd_ema(p, p, p, p, p, p, p, 1 << 22, 256, 32, 4, 0.25, 1, 0, p, 1 << 40, None) < 0 and "2^24" in err()
    assert lib.b200vq_vq_ema_update(p, p, p, p, p, 256, 16, 0.99, 1e-5, None) < 0 and "embed_dim" in err()
    assert lib.b200vq_vq_ema_update(p, p, p, p, p, 256, 32, 1.5, 1e-5, None) < 0 and "decay" in err()
    assert lib.b200vq_vq_ema_update(p, p, p, p, p, 256, 32, 0.99, -1.0, None) < 0 and "eps" in err()
    assert lib.b200vq_vq_ema_update(p, None, p, p, p, 256, 32, 0.99, 1e-5, None) < 0 and "null" in err()
