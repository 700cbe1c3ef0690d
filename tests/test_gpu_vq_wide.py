"""GPU checks of the quantiser at code widths above 32 (embed_dim 64 .. 256): the lookup, both backwards, vq_embed and the
EMA statistics against the reference's outputs (tests/golden/vq_wide.npz), the numpy / fp64 oracles at full size, and
the modules end to end against the fp64 oracle."""
import copy
import os

import numpy as np
import pytest
import torch

import enhancing_transformers_b200 as etb
from oracle import ema_oracle as EO
from oracle import vitvq_oracle as O
from oracle.gen_golden_vq_wide import CASES

pytestmark = pytest.mark.gpu
ops = etb.ops
DEV = torch.device("cuda", 0)
TAGS = [(tag, kw) for tag, _, kw in CASES] + [("d256.clustered", {})]


def _rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


@pytest.fixture(autouse=True)
def _restore():
    prev = etb.get_precision()
    yield
    etb.set_precision(prev)


@pytest.mark.parametrize("tag,kw", TAGS, ids=[t for t, _ in TAGS])
def test_matches_reference_golden(golden_dir, tag, kw):
    g = O.load_golden(os.path.join(golden_dir, "vq_wide.npz"))
    depth = kw.get("num_quantizers", 1)
    use_norm = kw.get("use_norm", True)
    z, E = torch.from_numpy(g[f"{tag}.z"]).to(DEV), torch.from_numpy(g[f"{tag}.E"]).to(DEV)
    D = E.shape[1]
    out, loss, idx = ops.vq_fwd(z, E, depth, 0.25, use_norm)
    np.testing.assert_array_equal(idx.cpu().numpy().reshape(g[f"{tag}.idx"].shape), g[f"{tag}.idx"])   # bit-exact codes
    np.testing.assert_allclose(out.cpu().numpy(), g[f"{tag}.zq"], rtol=0, atol=3e-7)
    np.testing.assert_allclose(loss.item(), float(g[f"{tag}.loss"]), rtol=1e-5)
    g_out = torch.from_numpy(g[f"{tag}.g_out"]).to(DEV)
    gl = torch.tensor(float(g[f"{tag}.g_loss"]), device=DEV)
    gz, gE = ops.vq_bwd(z, E, idx, g_out, gl, depth > 1, 0.25, use_norm)
    gz_d, gE_d = ops.vq_bwd_deterministic(z, E, idx, g_out, gl, depth > 1, 0.25, use_norm)
    assert torch.equal(gz, gz_d)                                                    # one per-token routine
    for name, got in (("gz", gz), ("gE", gE), ("gE_det", gE_d)):
        err = _rel_l2(got.cpu().numpy(), g[f"{tag}.{'gz' if name == 'gz' else 'gE'}"])
        assert err < 1e-5, (name, err)
    emb = ops.vq_embed(E, idx, depth, use_norm)                                     # decode_codes: the accumulated code
    np.testing.assert_allclose(emb.cpu().numpy(), out.reshape(-1, D).cpu().numpy(), atol=1e-6)


@pytest.mark.parametrize("D", [64, 256])
def test_codes_bit_exact_vs_oracle_with_near_tie_audit(D):
    M, K = 16384, 8192
    g = torch.Generator().manual_seed(D)
    z, E = torch.randn(M, D, generator=g), torch.randn(K, D, generator=g)
    ref = O.vq_lookup_np(z.numpy(), E.numpy())
    _, _, idx = ops.vq_fwd(z.to(DEV), E.to(DEV), 1, 0.25)
    mism = np.nonzero(idx.cpu().numpy()[:, 0] != ref)[0]
    if len(mism):   # only fp32 near-ties may differ
        assert len(mism) <= 2 and (O.vq_top2_gap_f64(z.numpy()[mism], E.numpy()) < 1e-6).all(), mism


@pytest.mark.parametrize("D", [64, 128, 256])
def test_full_size_properties(D):
    M, K = 131072, 8192
    g = torch.Generator(device=DEV).manual_seed(D)
    z, E = torch.randn(M, D, device=DEV, generator=g), torch.randn(K, D, device=DEV, generator=g)
    out, loss, idx = ops.vq_fwd(z, E, 1, 0.25)
    assert idx.min() >= 0 and idx.max() < K and idx.dtype == torch.int64
    q = torch.nn.functional.normalize(E[idx[:, 0]], dim=-1)
    assert (out - q).abs().max() < 1e-6
    zn = torch.nn.functional.normalize(z, dim=-1)
    np.testing.assert_allclose(loss.item(), 1.25 * ((q - zn) ** 2).mean().item(), rtol=1e-5)
    rnd = torch.randint(0, K, (M, 32), device=DEV, generator=g)
    en = torch.nn.functional.normalize(E, dim=-1)
    d_best = ((zn - en[idx[:, 0]]) ** 2).sum(-1)
    d_rnd = torch.stack([((zn - en[rnd[:, j]]) ** 2).sum(-1) for j in range(32)], 1).min(dim=1).values
    assert (d_best <= d_rnd + 1e-6).all()
    _, _, idx2 = ops.vq_fwd(q.contiguous(), E, 1, 0.25)
    assert (idx2 == idx).float().mean().item() > 0.9999
    out4, _, idx4 = ops.vq_fwd(z, E, 4, 0.25)
    assert torch.equal(idx4[:, 0], idx[:, 0])
    np.testing.assert_allclose(ops.vq_embed(E, idx, 1).cpu().numpy(), out.cpu().numpy(), atol=1e-6)
    np.testing.assert_allclose(ops.vq_embed(E, idx4, 4).cpu().numpy(), out4.cpu().numpy(), atol=1e-5)


@pytest.mark.parametrize("deterministic", [False, True], ids=["atomic", "deterministic"])
@pytest.mark.parametrize("use_norm", [True, False], ids=["norm", "raw"])
@pytest.mark.parametrize("depth", [1, 4])
@pytest.mark.parametrize("D", [64, 256])
def test_ema_statistics_and_update_against_fp64(D, depth, use_norm, deterministic):
    M, K = 32768, 4096
    g = torch.Generator().manual_seed(3)
    E = torch.randn(K, D, generator=g)
    z = E[torch.randint(0, 200, (M,), generator=g)] + 0.01 * torch.randn(M, D, generator=g)   # clustered, as at init
    zd, Ed = z.to(DEV), E.to(DEV)
    out, loss, idx, buf = ops.vq_fwd_ema(zd, Ed, depth, 0.25, use_norm, True, deterministic)
    out0, _, idx0 = ops.vq_fwd(zd, Ed, depth, 0.25, use_norm)
    assert torch.equal(idx, idx0) and torch.equal(out, out0)
    n, s = buf[K * D:].cpu().numpy(), buf[:K * D].view(K, D).cpu().double().numpy()
    n_ref, s_ref = EO.statistics(z.numpy(), E.numpy(), idx.cpu().numpy(), use_norm)
    np.testing.assert_array_equal(n, n_ref.astype(np.float32))
    assert _rel_l2(s, s_ref) < 1e-5
    want = EO.loss(z.numpy(), E.numpy(), idx.cpu().numpy(), 0.25, use_norm)
    assert abs(loss.item() - want) <= 1e-5 * abs(want) + 1e-12
    if deterministic:
        _, _, _, buf2 = ops.vq_fwd_ema(zd, Ed, depth, 0.25, use_norm, True, True)
        assert torch.equal(buf, buf2)
    cs = torch.rand(K, generator=g) * 20
    ea = torch.randn(K, D, generator=g)
    cs_ref, ea_ref, w_ref = EO.update(cs.numpy(), ea.numpy(), n, s, 0.99, 1e-5)
    csd, ead, wd = cs.to(DEV), ea.to(DEV), torch.empty(K, D, device=DEV)
    ops.vq_ema_update(buf, csd, ead, wd, 0.99, 1e-5)
    assert _rel_l2(csd.cpu().numpy(), cs_ref) < 1e-6
    assert _rel_l2(ead.cpu().numpy(), ea_ref) < 1e-6
    assert np.abs(wd.cpu().double().numpy() - w_ref).max() / np.abs(w_ref).max() < 1e-5


def test_deterministic_codebook_gradient_is_byte_identical():
    M, D, K = 65536, 256, 8192
    g = torch.Generator().manual_seed(9)
    E = torch.randn(K, D, generator=g).to(DEV)
    z = (E[torch.randint(0, 300, (M,), generator=g).to(DEV)] + 0.05 * torch.randn(M, D, generator=g).to(DEV))
    g_out = torch.randn(M, D, generator=g).to(DEV)
    grads = []
    torch.use_deterministic_algorithms(True, warn_only=True)   # what B200VQ_DETERMINISTIC=1 selects at import
    try:
        _two_runs(z, E, g_out, D, K, grads)
    finally:
        torch.use_deterministic_algorithms(False)
    assert torch.equal(grads[0][0], grads[1][0])
    assert grads[0][1].cpu().numpy().tobytes() == grads[1][1].cpu().numpy().tobytes()


def _two_runs(z, E, g_out, D, K, grads):
    for _ in range(2):
        vq = etb.VectorQuantizer(D, K, use_residual=True, num_quantizers=4).to(DEV)
        vq.embedding.weight.data.copy_(E)
        zz = z.clone().requires_grad_(True)
        out, loss, _ = vq(zz)
        ((out * g_out).sum() + loss).backward()
        grads.append((zz.grad.clone(), vq.embedding.weight.grad.clone()))


def _vq_f64(z, E, idx, qc, use_norm):
    """quantizers.py:38-63,85-92 in float64 with the codes given, norm = identity when use_norm is False"""
    beta = qc.get("beta", 0.25)
    nrm = O.l2norm if use_norm else (lambda x: x)

    def one(r, i):
        zq_n, z_n = nrm(E[i]), nrm(r)
        return zq_n, beta * ((zq_n.detach() - z_n) ** 2).mean() + ((zq_n - z_n.detach()) ** 2).mean()
    if not qc.get("use_residual", False):
        zq, loss = one(z, idx)
    else:
        zq, r, losses = torch.zeros_like(z), z.detach().clone(), []
        for t in range(int(qc["num_quantizers"])):
            q, l = one(r, idx[..., t])
            r, zq = r - q, zq + q
            losses.append(l)
        loss = torch.stack(losses, dim=-1).mean()
    return z + (zq - z).detach(), loss


MODULE_CASES = [(D, res, norm, False) for D in (64, 256) for res in (False, True) for norm in (True, False)] + [(256, True, True, True)]


@pytest.mark.parametrize("D,residual,use_norm,ema", MODULE_CASES,
                         ids=[f"d{D}-{'rq4' if r else 'plain'}-{'norm' if n else 'raw'}{'-ema' if e else ''}" for D, r, n, e in MODULE_CASES])
def test_vitvq_modules_vs_fp64_oracle(D, residual, use_norm, ema):
    torch.backends.cuda.matmul.allow_tf32 = False
    etb.set_precision("parity")
    cfg = copy.deepcopy(O.CONFIGS["tiny"])
    qc = cfg["quantizer"]
    qc.update(embed_dim=D, use_norm=use_norm)
    if residual:
        qc.update(use_residual=True, num_quantizers=4)
    sd = O.init_vitvq_sd(cfg, seed=1)
    B = 2
    img = torch.rand(B, 3, 64, 64, generator=torch.Generator().manual_seed(2)).to(DEV)
    p, gg = cfg["patch_size"], cfg["image_size"] // cfg["patch_size"]
    e, d = cfg["encoder"], cfg["decoder"]
    E = sd["quantizer.embedding.weight"].to(DEV)
    mods = dict(encoder=etb.ViTEncoder(cfg["image_size"], p, **e), decoder=etb.ViTDecoder(cfg["image_size"], p, **d),
                quantizer=(etb.EMAVectorQuantizer if ema else etb.VectorQuantizer)(**qc),
                pre_quant=etb.QuantLinear(e["dim"], D), post_quant=etb.QuantLinear(D, d["dim"]))
    for name, m in mods.items():
        m.load_state_dict({k[len(name) + 1:]: v for k, v in sd.items() if k.startswith(name + ".")}, strict=not ema)
        m.to(DEV)
    z = mods["pre_quant"](mods["encoder"](img))
    zq, qloss, idx = mods["quantizer"](z)
    rec = mods["decoder"](mods["post_quant"](zq))
    loss = ((rec - img) ** 2).mean() + qloss
    loss.backward()
    # codes bit-exact on identical z against the fp32 lookup (reference arithmetic); near ties audited
    with torch.no_grad():
        zf = z.detach().reshape(-1, D).cpu()
        if use_norm and not residual:
            ref = torch.from_numpy(O.vq_lookup_np(zf.numpy(), E.cpu().numpy()))
            mism = (idx.reshape(-1).cpu() != ref).nonzero().view(-1).numpy()
            assert len(mism) <= 2 and (O.vq_top2_gap_f64(zf.numpy()[mism], E.cpu().numpy()) < 2e-6).all()
    # fp64 oracle on the library's codes: forward and every parameter gradient
    sd64 = {k: v.double().to(DEV).requires_grad_(v.is_floating_point() and "pos_embedding" not in k) for k, v in sd.items()}
    h64 = O.vit_encoder(sd64, img.double(), patch=p, depth=e["depth"], heads=e["heads"], prefix="encoder.")
    z64 = h64 @ sd64["pre_quant.weight"].t() + sd64["pre_quant.bias"]
    assert (z.double() - z64).abs().max() / z64.abs().max() < 5e-5
    Eq = sd64["quantizer.embedding.weight"] if not ema else sd64["quantizer.embedding.weight"].detach()
    zq64, qloss64 = _vq_f64(z64, Eq, idx, qc, use_norm)
    t64 = zq64 @ sd64["post_quant.weight"].t() + sd64["post_quant.bias"]
    rec64 = O.vit_decoder(sd64, t64, patch=p, depth=d["depth"], heads=d["heads"], grid_hw=(gg, gg), prefix="decoder.")
    assert (rec.double() - rec64).abs().max() / rec64.abs().max() < 5e-5
    if not ema:   # the EMA codebook has its own loss and no codebook gradient (tests/test_gpu_ema_codebook.py)
        loss64 = ((rec64 - img.double()) ** 2).mean() + qloss64
        assert abs(loss.item() - loss64.item()) < 5e-5 * abs(loss64.item())
        loss64.backward()
        for k, v in sd64.items():
            if v.grad is None or v.grad.norm() == 0:
                continue
            mod, _, pname = k.partition(".")
            pp = dict(mods[mod].named_parameters())[pname]
            rel = ((pp.grad.double() - v.grad).norm() / v.grad.norm()).item()
            assert rel < 2e-4, (k, rel)
    # decode_codes == decoder(post_quant(embed_codes)) against the fp64 oracle (the EMA module's weight has been updated)
    with torch.no_grad():
        dec = mods["decoder"](mods["post_quant"](mods["quantizer"].embed_codes(idx)))
        W = mods["quantizer"].embedding.weight.detach().double()
        q64 = (O.l2norm(W) if use_norm else W)[idx]
        q64 = q64.sum(-2) if residual else q64
        t2 = q64 @ sd64["post_quant.weight"].t() + sd64["post_quant.bias"]
        dec64 = O.vit_decoder(sd64, t2, patch=p, depth=d["depth"], heads=d["heads"], grid_hw=(gg, gg), prefix="decoder.")
    assert (dec.double() - dec64).abs().max() / dec64.abs().max() < 5e-5
