"""Generate tests/golden/*.npz by running the UNMODIFIED reference modules.

Needs a checkout of the reference (B200VQ_REFERENCE).  The reference is imported by file
path (its package __init__ pulls in pytorch_lightning / omegaconf, absent here -- SURVEY.md
section 8c) with one harness-side shim: ``np.float = float`` (reference layers.py:57 uses the
alias numpy removed in 1.24).  No reference source is copied; only its outputs are stored.

    python oracle/gen_golden.py            # rewrites tests/golden/

The fixtures are what pins oracle/vitvq_oracle.py (tests/test_oracle_golden.py) and, through
it, the CUDA path.
"""
import importlib.util
import os
import sys

import numpy as np
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import vitvq_oracle as O  # noqa: E402

REF = os.environ.get("B200VQ_REFERENCE", "")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")


def load_reference():
    np.float = float  # shim for reference layers.py:57
    mods = {}
    for name in ("layers", "quantizers"):
        path = os.path.join(REF, "enhancing", "modules", "stage1", name + ".py")
        spec = importlib.util.spec_from_file_location("ref_stage1_" + name, path)
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
        mods[name] = m
    return mods["layers"], mods["quantizers"]


def npd(sd):
    return {k: v.detach().cpu().numpy() for k, v in sd.items()}


def gen_vit(L, Q):
    """tiny ViT-VQ wired like ViTVQ.__init__/forward (vitvqgan.py:35-39,44-48,61-72)."""
    torch.manual_seed(1234)
    image, patch = 32, 8
    enc_cfg = dict(dim=64, depth=2, heads=2, mlp_dim=128)
    dec_cfg = dict(dim=96, depth=2, heads=3, mlp_dim=160, dim_head=32)
    enc = L.ViTEncoder(image_size=image, patch_size=patch, **enc_cfg)
    dec = L.ViTDecoder(image_size=image, patch_size=patch, **dec_cfg)
    vq = Q.VectorQuantizer(embed_dim=32, n_embed=256)
    pre, post = nn.Linear(64, 32), nn.Linear(32, 96)
    # give LN affine / biases non-trivial values so the fixtures exercise them
    with torch.no_grad():
        for m in list(enc.modules()) + list(dec.modules()):
            if isinstance(m, nn.LayerNorm):
                m.weight.add_(0.1 * torch.randn_like(m.weight))
                m.bias.add_(0.1 * torch.randn_like(m.bias))
            if isinstance(m, nn.Linear) and m.bias is not None:
                m.bias.add_(0.05 * torch.randn_like(m.bias))
    img = torch.rand(2, 3, image, image)
    h = enc(img)
    z = pre(h)
    zq, qloss, idx = vq(z)
    rec = dec(post(zq))
    loss = ((rec - img) ** 2).mean() + qloss
    loss.backward()
    sd = {}
    for pfx, mod in (("encoder.", enc), ("decoder.", dec), ("quantizer.", vq), ("pre_quant.", pre), ("post_quant.", post)):
        sd.update({pfx + k: v for k, v in mod.state_dict().items()})
    grads = {}
    for pfx, mod in (("encoder.", enc), ("decoder.", dec), ("quantizer.", vq), ("pre_quant.", pre), ("post_quant.", post)):
        for k, p in mod.named_parameters():
            # keep the fixture small: one representative of every parameter kind
            keep = ("to_patch_embedding", "layers.0.", "transformer.norm", "to_pixel", "embedding", "weight", "bias")
            full = pfx + k
            if p.grad is not None and (("layers." not in full) or "layers.0." in full or "layers.1.1" in full) \
                    and any(s in full for s in keep):
                grads["grad." + full] = p.grad.numpy()
    out = {"sd." + k: v for k, v in npd(sd).items()}
    out.update(grads)
    out.update(img=img.numpy(), enc_out=h.detach().numpy(), z=z.detach().numpy(), zq=zq.detach().numpy(),
               qloss=qloss.detach().numpy(), idx=idx.numpy(), rec=rec.detach().numpy(), loss=loss.detach().numpy(),
               cfg_image=np.int64(image), cfg_patch=np.int64(patch))
    # decode_codes path (vitvqgan.py:81-90)
    with torch.no_grad():
        q = vq.norm(vq.embedding(idx))
        out["decode_codes"] = dec(post(q)).numpy()
    O.save_golden(os.path.join(OUT, "vit_tiny.npz"), out)       # more than 1 MB: vit_tiny.npz + continuation files
    print("vit_tiny: loss", float(loss), "qloss", float(qloss), "distinct codes", idx.unique().numel())


def gen_vq(Q):
    out = {}
    for tag, kw in (("plain", dict()), ("res4", dict(use_residual=True, num_quantizers=4)),
                    ("res2", dict(use_residual=True, num_quantizers=2))):
        torch.manual_seed(7)
        vq = Q.VectorQuantizer(embed_dim=32, n_embed=384, beta=0.25, **kw)
        z = torch.randn(3, 40, 32, requires_grad=True)
        zq, loss, idx = vq(z)
        g_out = torch.randn_like(zq)
        g_loss = 0.7
        (zq * g_out).sum().add(loss * g_loss).backward()
        out.update({f"{tag}.E": vq.embedding.weight.detach().numpy(), f"{tag}.z": z.detach().numpy(),
                    f"{tag}.zq": zq.detach().numpy(), f"{tag}.loss": loss.detach().numpy(), f"{tag}.idx": idx.numpy(),
                    f"{tag}.g_out": g_out.numpy(), f"{tag}.g_loss": np.float32(g_loss),
                    f"{tag}.gz": z.grad.numpy(), f"{tag}.gE": vq.embedding.weight.grad.numpy()})
        print("vq", tag, "loss", float(loss), "idx shape", tuple(idx.shape))
    # clustered inputs: many tokens per code (what real encoder outputs look like at init)
    torch.manual_seed(11)
    vq = Q.VectorQuantizer(embed_dim=32, n_embed=384)
    z = (torch.randn(1, 1, 32) + 0.01 * torch.randn(2, 64, 32)).requires_grad_(True)
    zq, loss, idx = vq(z)
    loss.backward()
    out.update({"clustered.E": vq.embedding.weight.detach().numpy(), "clustered.z": z.detach().numpy(),
                "clustered.zq": zq.detach().numpy(), "clustered.loss": loss.detach().numpy(), "clustered.idx": idx.numpy(),
                "clustered.gz": z.grad.numpy(), "clustered.gE": vq.embedding.weight.grad.numpy()})
    np.savez_compressed(os.path.join(OUT, "vq_cases.npz"), **out)


def gen_pos(L):
    out = {}
    for dim, g in ((64, (4, 4)), (96, (4, 6)), (768, (32, 32))):
        t = L.get_2d_sincos_pos_embed(dim, g).astype(np.float32)
        if t.size <= 4096:
            out[f"pos_{dim}_{g[0]}x{g[1]}"] = t
        else:  # big table: keep a strided sample and moments
            out[f"pos_{dim}_{g[0]}x{g[1]}_sample"] = t[::37, ::29].copy()
            out[f"pos_{dim}_{g[0]}x{g[1]}_sum"] = np.float64(t.astype(np.float64).sum())
            out[f"pos_{dim}_{g[0]}x{g[1]}_abs"] = np.float64(np.abs(t.astype(np.float64)).sum())
    np.savez_compressed(os.path.join(OUT, "pos_embed.npz"), **out)


def gen_blocks(L):
    """one Attention and one FeedForward / PreNorm in isolation, fwd + input/param grads."""
    torch.manual_seed(99)
    out = {}
    attn = L.Attention(64, heads=2, dim_head=32)
    x = torch.randn(2, 24, 64, requires_grad=True)
    y = attn(x)
    g = torch.randn_like(y)
    (y * g).sum().backward()
    out.update({"attn.x": x.detach().numpy(), "attn.y": y.detach().numpy(), "attn.g": g.numpy(), "attn.gx": x.grad.numpy(),
                "attn.w_qkv": attn.to_qkv.weight.detach().numpy(), "attn.w_out": attn.to_out.weight.detach().numpy(),
                "attn.b_out": attn.to_out.bias.detach().numpy(), "attn.gw_qkv": attn.to_qkv.weight.grad.numpy(),
                "attn.gw_out": attn.to_out.weight.grad.numpy(), "attn.gb_out": attn.to_out.bias.grad.numpy()})
    ff = L.PreNorm(64, L.FeedForward(64, 96))
    with torch.no_grad():
        ff.norm.weight.add_(0.2 * torch.randn(64))
        ff.norm.bias.add_(0.2 * torch.randn(64))
    x = torch.randn(2, 24, 64, requires_grad=True)
    y = ff(x)
    (y * g).sum().backward()
    out.update({"ff.x": x.detach().numpy(), "ff.y": y.detach().numpy(), "ff.g": g.numpy(), "ff.gx": x.grad.numpy()})
    out.update({"ff.sd." + k: v for k, v in npd(ff.state_dict()).items()})
    out.update({"ff.grad." + k: p.grad.numpy() for k, p in ff.named_parameters()})
    np.savez_compressed(os.path.join(OUT, "blocks.npz"), **out)


def gen_lossops():
    """the loss stage's two native ops through the reference's own CPU formulas (losses/op/upfirdn2d.py:168-206
    `upfirdn2d_native`, losses/op/fused_act.py:110-122), fwd + first and second order gradients.  The op modules JIT-compile
    their CUDA extension at import (`load(...)`): that call is stubbed, nothing else of the file is touched."""
    import torch.utils.cpp_extension as ce
    ce.load = lambda *a, **k: None
    ops = {}
    for name in ("upfirdn2d", "fused_act"):
        spec = importlib.util.spec_from_file_location("ref_lossop_" + name, os.path.join(REF, "enhancing", "losses", "op", name + ".py"))
        ops[name] = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(ops[name])
    torch.manual_seed(77)
    out = {}
    k1 = torch.tensor([1.0, 3.0, 3.0, 1.0])
    k = k1[None, :] * k1[:, None]
    k = k / k.sum()                                        # Blur kernel of every shipped discriminator (losses/layers.py:140-155)
    cases = [(1, 1, (2, 1)), (1, 1, (1, 1)), (2, 1, (2, 1, 1, 2)), (1, 2, (1, 1)), (2, 2, (0, 0)), (1, 1, (-1, 2, 0, -1)), (3, 2, (2, 2)),
             (1, 2, (0, 0))]
    x = torch.randn(2, 5, 12, 10)
    out["up.x"], out["up.kernel"] = x.numpy(), k.numpy()
    for i, (u, d, pad) in enumerate(cases):
        xi = x.clone().requires_grad_(True)
        y = ops["upfirdn2d"].upfirdn2d(xi, k, up=u, down=d, pad=pad)
        w = torch.randn_like(y)
        gx, = torch.autograd.grad((y * w).sum(), xi)
        out[f"up.{i}.cfg"] = np.array([u, d] + list(pad if len(pad) == 4 else (pad[0], pad[1], pad[0], pad[1])))
        out[f"up.{i}.y"], out[f"up.{i}.w"], out[f"up.{i}.gx"] = y.detach().numpy(), w.numpy(), gx.numpy()
    # asymmetric kernel: catches a missing flip
    ka = torch.randn(3, 4)
    xi = x.clone().requires_grad_(True)
    y = ops["upfirdn2d"].upfirdn2d(xi, ka, up=2, down=1, pad=(1, 2, 2, 1))
    w = torch.randn_like(y)
    out["up.asym.kernel"], out["up.asym.y"], out["up.asym.w"] = ka.numpy(), y.detach().numpy(), w.numpy()
    out["up.asym.gx"] = torch.autograd.grad((y * w).sum(), xi)[0].numpy()
    # fused bias + leaky ReLU (slope 0.2, gain sqrt(2)), 4-D and 2-D inputs, with and without bias, incl. double backward
    for tag, shape in (("4d", (3, 6, 7, 5)), ("2d", (9, 6))):
        xin = torch.randn(*shape, requires_grad=True)
        b = torch.randn(6, requires_grad=True)
        for use_b in (True, False):
            y = ops["fused_act"].fused_leaky_relu(xin, b if use_b else None)
            w = torch.randn_like(y)
            grads = torch.autograd.grad((y * w).sum(), [xin] + ([b] if use_b else []), create_graph=True)
            key = f"act.{tag}.{'b' if use_b else 'nob'}"
            out[key + ".y"], out[key + ".w"], out[key + ".gx"] = y.detach().numpy(), w.numpy(), grads[0].detach().numpy()
            if use_b:
                out[key + ".gb"] = grads[1].detach().numpy()
            # second order: d/dw-direction of sum(gx * v) -- what an R1 penalty differentiates
            v = torch.randn_like(xin)
            out[key + ".v"] = v.numpy()
        out[f"act.{tag}.x"], out[f"act.{tag}.bias"] = xin.detach().numpy(), b.detach().numpy()
    np.savez_compressed(os.path.join(OUT, "lossops.npz"), **out)


if __name__ == "__main__":
    if not os.path.isdir(REF):
        sys.exit(f"{REF} not present: golden vectors need a reference checkout (B200VQ_REFERENCE)")
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(4)
    L, Q = load_reference()
    gen_pos(L)
    gen_blocks(L)
    gen_vq(Q)
    gen_vit(L, Q)
    gen_lossops()
    for f in sorted(os.listdir(OUT)):
        print(f, os.path.getsize(os.path.join(OUT, f)))
