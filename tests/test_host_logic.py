"""Host logic of the stage-1 path on the CPU: the autograd Functions of functional.py (fused transformer stacks in all three
data paths, patch embed / to_pixel, QuantLinear, VectorQuantizeFn, the positional-table fusion) with every C-ABI call
replaced by a torch stand-in written from the contract in include/b200vq.h (tests/emulated_ops.py), against the outputs of the
UNMODIFIED reference (tests/golden/vit_tiny.npz).  What this can catch: wrong operand majors, a missing 1/S, a gradient
routed to the wrong parameter, a positional table added twice.  What it cannot: the kernels -- those are the -m gpu tests."""
import os
import sys

import numpy as np
import pytest
import torch

import enhancing_transformers_b200 as etb
from oracle import vitvq_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD_CFG = dict(image_size=32, patch_size=8, encoder=dict(dim=64, depth=2, heads=2, mlp_dim=128),
                decoder=dict(dim=96, depth=2, heads=3, mlp_dim=160, dim_head=32), quantizer=dict(embed_dim=32, n_embed=256))


def _build(sd, fuse_pos):
    cfg = GOLD_CFG
    e, d, q = cfg["encoder"], cfg["decoder"], cfg["quantizer"]

    class Holder(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.encoder = etb.ViTEncoder(cfg["image_size"], cfg["patch_size"], **e)
            self.decoder = etb.ViTDecoder(cfg["image_size"], cfg["patch_size"], **d)
            self.quantizer = etb.VectorQuantizer(**q)
            self.pre_quant = etb.QuantLinear(e["dim"], q["embed_dim"])
            self.post_quant = etb.QuantLinear(q["embed_dim"], d["dim"])
    m = Holder()
    m.load_state_dict(sd, strict=True)
    if fuse_pos:
        etb.fuse_post_quant_pos(m)
    return m


@pytest.mark.parametrize("mode,fuse_pos", [("parity", False), ("tf32", False), ("fp16", False), ("fp16", True)])
def test_vitvq_host_logic_with_emulated_kernels(golden_dir, monkeypatch, mode, fuse_pos):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import emulated_ops
    emulated_ops.install(monkeypatch)
    g = O.load_golden(os.path.join(golden_dir, "vit_tiny.npz"))
    sd = {k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("sd.")}
    prev = etb.set_precision(mode)
    try:
        m = _build(sd, fuse_pos)
        img = torch.from_numpy(g["img"])
        h = m.encoder(img)
        z = m.pre_quant(h)
        zq, qloss, idx = m.quantizer(z)
        rec = m.decoder(m.post_quant(zq))
        loss = ((rec - img) ** 2).mean() + qloss
        loss.backward()
        with torch.no_grad():
            dec_codes = m.decoder(m.post_quant(m.quantizer.embed_codes(torch.from_numpy(g["idx"]))))
    finally:
        etb.set_precision(prev)
    half = mode == "fp16"       # the stand-ins really round to fp16 there (dtype drives the scaling logic)
    tol = 2e-3 if half else 2e-5

    def rel(a, b):
        return ((a - b).abs().max() / b.abs().max()).item()
    assert rel(h.detach(), torch.from_numpy(g["enc_out"])) < tol
    assert rel(z.detach(), torch.from_numpy(g["z"])) < tol
    same_codes = torch.equal(idx, torch.from_numpy(g["idx"]))
    assert same_codes or half
    assert rel(dec_codes, torch.from_numpy(g["decode_codes"])) < tol
    if same_codes:
        assert rel(rec.detach(), torch.from_numpy(g["rec"])) < tol
        assert abs(loss.item() - float(g["loss"])) < tol * float(g["loss"])
    mods = dict(encoder=m.encoder, decoder=m.decoder, quantizer=m.quantizer, pre_quant=m.pre_quant, post_quant=m.post_quant)
    for k in g.files:
        if k.startswith("grad."):
            mod, _, pname = k[5:].partition(".")
            p = dict(mods[mod].named_parameters())[pname]
            want = torch.from_numpy(g[k])
            e = ((p.grad - want).norm() / want.norm().clamp_min(1e-30)).item()
            assert e < ((2e-2 if same_codes else 6e-2) if half else 2e-4), (k, e)
