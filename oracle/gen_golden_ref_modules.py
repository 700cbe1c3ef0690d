#!/usr/bin/env python
"""Golden vectors from the reference's own nn.Modules (the unmodified copies oracle/build_ref.py places under
oracle/_ref), for the tests that compare against them:

    python oracle/build_ref.py && python oracle/gen_golden_ref_modules.py

writes tests/golden/ref_nonsquare.npz, ref_gumbel.npz, ref_vitvq_small.npz, ref_gpt_class.npz and ref_gpt_sample.npz.
Everything runs on the CPU in fp32; the Gumbel noise comes from oracle.vitvq_oracle.seeded_gumbel_softmax so that a
GPU run can replay exactly the same draws."""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
from oracle import vitvq_oracle as O  # noqa: E402

REF_DIR = os.path.join(HERE, "_ref", "enhancing_ref")
OUT = os.path.join(ROOT, "tests", "golden")


def _load(name, file):
    if not hasattr(np, "float"):
        np.float = float
    if "omegaconf" not in sys.modules:                      # stage2 layers.py imports it for a type annotation only
        stub = types.ModuleType("omegaconf")
        stub.OmegaConf = type("OmegaConf", (), {})
        sys.modules["omegaconf"] = stub
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF_DIR, file))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def _np(t):
    return t.detach().cpu().numpy()


def nonsquare(RL):
    """ViTEncoder / ViTDecoder with (height, width) patches"""
    torch.manual_seed(0)
    kw = dict(image_size=(32, 48), patch_size=(8, 4), dim=64, depth=1, heads=2, mlp_dim=128, dim_head=32)
    e, d = RL.ViTEncoder(**kw), RL.ViTDecoder(**kw)
    img = torch.rand(2, 3, 32, 48)
    h = e(img)
    rec = d(h)
    out = {"img": _np(img), "h": _np(h), "rec": _np(rec)}
    out.update({"enc." + k: _np(v) for k, v in e.state_dict().items()})
    out.update({"dec." + k: _np(v) for k, v in d.state_dict().items()})
    np.savez_compressed(os.path.join(OUT, "ref_nonsquare.npz"), **out)


def gumbel(RQ):
    """GumbelQuantizer, train (soft samples, gradients) and eval (hard samples), plain and residual"""
    out = {}
    F = torch.nn.functional
    orig = F.gumbel_softmax
    try:
        for residual in (False, True):
            tag = "res" if residual else "plain"
            kw = dict(embed_dim=32, n_embed=512, temp_init=0.7, use_residual=residual, num_quantizers=3 if residual else None)
            torch.manual_seed(0)
            q = RQ.GumbelQuantizer(**kw)
            z0 = torch.randn(2, 96, 32)
            q.train()
            z = z0.clone().requires_grad_(True)
            F.gumbel_softmax = O.seeded_gumbel_softmax(123)
            zq, loss, idx = q(z)
            (zq.square().mean() + loss).backward()
            out.update({f"{tag}.z0": _np(z0), f"{tag}.zq": _np(zq), f"{tag}.loss": _np(loss), f"{tag}.idx": _np(idx),
                        f"{tag}.gE": _np(q.embedding.weight.grad)})
            if z.grad is not None:
                out[f"{tag}.gz"] = _np(z.grad)
            out.update({f"{tag}.sd.{k}": _np(v) for k, v in q.state_dict().items()})
            q.eval()
            F.gumbel_softmax = O.seeded_gumbel_softmax(7)
            with torch.no_grad():
                zq_e, _, idx_e = q(z0)
            out.update({f"{tag}.eval_zq": _np(zq_e), f"{tag}.eval_idx": _np(idx_e)})
    finally:
        F.gumbel_softmax = orig
    np.savez_compressed(os.path.join(OUT, "ref_gumbel.npz"), **out)


def vitvq_small(RL, RQ):
    """encoder -> pre_quant -> residual VQ -> post_quant -> decoder, fwd + bwd, on a config no other fixture covers
    (parameters from O.init_vitvq_sd(cfg, seed=7), image from seed 3)"""
    cfg = O.SMALL_REF_CFG
    sd = O.init_vitvq_sd(cfg, seed=7)
    e, d, q = cfg["encoder"], cfg["decoder"], cfg["quantizer"]
    ref = dict(encoder=RL.ViTEncoder(48, 8, **e), decoder=RL.ViTDecoder(48, 8, **d), quantizer=RQ.VectorQuantizer(**q),
               pre_quant=torch.nn.Linear(64, 32), post_quant=torch.nn.Linear(32, 64))
    for name, m in ref.items():
        m.load_state_dict({k[len(name) + 1:]: v for k, v in sd.items() if k.startswith(name + ".")}, strict=True)
    img = torch.rand(2, 3, 48, 48, generator=torch.Generator().manual_seed(3))
    quant, qloss, idx = ref["quantizer"](ref["pre_quant"](ref["encoder"](img)))
    rec = ref["decoder"](ref["post_quant"](quant))
    loss = ((rec - img) ** 2).mean() + qloss
    loss.backward()
    out = {"idx": _np(idx), "rec": _np(rec), "loss": _np(loss)}
    for name, m in ref.items():
        for pn, p in m.named_parameters():
            if p.grad is not None:
                out[f"grad.{name}.{pn}"] = _np(p.grad)
    np.savez_compressed(os.path.join(OUT, "ref_vitvq_small.npz"), **out)


def gpt_class(S):
    """GPT forward on a config no other fixture covers: no biases, a 3-token condition prefix, enlarged weights"""
    torch.manual_seed(3)
    cfg = dict(vocab_cond_size=7, vocab_img_size=33, embed_dim=96, cond_num_tokens=3, img_num_tokens=21, n_heads=3, n_layers=2,
               mlp_bias=False, attn_bias=False)
    ref = S.GPT(**cfg)
    with torch.no_grad():
        ref.pos_emb_code.normal_(0, 0.2)
        ref.pos_emb_cond.normal_(0, 0.2)
        for p in ref.parameters():
            if p.dim() == 2:
                p.mul_(6.0)
    codes = torch.randint(0, 33, (2, 21))
    conds = torch.randint(0, 7, (2, 3))
    out = {"codes": _np(codes), "conds": _np(conds), "logits": _np(ref(codes, conds))}
    out.update({"sd." + k: _np(v) for k, v in ref.state_dict().items()})
    np.savez_compressed(os.path.join(OUT, "ref_gpt_class.npz"), **out)


SAMPLE_KWARGS = (dict(top_k=7), dict(top_p=0.8), dict(top_k=12, top_p=0.6, softmax_temperature=0.7))


def gpt_sample(S):
    """GPT.sample with top-k / nucleus filtering: the codes drawn and the logits returned, torch RNG seeded with 123"""
    cfg = dict(vocab_cond_size=6, vocab_img_size=64, embed_dim=64, cond_num_tokens=2, img_num_tokens=9, n_heads=2, n_layers=1)
    torch.manual_seed(7)
    ref = S.GPT(**cfg).eval()
    with torch.no_grad():
        ref.pos_emb_code.normal_(0, 0.3)
        for p in ref.parameters():
            if p.dim() == 2:
                p.mul_(10.0)
    conds = torch.randint(0, 6, (3, 2))
    out = {"conds": _np(conds)}
    out.update({"sd." + k: _np(v) for k, v in ref.state_dict().items()})
    for i, kw in enumerate(SAMPLE_KWARGS):
        torch.manual_seed(123)
        with torch.no_grad():
            logits, codes = ref.sample(conds, use_fp16=False, **kw)
        out[f"logits.{i}"], out[f"codes.{i}"] = _np(logits), _np(codes)
    np.savez_compressed(os.path.join(OUT, "ref_gpt_sample.npz"), **out)


def main() -> int:
    if not os.path.exists(os.path.join(REF_DIR, "layers.py")):
        sys.exit(f"{REF_DIR} not present: run oracle/build_ref.py with a reference checkout first")
    RL = _load("enhancing_ref_g.layers", "layers.py")
    RQ = _load("enhancing_ref_g.quantizers", "quantizers.py")
    S = _load("enhancing_ref_g.stage2_layers", "stage2_layers.py")
    nonsquare(RL)
    gumbel(RQ)
    vitvq_small(RL, RQ)
    gpt_class(S)
    gpt_sample(S)
    for f in sorted(os.listdir(OUT)):
        if f.startswith("ref_"):
            print(f, os.path.getsize(os.path.join(OUT, f)))
    return 0


if __name__ == "__main__":
    sys.exit(main())
