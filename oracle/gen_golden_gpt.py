"""Generate tests/golden/gpt_tiny.npz by running the UNMODIFIED reference stage-2 ``GPT``
(enhancing/modules/stage2/layers.py of a reference checkout, B200VQ_REFERENCE).

The file is imported by path (the package __init__ needs pytorch_lightning); its one absent import, ``omegaconf`` (used
for a type annotation only), is stubbed in sys.modules.  No reference source is copied; only outputs are stored.

    python oracle/gen_golden_gpt.py
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

REF = os.environ.get("B200VQ_REFERENCE", "")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")

CFG = dict(vocab_cond_size=10, vocab_img_size=64, embed_dim=64, cond_num_tokens=2, img_num_tokens=30, n_heads=2, n_layers=2)


def load_reference_stage2(path=None):
    if "omegaconf" not in sys.modules:
        stub = types.ModuleType("omegaconf")
        stub.OmegaConf = type("OmegaConf", (), {})
        sys.modules["omegaconf"] = stub
    path = path or os.path.join(REF, "enhancing", "modules", "stage2", "layers.py")
    spec = importlib.util.spec_from_file_location("ref_stage2_layers", path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def perturb(gpt):
    """the reference initialises positional tables and biases to zero: give them values so the fixture exercises them"""
    g = torch.Generator().manual_seed(4321)
    with torch.no_grad():
        for m in gpt.modules():
            if isinstance(m, nn.LayerNorm):
                m.weight.add_(0.1 * torch.randn(m.weight.shape, generator=g))
                m.bias.add_(0.1 * torch.randn(m.bias.shape, generator=g))
            if isinstance(m, nn.Linear):
                m.weight.mul_(8.0)                       # std 0.02 -> 0.16: scores and logits that are not all ~0
                if m.bias is not None:
                    m.bias.add_(0.05 * torch.randn(m.bias.shape, generator=g))
        gpt.pos_emb_cond.add_(0.3 * torch.randn(gpt.pos_emb_cond.shape, generator=g))
        gpt.pos_emb_code.add_(0.3 * torch.randn(gpt.pos_emb_code.shape, generator=g))
        gpt.tok_emb_cond.weight.mul_(20.0)
        gpt.tok_emb_code.weight.mul_(20.0)


def main():
    S = load_reference_stage2()
    torch.manual_seed(2024)
    gpt = S.GPT(**CFG)
    perturb(gpt)
    B = 3
    g = torch.Generator().manual_seed(5)
    codes = torch.randint(0, CFG["vocab_img_size"], (B, CFG["img_num_tokens"]), generator=g)
    conds = torch.randint(0, CFG["vocab_cond_size"], (B, CFG["cond_num_tokens"]), generator=g)
    logits = gpt(codes, conds)
    loss = F.cross_entropy(logits.view(-1, logits.shape[-1]), codes.view(-1))      # stage2/transformer.py:118
    loss.backward()
    out = {"sd." + k: v.detach().numpy() for k, v in gpt.state_dict().items()}
    out.update({"grad." + k: p.grad.numpy() for k, p in gpt.named_parameters()})
    out.update(codes=codes.numpy(), conds=conds.numpy(), logits=logits.detach().numpy(), loss=loss.detach().numpy())
    out.update({"cfg." + k: np.int64(v) for k, v in CFG.items()})
    # sampling (layers.py:213-303) in fp32: the codes it drew and the logits it drew them from
    gpt.eval()
    torch.manual_seed(99)
    with torch.no_grad():
        s_logits, s_codes = gpt.sample(conds, top_k=None, top_p=None, softmax_temperature=1.0, use_fp16=False)
    out.update(sample_logits=s_logits.view(B, CFG["img_num_tokens"], -1).numpy(), sample_codes=s_codes.numpy())
    np.savez_compressed(os.path.join(OUT, "gpt_tiny.npz"), **out)
    print("gpt_tiny: loss", float(loss), "logits", tuple(logits.shape), "sampled", tuple(s_codes.shape),
          os.path.getsize(os.path.join(OUT, "gpt_tiny.npz")), "bytes")


if __name__ == "__main__":
    if not os.path.isdir(REF):
        sys.exit(f"{REF} not present: golden vectors need a reference checkout (B200VQ_REFERENCE)")
    torch.set_num_threads(4)
    main()
