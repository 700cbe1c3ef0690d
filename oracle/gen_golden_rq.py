"""Generate tests/golden/rq_tiny.npz and tests/golden/ref_rq_class.npz by running the UNMODIFIED reference stage-2
``RQTransformer`` (enhancing/modules/stage2/layers.py:306-547).

rq_tiny.npz comes from a reference checkout (B200VQ_REFERENCE), loaded as gen_golden_gpt.py loads it; ref_rq_class.npz from the
copy oracle/build_ref.py vendors into oracle/_ref.  No reference source is copied; only outputs are stored.

    B200VQ_REFERENCE=<checkout> python oracle/gen_golden_rq.py
"""
import hashlib
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle.gen_golden_gpt import REF, load_reference_stage2, perturb  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden")

CFG = dict(vocab_cond_size=10, vocab_img_size=64, embed_dim=64, cond_num_tokens=2, img_num_tokens=12, depth_num_tokens=4,
           spatial_n_heads=2, depth_n_heads=2, spatial_n_layers=2, depth_n_layers=2)
# a second config no other fixture covers: no biases, a 3-token prefix, 64- and 32-wide heads, D = 3
CLASS_CFG = dict(vocab_cond_size=7, vocab_img_size=128, embed_dim=64, cond_num_tokens=3, img_num_tokens=5, depth_num_tokens=3,
                 spatial_n_heads=1, depth_n_heads=2, spatial_n_layers=1, depth_n_layers=2, mlp_bias=False, attn_bias=False)


def sd_digest(sd):
    """sha256 over the state dict's keys (sorted) and raw fp32 bytes: the fixture stores this instead of the tables themselves
    (the tests rebuild them from the seed and `perturb`, and check the bits against it)"""
    h = hashlib.sha256()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(sd[k].detach().cpu().contiguous().numpy().tobytes())
    return h.hexdigest()


def _inputs(cfg, B, seed):
    g = torch.Generator().manual_seed(seed)
    codes = torch.randint(0, cfg["vocab_img_size"], (B, cfg["img_num_tokens"], cfg["depth_num_tokens"]), generator=g)
    conds = torch.randint(0, cfg["vocab_cond_size"], (B, cfg["cond_num_tokens"]), generator=g)
    return codes, conds


def tiny(S):
    torch.manual_seed(2024)
    rq = S.RQTransformer(**CFG)
    init = sd_digest(rq.state_dict())                   # seeded construction, untouched
    perturb(rq)
    B = 3
    codes, conds = _inputs(CFG, B, 5)
    logits = rq(codes, conds)
    loss = F.cross_entropy(logits.view(-1, logits.shape[-1]), codes.view(-1))      # stage2/transformer.py:56-65,118
    loss.backward()
    # the perturbed tables are rebuilt by the tests (torch.manual_seed(2024), construction, perturb) and checked against these
    out = {"init_sha256": np.array(init), "sd_sha256": np.array(sd_digest(rq.state_dict())), "seed": np.int64(2024)}
    out.update({"shape." + k: np.array(v.shape, dtype=np.int64) for k, v in rq.state_dict().items()})
    out.update({"grad." + k: p.grad.numpy() for k, p in rq.named_parameters()})
    out.update(codes=codes.numpy(), conds=conds.numpy(), logits=logits.detach().numpy(), loss=loss.detach().numpy())
    out.update({"cfg." + k: np.int64(v) for k, v in CFG.items()})
    rq.eval()
    torch.manual_seed(99)
    with torch.no_grad():
        s_logits, s_codes = rq.sample(conds, top_k=None, top_p=None, softmax_temperature=1.0, use_fp16=False)
    out.update(sample_logits=s_logits.numpy(), sample_codes=s_codes.numpy())
    path = os.path.join(OUT, "rq_tiny.npz")
    np.savez_compressed(path, **out)
    print("rq_tiny: loss", float(loss), "logits", tuple(logits.shape), "sampled", tuple(s_codes.shape), os.path.getsize(path), "bytes")


def rq_class(S):
    torch.manual_seed(77)
    rq = S.RQTransformer(**CLASS_CFG)
    perturb(rq)
    codes, conds = _inputs(CLASS_CFG, 2, 8)
    with torch.no_grad():
        logits = rq(codes, conds)
    out = {"sd." + k: v.numpy() for k, v in rq.state_dict().items()}
    out.update(codes=codes.numpy(), conds=conds.numpy(), logits=logits.numpy())
    out.update({"cfg." + k: np.int64(v) for k, v in CLASS_CFG.items()})
    path = os.path.join(OUT, "ref_rq_class.npz")
    np.savez_compressed(path, **out)
    print("ref_rq_class:", tuple(logits.shape), os.path.getsize(path), "bytes")


if __name__ == "__main__":
    torch.set_num_threads(4)
    if os.path.isdir(REF):
        tiny(load_reference_stage2())
    else:
        print(f"{REF!r} not present: rq_tiny.npz needs a reference checkout (B200VQ_REFERENCE)")
    vendored = os.path.join(HERE, "_ref", "enhancing_ref", "stage2_layers.py")
    if os.path.exists(vendored):
        rq_class(load_reference_stage2(vendored))
    else:
        print("oracle/_ref not built (oracle/build_ref.py): ref_rq_class.npz not written")
