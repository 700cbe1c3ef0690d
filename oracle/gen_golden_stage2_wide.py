"""Generate tests/golden/ref_stage2_wide.npz by running the UNMODIFIED reference stage-2 classes (the copy oracle/build_ref.py
vendors into oracle/_ref) at head sizes 96 and 128, on the CPU:

    gpt96   GPT, embed_dim 192 with 2 heads (96 wide)
    gpt128  GPT, embed_dim 256 with 2 heads (128 wide)
    rq      RQTransformer, embed_dim 384: 3 spatial heads (128 wide) and 4 depth heads (96 wide)

Per case: the forward logits and cross-entropy loss, every parameter gradient, the logits of the sampling steps (the reference's
own sample() under torch.manual_seed(99), with the codes it drew) and a seeded top-k / nucleus draw.  The state dicts are not
stored: they come from a seeded construction plus `perturb` (oracle/gen_golden_gpt.py), which the tests repeat with this
package's classes and check against the stored sha256 digests (as rq_tiny.npz does).  The weight matrices of these widths hold
up to 590 k entries each, so a gradient of more than GRAD_FULL entries is stored at GRAD_SAMPLE seeded positions (sorted flat
indices `grad_idx.<name>`); a relative l2 error over such a sample estimates the full one to a few per cent.  No reference source
is copied; only outputs are stored.

    python oracle/build_ref.py && python oracle/gen_golden_stage2_wide.py
"""
import os
import sys
import zlib

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle.gen_golden_gpt import load_reference_stage2, perturb  # noqa: E402
from oracle.gen_golden_rq import sd_digest  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden", "ref_stage2_wide.npz")
GRAD_FULL = 1024
GRAD_SAMPLE = 384

CASES = {
    "gpt96": ("GPT", 11, dict(vocab_cond_size=10, vocab_img_size=64, embed_dim=192, cond_num_tokens=2, img_num_tokens=10,
                              n_heads=2, n_layers=2)),
    "gpt128": ("GPT", 12, dict(vocab_cond_size=7, vocab_img_size=64, embed_dim=256, cond_num_tokens=3, img_num_tokens=9,
                               n_heads=2, n_layers=1, mlp_bias=False, attn_bias=False)),
    "rq": ("RQTransformer", 14, dict(vocab_cond_size=10, vocab_img_size=64, embed_dim=384, cond_num_tokens=2, img_num_tokens=5,
                                     depth_num_tokens=3, spatial_n_heads=3, depth_n_heads=4, spatial_n_layers=1, depth_n_layers=1)),
}
BATCH = 2
DRAW = dict(top_k=7, top_p=0.9, softmax_temperature=0.8)


def grad_positions(name, numel):
    """the flat positions stored for a gradient of `numel` entries (all of them up to GRAD_FULL)"""
    if numel <= GRAD_FULL:
        return None
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    return torch.randperm(numel, generator=g)[:GRAD_SAMPLE].sort().values.numpy().astype(np.int64)


def inputs(kind, cfg, seed):
    g = torch.Generator().manual_seed(seed)
    shape = (BATCH, cfg["img_num_tokens"]) + ((cfg["depth_num_tokens"],) if kind == "RQTransformer" else ())
    codes = torch.randint(0, cfg["vocab_img_size"], shape, generator=g)
    conds = torch.randint(0, cfg["vocab_cond_size"], (BATCH, cfg["cond_num_tokens"]), generator=g)
    return codes, conds


def case(S, name, kind, seed, cfg):
    torch.manual_seed(seed)
    model = getattr(S, kind)(**cfg)
    init = sd_digest(model.state_dict())
    perturb(model)
    codes, conds = inputs(kind, cfg, seed + 100)
    logits = model(codes, conds)
    loss = F.cross_entropy(logits.reshape(-1, logits.shape[-1]), codes.reshape(-1))
    loss.backward()
    p = name + "."
    out = {p + "init_sha256": np.array(init), p + "sd_sha256": np.array(sd_digest(model.state_dict())), p + "seed": np.int64(seed),
           p + "codes": codes.numpy(), p + "conds": conds.numpy(), p + "logits": logits.detach().numpy(),
           p + "loss": loss.detach().numpy()}
    out.update({p + "cfg." + k: np.int64(v) for k, v in cfg.items()})
    for n, prm in model.named_parameters():
        flat = prm.grad.reshape(-1)
        idx = grad_positions(n, flat.numel())
        if idx is None:
            out[p + "grad." + n] = prm.grad.numpy()
        else:
            out[p + "grad_idx." + n] = idx
            out[p + "grad." + n] = flat[torch.from_numpy(idx)].numpy()
    model.eval()
    torch.manual_seed(99)
    with torch.no_grad():
        s_logits, s_codes = model.sample(conds, top_k=None, top_p=None, softmax_temperature=1.0, use_fp16=False)
    out.update({p + "sample_logits": s_logits.numpy(), p + "sample_codes": s_codes.numpy()})
    torch.manual_seed(123)
    with torch.no_grad():
        d_logits, d_codes = model.sample(conds, use_fp16=False, **DRAW)
    out.update({p + "draw_logits": d_logits.numpy(), p + "draw_codes": d_codes.numpy()})
    print(f"{name}: loss {loss.item():.6f}, logits {tuple(logits.shape)}, sampled {tuple(s_codes.shape)}")
    return out


def main() -> int:
    vendored = os.path.join(HERE, "_ref", "enhancing_ref", "stage2_layers.py")
    if not os.path.exists(vendored):
        sys.exit("oracle/_ref not built: run oracle/build_ref.py with a reference checkout first")
    S = load_reference_stage2(vendored)
    out = {}
    for name, (kind, seed, cfg) in CASES.items():
        out.update(case(S, name, kind, seed, cfg))
    np.savez_compressed(OUT, **out)
    print("ref_stage2_wide.npz:", os.path.getsize(OUT), "bytes")
    return 0


if __name__ == "__main__":
    torch.set_num_threads(4)
    sys.exit(main())
