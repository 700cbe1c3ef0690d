#!/usr/bin/env python
"""Stage-2 GPT timing on one GPU (development probe, not the bench): fwd+bwd tokens/s of a reduced-width GPT at config 5's
sequence geometry (1 class token + 1024 codes, 8192-entry vocabulary), CUDA events, per data path.

    python tools/stage2_probe.py [embed_dim] [n_layers] [batch]"""
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import enhancing_transformers_b200 as etb  # noqa: E402


def flops_per_token(C, L, T, V):
    """fwd FLOPs per token: 12 C^2 per block in the six C x C / C x 4C products (key, query, value, proj, p0, p1), causal
    attention 2 * 2 * (T / 2) * C, vocabulary head 2 C V"""
    return L * (2 * 12 * C * C + 2 * T * C) + 2 * C * V


def main():
    C = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
    L = int(sys.argv[2]) if len(sys.argv) > 2 else 8
    B = int(sys.argv[3]) if len(sys.argv) > 3 else 8
    cfg = dict(vocab_cond_size=1000, vocab_img_size=8192, embed_dim=C, cond_num_tokens=1, img_num_tokens=1024, n_heads=C // 64, n_layers=L)
    torch.manual_seed(0)
    model = etb.GPT(**cfg).cuda()
    codes = torch.randint(0, 8192, (B, 1024), device="cuda")
    conds = torch.randint(0, 1000, (B, 1), device="cuda")
    out = {"config": cfg, "batch": B}
    for mode in ("fp16", "tf32", "parity"):
        etb.set_precision(mode)
        def step():
            model.zero_grad(set_to_none=True)
            logits = model(codes, conds)
            F.cross_entropy(logits.view(-1, 8192), codes.view(-1)).backward()
        for _ in range(2):
            step()
        n0 = etb.ops.launch_count()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        iters = 2 if mode == "parity" else 5
        for _ in range(iters):
            step()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        tok = B * 1025
        out[mode] = {"ms_per_step": round(ms, 3), "tokens_per_s": round(tok / ms * 1e3, 1),
                     "model_tflops": round(3 * flops_per_token(C, L, 1025, 8192) * tok / ms / 1e9, 2),
                     "launches_per_step": (etb.ops.launch_count() - n0) // iters}
    etb.set_precision("fp16")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
