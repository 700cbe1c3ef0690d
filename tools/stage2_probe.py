#!/usr/bin/env python
"""Stage-2 GPT timing on one GPU (development probe, not the bench): fwd+bwd tokens/s of a reduced-depth GPT at config 5's
sequence geometry (1 class token + 1024 codes, 8192-entry vocabulary), CUDA events, per data path.

    python tools/stage2_probe.py [embed_dim] [n_layers] [batch] [head_size] [--attn-profile]

head_size (default 64) sets n_heads = embed_dim // head_size.  --attn-profile adds, per data path, the attention kernels' own
CUDA time per step (forward, key-side and query-side backward, delta) from torch.profiler, in a separate profiled run after the
timed one.  At a fixed embed_dim every head size has the same attention FLOPs, so two head sizes compare like for like."""
import argparse
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


def attention_kernel_ms(step, iters):
    """CUDA time per step of every kernel whose name starts with attn_ (the stage-2 attention core), by kernel"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            step()
        torch.cuda.synchronize()
    per = {}
    for ev in prof.key_averages():
        name = ev.key.split("<")[0].split("(")[0].replace("void ", "").replace("b200::", "")
        if name.startswith("attn_"):
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            per[name] = per.get(name, 0.0) + t / 1e3 / iters
    return {"total": round(sum(per.values()), 3), **{k: round(v, 3) for k, v in sorted(per.items())}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("embed_dim", nargs="?", type=int, default=1024)
    ap.add_argument("n_layers", nargs="?", type=int, default=8)
    ap.add_argument("batch", nargs="?", type=int, default=8)
    ap.add_argument("head_size", nargs="?", type=int, default=64)
    ap.add_argument("--attn-profile", action="store_true")
    a = ap.parse_args()
    C, L, B, hs = a.embed_dim, a.n_layers, a.batch, a.head_size
    cfg = dict(vocab_cond_size=1000, vocab_img_size=8192, embed_dim=C, cond_num_tokens=1, img_num_tokens=1024, n_heads=C // hs, n_layers=L)
    torch.manual_seed(0)
    model = etb.GPT(**cfg).cuda()
    codes = torch.randint(0, 8192, (B, 1024), device="cuda")
    conds = torch.randint(0, 1000, (B, 1), device="cuda")
    out = {"config": cfg, "batch": B, "head_size": hs, "device": torch.cuda.get_device_name()}
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
        if a.attn_profile:
            out[mode]["attention_ms_per_step"] = attention_kernel_ms(step, 2)
    etb.set_precision("fp16")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
