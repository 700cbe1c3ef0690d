#!/usr/bin/env python
"""Throughput of the stage-2 RQTransformer prior (reference stage2/layers.py:306-547) on one GPU.

    python tools/rq_probe.py [--batch 16] [--steps 10] [--trace FILE.json]

Prints, as JSON lines:
  - forward + backward tokens/s (B * T code positions per second) per data path, at C 1024, 8 spatial + 4 depth layers, D 4,
    T 1024, vocab 8192 (device events around `steps` steps after warm-up);
  - a torch.profiler split of one fp16 step's kernel time: GEMM, spatial attention, depth attention, embeddings, LayerNorm, other;
  - the short-attention kernels' call time against their HBM bound (bytes from the shapes over 3.35 TB/s, NVIDIA's H100 SXM
    data-sheet figure -- a bound, not a measurement);
  - seconds per sampled batch at a small config;
  - the card's name, power limit and SM clock, read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import enhancing_transformers_b200 as etb  # noqa: E402
from enhancing_transformers_b200 import ops  # noqa: E402

HBM = 3.35e12
CFG = dict(vocab_cond_size=1000, vocab_img_size=8192, embed_dim=1024, cond_num_tokens=1, img_num_tokens=1024, depth_num_tokens=4,
           spatial_n_heads=16, depth_n_heads=16, spatial_n_layers=8, depth_n_layers=4)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def timed(fn, steps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / 1e3 / steps


def kind(name):
    n = name.lower()
    if "short_attention" in n:
        return "depth attention"
    if "attn_" in n or "attention" in n:
        return "spatial attention"
    if "gemm" in n or "splitk" in n:
        return "GEMM"
    if "embed" in n or "scan" in n or "scatter" in n or "compact_ids" in n or "colsum_fixed" in n:
        return "embeddings"
    if "ln_" in n or "layernorm" in n:
        return "LayerNorm"
    return "other"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--trace", default=None, help="also write the profiled step's Chrome trace here")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "rq_probe needs a GPU"
    print(json.dumps({"card": card()}))
    B, T, D, S = a.batch, CFG["img_num_tokens"], CFG["depth_num_tokens"], CFG["vocab_img_size"]
    torch.manual_seed(0)
    model = etb.RQTransformer(**CFG).cuda()
    codes = torch.randint(0, S, (B, T, D), device="cuda")
    conds = torch.randint(0, 1000, (B, 1), device="cuda")

    def step():
        model.zero_grad(set_to_none=True)
        F.cross_entropy(model(codes, conds).view(-1, S), codes.view(-1)).backward()

    for mode in ("fp16", "tf32", "parity"):
        etb.set_precision(mode)
        torch.cuda.reset_peak_memory_stats()
        timed(step, 2)
        s = timed(step, a.steps)
        print(json.dumps({"mode": mode, "batch": B, "step_s": round(s, 4), "tokens_per_s": round(B * T / s, 1),
                          "peak_mem_GB": round(torch.cuda.max_memory_allocated() / 1e9, 2)}))
    etb.set_precision("fp16")

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    split = {}
    for ev in prof.key_averages():
        split[kind(ev.key)] = split.get(kind(ev.key), 0.0) + ev.device_time_total / 1e3
    print(json.dumps({"profile_ms_per_step": {k: round(v, 2) for k, v in sorted(split.items())}, "card": card()}))
    if a.trace:
        prof.export_chrome_trace(a.trace)

    C, heads, hs = CFG["embed_dim"], CFG["depth_n_heads"], CFG["embed_dim"] // CFG["depth_n_heads"]
    nseq = B * T
    qkv = torch.randn(nseq * D, 3 * C, device="cuda")
    dout = torch.randn(nseq * D, C, device="cuda")
    fwd = timed(lambda: ops.short_attention_fwd(qkv, nseq, D, heads, hs, hs ** -0.5), 3)
    fwd = timed(lambda: ops.short_attention_fwd(qkv, nseq, D, heads, hs, hs ** -0.5), 20)
    bwd = timed(lambda: ops.short_attention_bwd(qkv, dout, nseq, D, heads, hs, hs ** -0.5), 3)
    bwd = timed(lambda: ops.short_attention_bwd(qkv, dout, nseq, D, heads, hs, hs ** -0.5), 20)
    fb, bb = nseq * D * 4 * C * 4, nseq * D * 7 * C * 4            # fwd: qkv (3C) + o (C); bwd: qkv (3C) + dO (C) + dqkv (3C)
    print(json.dumps({"short_attention": {"nseq": nseq, "D": D, "heads": heads, "hs": hs,
                                          "fwd_ms": round(fwd * 1e3, 3), "fwd_GB": round(fb / 1e9, 3),
                                          "fwd_hbm_bound_ms": round(fb / HBM * 1e3, 3), "fwd_share_of_bound": round(fb / HBM / fwd, 3),
                                          "bwd_ms": round(bwd * 1e3, 3), "bwd_GB": round(bb / 1e9, 3),
                                          "bwd_hbm_bound_ms": round(bb / HBM * 1e3, 3), "bwd_share_of_bound": round(bb / HBM / bwd, 3),
                                          "bound": "bytes / 3.35 TB/s (H100 SXM data sheet)"}, "card": card()}))

    small = dict(CFG, embed_dim=256, spatial_n_heads=4, depth_n_heads=4, spatial_n_layers=4, depth_n_layers=2, img_num_tokens=256)
    sm = etb.RQTransformer(**small).cuda().eval()
    sc = torch.randint(0, 1000, (8, 1), device="cuda")
    sm.sample(sc[:, :1], top_k=100)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sm.sample(sc, top_k=100)
    torch.cuda.synchronize()
    print(json.dumps({"sample": {"batch": 8, "T": 256, "D": 4, "C": 256, "layers": "4+2", "s_per_batch": round(time.perf_counter() - t0, 3)},
                      "card": card()}))


if __name__ == "__main__":
    main()
