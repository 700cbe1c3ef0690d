"""Per-shape timing of the fp16 GEMMs of one transformer block of the base config (D = 768, mlp = 3072, 12 x 64 heads)
at M = 131 072 tokens (batch 128 of 256 x 256 images, 8 x 8 patches): the twelve products of functional.py's fp16 block
forward and backward, each through ops.gemm with its real epilogue, alpha and split count.

Per shape: CUDA-event time over --iters launches after --warmup, TFLOP/s, GB/s of the algorithmic traffic (operands,
epilogue input, output), and the larger of the two bounds (989 TFLOP/s dense f16, 3.35 TB/s HBM3: H100 SXM data
sheet) over the measured time, naming the bound that binds.  The card's name, power limit and SM clock are read in the
same run.  A wgrad with splits > 1 is timed without its split-K reduction (ops.splitk_reduce, a separate kernel).

    python tools/gemm_shapes.py [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import enhancing_transformers_b200 as etb  # noqa: E402

ops = etb.ops
PEAK_TFLOPS = 989.0
PEAK_GBS = 3350.0


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"nvidia-smi unavailable ({e})"
    return {"query": q, "value": out, "torch_name": torch.cuda.get_device_name()}


def shapes(M, D=768, mlp=3072, inner=768):
    """(name, thunk, flops, bytes) of every fp16 GEMM of one block; operands are seeded random, activations fp16"""
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)

    def h(*s, scale=1.0):
        return (torch.randn(*s, device=dev, generator=g) * scale).half()

    def f(*s):
        return torch.randn(*s, device=dev, generator=g)

    x, h1, h2, o = f(M, D), h(M, D), h(M, D), h(M, inner)
    t = torch.tanh(f(M, mlp)).half()
    wq, wo, w1, w2 = h(3 * inner, D, scale=0.03), h(D, inner, scale=0.03), h(mlp, D, scale=0.03), h(D, mlp, scale=0.03)
    bo, b1, b2 = f(D), f(mlp), f(D)
    x1 = f(M, D)
    gh, dt, g1h, dqkv = h(M, D), h(M, mlp), h(M, D), h(M, 3 * inner)
    inv = torch.tensor([1.0 / 64], device=dev)
    out = []

    def add(name, fn, n, k, in_bytes, out_bytes):
        out.append((name, fn, 2.0 * M * n * k, 2.0 * (M * k + n * k) + in_bytes + out_bytes))

    add("qkv fwd", lambda: ops.gemm(h1, wq, M, 3 * inner, D, out_half=True), 3 * inner, D, 0, 2 * M * 3 * inner)
    add("out-proj fwd", lambda: ops.gemm(o, wo, M, D, inner, bias=bo, res=x), D, inner, 4 * M * D, 4 * M * D)
    add("fc1 fwd", lambda: ops.gemm(h2, w1, M, mlp, D, bias=b1, act=1, out_half=True), mlp, D, 0, 2 * M * mlp)
    add("fc2 fwd", lambda: ops.gemm(t, w2, M, D, mlp, bias=b2, res=x1), D, mlp, 4 * M * D, 4 * M * D)
    add("dt dgrad", lambda: ops.gemm(gh, w2, M, mlp, D, b_major=1, aux=t, out_half=True, want_colsum=True), mlp, D,
        2 * M * mlp, 2 * M * mlp)
    add("dh2 dgrad", lambda: ops.gemm(dt, w1, M, D, mlp, b_major=1, out_half=True), D, mlp, 0, 2 * M * D)
    add("do dgrad", lambda: ops.gemm(g1h, wo, M, inner, D, b_major=1, out_half=True), inner, D, 0, 2 * M * inner)
    add("dh1 dgrad", lambda: ops.gemm(dqkv, wq, M, D, 3 * inner, b_major=1, out_half=True), D, 3 * inner, 0, 2 * M * D)
    for name, dy, xx, rows, cols in [("qkv wgrad", dqkv, h1, 3 * inner, D), ("out-proj wgrad", gh, o, D, inner),
                                     ("fc1 wgrad", dt, h2, mlp, D), ("fc2 wgrad", gh, t, D, mlp)]:
        s = ops.pick_splits(M, rows, cols, k_atom=64)
        if s == 1:
            fn = (lambda dy=dy, xx=xx, rows=rows, cols=cols: ops.gemm(dy, xx, rows, cols, M, a_major=1, b_major=1, alpha=inv))
        else:
            fn = (lambda dy=dy, xx=xx, rows=rows, cols=cols, s=s:
                  ops.gemm(dy, xx, rows, cols, M // s, a_major=1, b_major=1, splits=s))
        out.append((f"{name} (splits {s})", fn, 2.0 * M * rows * cols, 2.0 * M * (rows + cols) + 4.0 * s * rows * cols))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--tokens", type=int, default=131072)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the table as JSON here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "gemm_shapes.py times the GEMMs on a CUDA device"
    if args.iters < 20:
        ap.error("--iters must be at least 20")
    info = {"card": card(), "lib": etb._lib.LIB_PATH, "tokens": args.tokens, "iters": args.iters, "rows": []}
    print(f"# {info['card']['query']}: {info['card']['value']}")
    print(f"# library {info['lib']}, M = {args.tokens}, {args.iters} launches per shape after {args.warmup} warm-up")
    print(f"{'GEMM':<26}{'ms':>9}{'TFLOP/s':>9}{'GB/s':>8}{'of bound':>10}  bound")
    tot_ms = tot_flops = 0.0
    for name, fn, flops, nbytes in shapes(args.tokens):
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.iters
        t_flop, t_byte = flops / (PEAK_TFLOPS * 1e12) * 1e3, nbytes / (PEAK_GBS * 1e9) * 1e3
        bound = "tensor" if t_flop >= t_byte else "HBM"
        row = {"gemm": name, "ms": ms, "tflops": flops / ms / 1e9, "gbs": nbytes / ms / 1e6,
               "frac_of_bound": max(t_flop, t_byte) / ms, "bound": bound}
        info["rows"].append(row)
        tot_ms += ms
        tot_flops += flops
        print(f"{name:<26}{ms:9.3f}{row['tflops']:9.1f}{row['gbs']:8.0f}{row['frac_of_bound']:10.2f}  {bound}")
    info["total_ms"], info["total_tflops"] = tot_ms, tot_flops / tot_ms / 1e9
    print(f"{'total':<26}{tot_ms:9.3f}{info['total_tflops']:9.1f}")
    info["card_after"] = card()
    print(f"# after: {info['card_after']['value']}")
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(info, fh, indent=1)


if __name__ == "__main__":
    main()
