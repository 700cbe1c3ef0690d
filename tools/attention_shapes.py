"""Timing of the fp16 attention core (ops.attention_f16_fwd / ops.attention_f16_bwd) at the model's shapes, and, with
--step, a kernel-time breakdown of the base benchmark step.

Shapes (N = 1024 tokens = 256 x 256 images in 8 x 8 patches, head size 64): base (B 128, 12 heads), small (B 128,
8 heads), large decoder (B 32, 16 heads).  Per call: CUDA-event time over --iters launches after --warmup, on seeded fp16
inputs.  Reported beside it:
  - algorithmic TFLOP/s: forward 4 B h N^2 d (QK^T and PV), backward 8 B h N^2 d (the four products of its gradient);
  - executed TFLOP/s: the products the kernels run, 2 B h N^2 d each -- forward 2, backward 7 (key side: KQ^T, P^T dO,
    V dO^T, dS^T Q; query side: QK^T, dO V^T, dS K: the scores are recomputed on both sides instead of exchanged);
  - ex2/s: one exponential per score and pass (forward 1, backward 2);
  - the share of the binding bound: the larger of executed FLOP over 989 TFLOP/s (dense fp16, H100 SXM data sheet) and
    exponentials over 3.9 T/s (the MUFU ex2 rate the FlashAttention-3 paper gives for the H100 SXM), over the time.
The backward includes its delta = rowsum(dO * O) kernel.  The card's name, power limit and SM clock are read before and
after, in the same run.

--step runs torch.profiler (CUDA activities) over --steps steps of the base benchmark step (batch --batch, fp16 data
path, built as bench.py builds it) after three warm-up steps, sums kernel time into GEMM, attention (fwd, delta, dkv,
dq), LayerNorm, VQ and other, and writes the table and a Chrome trace under --out.

    python tools/attention_shapes.py [--json out.json]
    python tools/attention_shapes.py --step --out DIR
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
PEAK_EX2 = 3.9e12
SHAPES = [("base", 128, 12), ("small", 128, 8), ("large decoder", 32, 16)]
N, DH = 1024, 64


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"nvidia-smi unavailable ({e})"
    return {"query": q, "value": out, "torch_name": torch.cuda.get_device_name()}


def counts(B, heads):
    """(algorithmic flops, executed flops, exponentials) of the forward and the backward"""
    prod = 2.0 * B * heads * N * N * DH
    scores = float(B * heads * N * N)
    return {"fwd": (2 * prod, 2 * prod, scores), "bwd": (4 * prod, 7 * prod, 2 * scores)}


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def shapes_table(args):
    info = {"card": card(), "lib": etb._lib.LIB_PATH, "iters": args.iters, "rows": []}
    print(f"# {info['card']['query']}: {info['card']['value']}")
    print(f"# library {info['lib']}, N = {N}, head size {DH}, {args.iters} launches per call after {args.warmup} warm-up")
    print(f"{'shape':<15}{'call':<5}{'ms':>9}{'alg TF/s':>10}{'exec TF/s':>10}{'ex2 T/s':>9}{'of bound':>10}  bound")
    dev = "cuda"
    for name, B, heads in SHAPES:
        g = torch.Generator(device=dev).manual_seed(0)
        inner = heads * DH
        qkv = (torch.randn(B * N, 3 * inner, device=dev, generator=g) * 0.5).half()
        dout = (torch.randn(B * N, inner, device=dev, generator=g) * 2.0 ** -10).half()    # the scale the gradient travels at
        scale = DH ** -0.5
        o, lse = ops.attention_f16_fwd(qkv, B, N, heads, DH, scale)
        calls = {"fwd": lambda: ops.attention_f16_fwd(qkv, B, N, heads, DH, scale),
                 "bwd": lambda: ops.attention_f16_bwd(qkv, o, lse, dout, B, N, heads, DH, scale)}
        for call, fn in calls.items():
            ms = time_ms(fn, args.iters, args.warmup)
            alg, exe, ex2 = counts(B, heads)[call]
            t_mma, t_ex2 = exe / (PEAK_TFLOPS * 1e12) * 1e3, ex2 / PEAK_EX2 * 1e3
            bound = "tensor" if t_mma >= t_ex2 else "ex2"
            row = {"shape": name, "B": B, "heads": heads, "call": call, "ms": ms, "alg_tflops": alg / ms / 1e9,
                   "exec_tflops": exe / ms / 1e9, "ex2_per_s": ex2 / ms * 1e3, "frac_of_bound": max(t_mma, t_ex2) / ms,
                   "bound": bound}
            info["rows"].append(row)
            print(f"{name:<15}{call:<5}{ms:9.3f}{row['alg_tflops']:10.1f}{row['exec_tflops']:10.1f}"
                  f"{row['ex2_per_s'] / 1e12:9.2f}{row['frac_of_bound']:10.2f}  {bound}")
        del qkv, dout, o, lse
    info["card_after"] = card()
    print(f"# after: {info['card_after']['value']}")
    return info


def category(kernel):
    k = kernel.lower()
    if "attn" in k or "attention" in k:
        for part in ("delta", "dkv", "dq", "fwd"):
            if part in k:
                return "attention " + part
        return "attention other"
    if "gemm" in k or "splitk_reduce" in k or "colpart_reduce" in k:
        return "GEMM"
    if "ln_" in k or "layernorm" in k:
        return "LayerNorm"
    if "vq_" in k:
        return "VQ"
    return "other"


def step_breakdown(args):
    import torch.nn as nn
    from torch.profiler import ProfilerActivity, profile

    from enhancing_transformers_b200.configs import CONFIGS

    dev = torch.device("cuda", 0)
    cfg = CONFIGS["base"]

    class HotPath(nn.Module):
        """bench.py's step: encoder -> pre_quant -> quantizer -> post_quant (+ positional add) -> decoder -> loss"""

        def __init__(self):
            super().__init__()
            e, d, q = cfg["encoder"], cfg["decoder"], cfg["quantizer"]
            self.encoder = etb.ViTEncoder(cfg["image_size"], cfg["patch_size"], **e)
            self.decoder = etb.ViTDecoder(cfg["image_size"], cfg["patch_size"], **d)
            self.quantizer = etb.VectorQuantizer(**q)
            self.pre_quant = etb.QuantLinear(e["dim"], q["embed_dim"])
            self.post_quant = etb.QuantLinear(q["embed_dim"], d["dim"])
            etb.fuse_post_quant_pos(self)

        def forward(self, x):
            quant, qloss, _ = self.quantizer(self.pre_quant(self.encoder(x)))
            rec = self.decoder(self.post_quant(quant))
            return ((rec - x) ** 2).mean() + qloss

    torch.manual_seed(0)
    model = HotPath().to(dev)
    params = list(model.parameters())
    x = torch.rand(args.batch, 3, cfg["image_size"], cfg["image_size"], generator=torch.Generator().manual_seed(1234)).to(dev)

    def step():
        for p in params:
            p.grad = None
        model(x).backward()

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    info = {"card": card(), "lib": etb._lib.LIB_PATH, "batch": args.batch, "steps": args.steps}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
    info["card_after"] = card()
    os.makedirs(args.out, exist_ok=True)
    prof.export_chrome_trace(os.path.join(args.out, "step_trace.json"))
    sums = {}
    for ev in prof.key_averages():
        t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        if t <= 0:
            continue
        c = category(ev.key)
        sums[c] = sums.get(c, 0.0) + t / 1e3 / args.steps          # ms per step
    total = sum(sums.values())
    order = ["GEMM", "attention fwd", "attention delta", "attention dkv", "attention dq", "attention other", "LayerNorm",
             "VQ", "other"]
    info["ms_per_step"] = {c: sums.get(c, 0.0) for c in order}
    info["kernel_ms_per_step"] = total
    print(f"# {info['card']['query']}: {info['card']['value']}")
    print(f"# library {info['lib']}, base config, batch {args.batch}, {args.steps} profiled steps")
    print(f"{'category':<18}{'ms/step':>9}{'share':>8}")
    for c in order:
        print(f"{c:<18}{sums.get(c, 0.0):9.2f}{sums.get(c, 0.0) / total:8.1%}")
    att = sum(v for c, v in sums.items() if c.startswith("attention"))
    print(f"{'attention, all':<18}{att:9.2f}{att / total:8.1%}")
    print(f"{'kernels, total':<18}{total:9.2f}")
    print(f"# after: {info['card_after']['value']}")
    return info


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--step", action="store_true", help="profile base benchmark steps instead of timing the shapes")
    ap.add_argument("--steps", type=int, default=2, help="--step: profiled steps")
    ap.add_argument("--batch", type=int, default=128, help="--step: images per step")
    ap.add_argument("--out", default="attention_step", help="--step: directory for the table and the trace")
    ap.add_argument("--json", default=None, help="also write the table as JSON here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "attention_shapes.py times the attention core on a CUDA device"
    if args.iters < 20:
        ap.error("--iters must be at least 20")
    info = step_breakdown(args) if args.step else shapes_table(args)
    if args.step:
        with open(os.path.join(args.out, "step_breakdown.json"), "w") as fh:
            json.dump(info, fh, indent=1)
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(info, fh, indent=1)


if __name__ == "__main__":
    main()
