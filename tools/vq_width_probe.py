#!/usr/bin/env python
"""Cost of the quantiser against its code width on one GPU.

    python tools/vq_width_probe.py [--steps 4] [--widths 32,64,128,256]

Prints, as JSON lines:
  - the card's name, power limit and SM clock, read in the same run;
  - at M 131072, K 8192 and 16384, D 32 / 64 / 128 / 256, depth 1 and 4: vq_fwd, the EMA lookup (vq_fwd_ema with atomic and
    with deterministic statistics) and both backwards (vq_bwd, vq_bwd_deterministic).  CUDA events over 30 launches after
    warm-up, a 160 MB buffer written before each launch so that L2 starts cold (the method of tools/ema_probe.py).  The
    lookup's rate counts 2 * D * K FLOP per token and depth, against the 67 TFLOP/s fp32 figure of the H100 SXM data sheet;
  - the base training step (batch 128, fwd + bwd + AdamW on flat gradients) with residual depth 4 at D 256, K 16384 next to
    the same step at D 32, K 16384, alternated in one session."""
import argparse
import copy
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import enhancing_transformers_b200 as etb  # noqa: E402
from enhancing_transformers_b200 import ops  # noqa: E402
from tools.ema_probe import card, timed_cold  # noqa: E402

FP32_PEAK = 67e12


def lookup(dev, widths):
    M = 131072
    flush = torch.empty(160 * 2 ** 20 // 4, device=dev)
    for D in widths:
        g = torch.Generator().manual_seed(D)
        z = torch.randn(M, D, generator=g).to(dev)
        for K in (8192, 16384):
            E = torch.randn(K, D, generator=g).to(dev)
            for depth in (1, 4):
                row = dict(what="lookup", D=D, n_embed=K, depth=depth, tokens=M)
                row["vq_fwd_ms"] = timed_cold(lambda: ops.vq_fwd(z, E, depth, 0.25), flush)
                row["ema_atomic_ms"] = timed_cold(lambda: ops.vq_fwd_ema(z, E, depth, 0.25, True, True, False), flush)
                row["ema_deterministic_ms"] = timed_cold(lambda: ops.vq_fwd_ema(z, E, depth, 0.25, True, True, True), flush)
                _, _, idx = ops.vq_fwd(z, E, depth, 0.25)
                g_out, g_loss = torch.randn_like(z), torch.tensor(1.0, device=dev)
                row["bwd_atomic_ms"] = timed_cold(lambda: ops.vq_bwd(z, E, idx, g_out, g_loss, depth > 1, 0.25), flush)
                row["bwd_deterministic_ms"] = timed_cold(lambda: ops.vq_bwd_deterministic(z, E, idx, g_out, g_loss, depth > 1, 0.25),
                                                         flush)
                flop = 2.0 * D * K * M * depth
                row["vq_fwd_tflops"] = flop / (row["vq_fwd_ms"] * 1e-3) / 1e12
                row["vq_fwd_share_of_fp32_peak"] = flop / (row["vq_fwd_ms"] * 1e-3) / FP32_PEAK
                print(json.dumps(row), flush=True)
                del idx, g_out
            del E
        del z


def step_rate(dev, steps):
    from enhancing_transformers_b200.configs import CONFIGS
    batch = 128
    imgs = None

    def build(D):
        cfg = copy.deepcopy(CONFIGS["base"])
        cfg["quantizer"].update(embed_dim=D, n_embed=16384, use_residual=True, num_quantizers=4)
        e, d, q = cfg["encoder"], cfg["decoder"], cfg["quantizer"]
        torch.manual_seed(0)
        mods = torch.nn.ModuleDict(dict(
            encoder=etb.ViTEncoder(cfg["image_size"], cfg["patch_size"], **e),
            decoder=etb.ViTDecoder(cfg["image_size"], cfg["patch_size"], **d),
            quantizer=etb.VectorQuantizer(**q), pre_quant=etb.QuantLinear(e["dim"], D),
            post_quant=etb.QuantLinear(D, d["dim"]))).to(dev)
        etb.fuse_post_quant_pos(mods)
        fg = etb.FlatGradients(mods.parameters())
        return mods, fg, torch.optim.AdamW(fg.params, lr=1e-4), cfg["image_size"]

    runs = {f"rq4_D{D}_K16384": build(D) for D in (32, 256)}
    size = next(iter(runs.values()))[3]
    imgs = torch.rand(batch, 3, size, size, generator=torch.Generator().manual_seed(1)).to(dev)

    def step(mods, fg, opt, _):
        fg.zero_()
        zq, qloss, _ = mods["quantizer"](mods["pre_quant"](mods["encoder"](imgs)))
        loss = ((mods["decoder"](mods["post_quant"](zq)) - imgs) ** 2).mean() + qloss
        loss.backward()
        opt.step()

    for r in runs.values():
        for _ in range(3):
            step(*r)
    torch.cuda.synchronize()
    ms = {k: [] for k in runs}
    for _ in range(3):                       # alternated
        for name, r in runs.items():
            s, e_ = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(steps):
                step(*r)
            e_.record()
            torch.cuda.synchronize()
            ms[name].append(s.elapsed_time(e_) / steps)
    print(json.dumps(dict(what="base_step", batch=batch, steps_per_run=steps, ms_per_step=ms,
                          images_per_s={k: [batch / (t / 1e3) for t in v] for k, v in ms.items()})), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--widths", default="32,64,128,256")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vq_width_probe needs a CUDA device")
    dev = torch.device("cuda", 0)
    print(json.dumps(dict(what="card", card=card(), precision=etb.get_precision())), flush=True)
    lookup(dev, [int(w) for w in args.widths.split(",")])
    step_rate(dev, args.steps)
    print(json.dumps(dict(what="card_after", card=card())), flush=True)


if __name__ == "__main__":
    main()
