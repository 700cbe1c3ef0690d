#!/usr/bin/env python
"""Cost of the EMA codebook (EMAVectorQuantizer) on one GPU.

    python tools/ema_probe.py [--steps 6]

Prints, as JSON lines:
  - the card's name, power limit and SM clock, read in the same run;
  - the VQ lookup at M 131072, K 8192, D 32, depth 1 and 4, uniform and clustered z (bench.py's VQ block: 45 codes + 0.01
    noise): vq_fwd, and vq_fwd_ema with statistics off, atomic and deterministic.  CUDA events over 30 launches after
    warm-up, a 160 MB buffer written before each launch so that L2 starts cold, as bench.py's VQ block does;
  - the update kernel (vq_ema_update) at K 8192;
  - the base training step (bench.py's base config, batch 128, fwd + bwd + the flat-gradient step) with EMAVectorQuantizer
    against VectorQuantizer in images/s, the two alternated in one session."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import enhancing_transformers_b200 as etb  # noqa: E402
from enhancing_transformers_b200 import ops  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def timed_cold(fn, flush, iters=30):
    for _ in range(3):
        fn()
    tot = 0.0
    for _ in range(iters):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        tot += s.elapsed_time(e)
    return tot / iters


def lookup(dev):
    M, K, D = 131072, 8192, 32
    g = torch.Generator().manual_seed(0)
    E = torch.randn(K, D, generator=g).to(dev)
    zs = {"uniform": torch.randn(M, D, generator=g).to(dev),
          "clustered": (E[torch.randint(0, 45, (M,), generator=g).to(dev)] + 0.01 * torch.randn(M, D, generator=g).to(dev)).contiguous()}
    flush = torch.empty(160 * 2 ** 20 // 4, device=dev)
    for kind, z in zs.items():
        for depth in (1, 4):
            row = dict(what="lookup", z=kind, depth=depth, tokens=M, n_embed=K)
            row["vq_fwd_ms"] = timed_cold(lambda: ops.vq_fwd(z, E, depth, 0.25), flush)
            row["ema_stats_off_ms"] = timed_cold(lambda: ops.vq_fwd_ema(z, E, depth, 0.25, True, False), flush)
            row["ema_atomic_ms"] = timed_cold(lambda: ops.vq_fwd_ema(z, E, depth, 0.25, True, True, False), flush)
            row["ema_deterministic_ms"] = timed_cold(lambda: ops.vq_fwd_ema(z, E, depth, 0.25, True, True, True), flush)
            print(json.dumps(row), flush=True)
    _, _, _, buf = ops.vq_fwd_ema(zs["clustered"], E, 1, 0.25)
    cs, ea, w = torch.zeros(K, device=dev), E.clone(), E.clone()
    ms = timed_cold(lambda: ops.vq_ema_update(buf, cs, ea, w, 0.99, 1e-5), flush)
    print(json.dumps(dict(what="update", n_embed=K, ms=ms)), flush=True)


def step_rate(dev, steps):
    from enhancing_transformers_b200.configs import CONFIGS
    cfg = CONFIGS["base"]
    e, d, q = cfg["encoder"], cfg["decoder"], cfg["quantizer"]
    batch = 128

    def build(cls):
        torch.manual_seed(0)
        mods = torch.nn.ModuleDict(dict(
            encoder=etb.ViTEncoder(cfg["image_size"], cfg["patch_size"], **e),
            decoder=etb.ViTDecoder(cfg["image_size"], cfg["patch_size"], **d),
            quantizer=cls(**q), pre_quant=etb.QuantLinear(e["dim"], q["embed_dim"]),
            post_quant=etb.QuantLinear(q["embed_dim"], d["dim"]))).to(dev)
        etb.fuse_post_quant_pos(mods)
        fg = etb.FlatGradients(mods.parameters())
        opt = torch.optim.AdamW(fg.params, lr=1e-4)
        return mods, fg, opt

    imgs = torch.rand(batch, 3, cfg["image_size"], cfg["image_size"], generator=torch.Generator().manual_seed(1)).to(dev)
    runs = {}
    for name, cls in (("VectorQuantizer", etb.VectorQuantizer), ("EMAVectorQuantizer", etb.EMAVectorQuantizer)):
        runs[name] = build(cls)

    def step(mods, fg, opt):
        fg.zero_()
        zq, qloss, _ = mods["quantizer"](mods["pre_quant"](mods["encoder"](imgs)))
        loss = ((mods["decoder"](mods["post_quant"](zq)) - imgs) ** 2).mean() + qloss
        loss.backward()
        opt.step()

    for r in runs.values():
        for _ in range(3):
            step(*r)
    torch.cuda.synchronize()
    rates = {k: [] for k in runs}
    for _ in range(3):                       # alternated
        for name, r in runs.items():
            s, e_ = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(steps):
                step(*r)
            e_.record()
            torch.cuda.synchronize()
            rates[name].append(batch * steps / (s.elapsed_time(e_) / 1e3))
    print(json.dumps(dict(what="base_step", batch=batch, steps_per_run=steps, images_per_s=rates)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=6)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ema_probe needs a CUDA device")
    dev = torch.device("cuda", 0)
    print(json.dumps(dict(what="card", card=card(), precision=etb.get_precision())), flush=True)
    lookup(dev)
    step_rate(dev, args.steps)
    print(json.dumps(dict(what="card_after", card=card())), flush=True)


if __name__ == "__main__":
    main()
