"""Timing of the two backward paths that scatter rows by id: the default one (float atomics) and the opt-in deterministic
one (stable radix sort by id + fixed-order segmented sum, scatter_det.cu).

Shapes:
  - VQ backward (ops.vq_bwd vs ops.vq_bwd_deterministic): M = 131 072 tokens (base, batch 128), 8192 codes, D = 32,
    depth 1 and 4, three kinds of z: uniform (randn), clustered (45 codebook rows + 0.01 randn, as in bench.py's VQ
    block) and one code (every token on codebook row 0 + 0.01 randn: a single id collects all M contributions at depth 1);
  - stage-2 token-embedding backward (ops.token_embed_bwd vs ops.token_embed_bwd_deterministic): B 4, 1 + 1024 tokens,
    C 1024, condition vocabulary 1000, code vocabulary 8192, random ids and all ids equal.
Per call: CUDA-event time over --iters launches after --warmup, on seeded inputs.  The card's name, power limit and SM
clock are read in the same run.

    python tools/scatter_shapes.py [--json out.json]
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


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"nvidia-smi unavailable ({e})"
    return {"query": q, "value": out, "torch_name": torch.cuda.get_device_name()}


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


def vq_cases():
    M, K, D = 131072, 8192, 32
    g = torch.Generator(device="cuda").manual_seed(0)
    E = torch.randn(K, D, device="cuda", generator=g)
    zs = {"uniform": torch.randn(M, D, device="cuda", generator=g),
          "clustered": (E[torch.randint(0, 45, (M,), device="cuda", generator=g)]
                        + 0.01 * torch.randn(M, D, device="cuda", generator=g)).contiguous(),
          "one code": (E[torch.zeros(M, dtype=torch.int64, device="cuda")]
                       + 0.01 * torch.randn(M, D, device="cuda", generator=g)).contiguous()}
    g_out, g_loss = torch.randn(M, D, device="cuda", generator=g), torch.ones((), device="cuda")
    for depth in (1, 4):
        for kind, z in zs.items():
            _, _, idx = ops.vq_fwd(z, E, depth, 0.25)
            args = (z, E, idx, g_out, g_loss, depth > 1, 0.25)
            yield (f"vq depth {depth}, {kind}", int(idx[:, 0].unique().numel()),
                   lambda a=args: ops.vq_bwd(*a), lambda a=args: ops.vq_bwd_deterministic(*a))


def token_cases():
    B, Tc, Ti, C, Vc, Vi = 4, 1, 1024, 1024, 1000, 8192
    g = torch.Generator(device="cuda").manual_seed(0)
    grad = torch.randn(B * (Tc + Ti), C, device="cuda", generator=g)
    ids = {"random": (torch.randint(0, Vc, (B, Tc), device="cuda", generator=g), torch.randint(0, Vi, (B, Ti), device="cuda", generator=g)),
           "equal": (torch.full((B, Tc), 7, dtype=torch.int64, device="cuda"), torch.full((B, Ti), 11, dtype=torch.int64, device="cuda"))}
    for kind, (conds, codes) in ids.items():
        args = (conds, codes, grad, Vc, Vi)
        yield (f"token embed, {kind} ids", int(codes.unique().numel()),
               lambda a=args: ops.token_embed_bwd(*a), lambda a=args: ops.token_embed_bwd_deterministic(*a))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("scatter_shapes.py times CUDA kernels and needs a GPU")
    info = {"card_before": card(), "lib": etb._lib.LIB_PATH, "iters": args.iters, "rows": []}
    print(f"# {info['card_before']['query']}: {info['card_before']['value']}")
    print(f"# library {info['lib']}, {args.iters} launches per call after {args.warmup} warm-up")
    print(f"{'case':<32}{'ids hit':>9}{'atomic ms':>11}{'determ. ms':>12}{'ratio':>8}")
    for name, hit, atomic, det in list(vq_cases()) + list(token_cases()):
        ms_a = time_ms(atomic, args.iters, args.warmup)
        ms_d = time_ms(det, args.iters, args.warmup)
        info["rows"].append(dict(case=name, ids_hit=hit, atomic_ms=ms_a, deterministic_ms=ms_d))
        print(f"{name:<32}{hit:>9}{ms_a:>11.3f}{ms_d:>12.3f}{ms_d / ms_a:>8.2f}", flush=True)
    info["card_after"] = card()
    print(f"# after: {info['card_after']['value']}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
