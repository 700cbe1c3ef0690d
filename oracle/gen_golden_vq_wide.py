"""Generate tests/golden/vq_wide.npz: the reference's unmodified VectorQuantizer at code widths above 32.

Needs a checkout of the reference (B200VQ_REFERENCE); its quantizers.py is imported by file path, as gen_golden.py
does.  Only its outputs are stored.

    python oracle/gen_golden_vq_wide.py

Cases, at D in {64, 96, 256}: the plain quantiser, residual depth 4, and use_norm=False; plus one clustered case (many
tokens on a few codes) at D = 256.  tests/test_vq_wide.py pins the oracle against the fixture and
tests/test_gpu_vq_wide.py the kernels.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import vitvq_oracle as O  # noqa: E402
from oracle.gen_golden import OUT, REF, load_reference  # noqa: E402

CASES = [(f"d{D}.{tag}", D, kw) for D in (64, 96, 256)
         for tag, kw in (("plain", {}), ("res4", dict(use_residual=True, num_quantizers=4)), ("nonorm", dict(use_norm=False)))]


def gen_vq_wide(Q):
    out = {}
    for i, (tag, D, kw) in enumerate(CASES):
        torch.manual_seed(100 + i)
        vq = Q.VectorQuantizer(embed_dim=D, n_embed=320, beta=0.25, **kw)
        z = torch.randn(2, 24, D, requires_grad=True)
        zq, loss, idx = vq(z)
        g_out = torch.randn_like(zq)
        g_loss = 0.7
        (zq * g_out).sum().add(loss * g_loss).backward()
        out.update({f"{tag}.E": vq.embedding.weight.detach().numpy(), f"{tag}.z": z.detach().numpy(),
                    f"{tag}.zq": zq.detach().numpy(), f"{tag}.loss": loss.detach().numpy(), f"{tag}.idx": idx.numpy(),
                    f"{tag}.g_out": g_out.numpy(), f"{tag}.g_loss": np.float32(g_loss),
                    f"{tag}.gz": z.grad.numpy(), f"{tag}.gE": vq.embedding.weight.grad.numpy()})
        print("vq_wide", tag, "loss", float(loss), "distinct codes", idx.unique().numel())
    torch.manual_seed(11)
    vq = Q.VectorQuantizer(embed_dim=256, n_embed=320)
    z = (torch.randn(1, 1, 256) + 0.01 * torch.randn(2, 32, 256)).requires_grad_(True)
    zq, loss, idx = vq(z)
    g_out = torch.zeros_like(zq)
    loss.backward()
    out.update({"d256.clustered.E": vq.embedding.weight.detach().numpy(), "d256.clustered.z": z.detach().numpy(),
                "d256.clustered.zq": zq.detach().numpy(), "d256.clustered.loss": loss.detach().numpy(),
                "d256.clustered.idx": idx.numpy(), "d256.clustered.g_out": g_out.numpy(),
                "d256.clustered.g_loss": np.float32(1.0), "d256.clustered.gz": z.grad.numpy(),
                "d256.clustered.gE": vq.embedding.weight.grad.numpy()})
    print("vq_wide d256.clustered distinct codes", idx.unique().numel())
    O.save_golden(os.path.join(OUT, "vq_wide.npz"), out)


if __name__ == "__main__":
    if not os.path.isdir(REF):
        sys.exit(f"{REF} not present: golden vectors need a reference checkout (B200VQ_REFERENCE)")
    torch.set_num_threads(4)
    _, Q = load_reference()
    gen_vq_wide(Q)
    for f in sorted(os.listdir(OUT)):
        if f.startswith("vq_wide"):
            print(f, os.path.getsize(os.path.join(OUT, f)))
