"""Every epilogue form of the fp16 GEMM must give the same bits as the library it replaced: the epilogue loads its
inputs ahead of its stores, but each output element still goes through the same operations in the same order.  The
SHA-256 digests in tests/golden/gemm_epilogue_digests.json were written by this file run as a script
(`python tests/test_gpu_gemm_epilogue_bits.py > tests/golden/gemm_epilogue_digests.json`) with the library of commit
3bfcff0, whose epilogue loaded each element pair's inputs right before storing it, on an H100."""
import hashlib
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import enhancing_transformers_b200 as etb  # noqa: E402

ops = etb.ops
GOLDEN = os.path.join(ROOT, "tests", "golden", "gemm_epilogue_digests.json")
# the last row block is 104 rows; N = 648 is not a multiple of 64, 128 or 256.  An MN-major B (the dgrad form) needs
# N % 64 == 0: ND = 640 is two and a half 256-column tiles.
M, N, ND, K = 1000, 648, 640, 320


def _inputs():
    g = torch.Generator(device="cuda").manual_seed(11)

    def h(*s, scale=1.0):
        return (torch.randn(*s, device="cuda", generator=g) * scale).half()

    def f(*s):
        return torch.randn(*s, device="cuda", generator=g)

    return dict(a=h(M, K), w=h(N, K, scale=0.1), wt=h(K, ND, scale=0.1), bias=f(N), res=f(M, N), table=f(200, N),
                t=torch.tanh(f(M, ND)).half(), alpha=torch.tensor([1.0 / 64], device="cuda"),
                dy=h(640, 576), x=h(640, 448))


def cases():
    """name -> thunk returning the tensors whose bits are pinned"""
    d = _inputs()
    return {
        "fp16 out": lambda: [ops.gemm(d["a"], d["w"], M, N, K, out_half=True)],
        "alpha, fp32 out, dgrad": lambda: [ops.gemm(d["a"], d["wt"], M, ND, K, b_major=1, alpha=d["alpha"])],
        "bias + tanh, fp16 out": lambda: [ops.gemm(d["a"], d["w"], M, N, K, bias=d["bias"], act=1, out_half=True)],
        "bias + fp32 residual": lambda: [ops.gemm(d["a"], d["w"], M, N, K, bias=d["bias"], res=d["res"])],
        "bias + row-periodic table": lambda: [ops.gemm(d["a"], d["w"], M, N, K, bias=d["bias"], res=d["table"], res_row_mod=200)],
        "tanh' of fp16 t + column sums": lambda: list(ops.gemm(d["a"], d["wt"], M, ND, K, b_major=1, aux=d["t"], out_half=True,
                                                                want_colsum=True)),
        "split-K wgrad": lambda: [ops.gemm(d["dy"], d["x"], 576, 448, 320, a_major=1, b_major=1, splits=2)],
    }


def digests():
    out = {}
    for name, fn in cases().items():
        hs = hashlib.sha256()
        for t in fn():
            hs.update(t.contiguous().cpu().numpy().tobytes())
        out[name] = hs.hexdigest()
    torch.cuda.synchronize()
    return out


@pytest.mark.gpu
def test_epilogue_bits_match_previous_library():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    with open(GOLDEN) as fh:
        want = json.load(fh)
    got = digests()
    assert set(got) == set(want)
    bad = [k for k in want if got[k] != want[k]]
    assert not bad, f"epilogue forms whose bits changed: {bad}"


if __name__ == "__main__":
    print(json.dumps(digests(), indent=1))
