"""Every form of the mma.sync attention core (tf32 and 3xTF32, head sizes 32 to 128, unmasked and with the stage-2 mask,
fp32 and fp16 outputs) and the delta = rowsum(dO * O) kernel of its backward must give the same bits as the library they
replaced, which had separate kernels for head sizes 96 and 128.  The SHA-256 digests in
tests/golden/attention_mma_digests.json were written by this file run as a script
(`python tests/test_gpu_attention_mma_bits.py > tests/golden/attention_mma_digests.json`) with the library of commit
27d6a78 on an H100.  Each case digests every tensor the forward and backward return."""
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
GOLDEN = os.path.join(ROOT, "tests", "golden", "attention_mma_digests.json")
# B and heads give several CTAs along the grid's y and z axes; N = 300 gives several along x for every tile height
# (32, 64, 128 rows) and, like 77, is ragged against each of them
B, HEADS = 2, 3
NS = (1, 77, 300)


def _cond_lens(N):
    """cond_len 0 (plain causal), 1, a value inside a tile, and N (no mask at all)"""
    return sorted({0, 1, N // 2 + 3 if N > 2 else 1, N})


def _inputs(N, dh, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = torch.randn(B * N, 3 * HEADS * dh, device="cuda", generator=g)
    dout = torch.randn(B * N, HEADS * dh, device="cuda", generator=g)
    return qkv, dout


def cases():
    """name -> thunk returning the tensors whose bits are pinned"""
    out = {}
    seed = 100
    for dh in (32, 64):
        for N in NS:
            seed += 1
            qkv, dout = _inputs(N, dh, seed)
            scale = dh ** -0.5
            half_scale = torch.tensor([256.0], device="cuda")
            for out_half in (False, True):
                for form in ("round 0", "round 1", "fp16 dqkv"):
                    round_out = form == "round 1"
                    hs = half_scale if form == "fp16 dqkv" else None

                    def fn(qkv=qkv, dout=dout, N=N, dh=dh, scale=scale, out_half=out_half, round_out=round_out, hs=hs):
                        o, lse = ops.attention_fwd(qkv, B, N, HEADS, dh, scale, round_out, out_half=out_half)
                        return [o, lse, ops.attention_bwd(qkv, o, lse, dout, B, N, HEADS, dh, scale, round_out, half_scale=hs)]

                    out[f"tf32 dh {dh} N {N} {'fp16' if out_half else 'fp32'} O, {form}"] = fn

            def fn_exact(qkv=qkv, dout=dout, N=N, dh=dh, scale=scale):
                o, lse = ops.attention_exact_fwd(qkv, B, N, HEADS, dh, scale)
                return [o, lse, ops.attention_exact_bwd(qkv, o, lse, dout, B, N, HEADS, dh, scale)]

            out[f"3xtf32 dh {dh} N {N}"] = fn_exact
    for dh in (32, 64, 96, 128):
        for N in NS:
            seed += 1
            qkv, dout = _inputs(N, dh, seed)
            scale = dh ** -0.5
            for cond in _cond_lens(N):
                for exact in (False, True):
                    for round_out in (False, True):
                        def fn(qkv=qkv, dout=dout, N=N, dh=dh, scale=scale, cond=cond, exact=exact, round_out=round_out):
                            o, lse = ops.attention_causal_fwd(qkv, B, N, HEADS, dh, scale, cond, exact, round_out)
                            return [o, lse, ops.attention_causal_bwd(qkv, o, lse, dout, B, N, HEADS, dh, scale, cond, exact, round_out)]

                        out[f"causal dh {dh} N {N} cond {cond} exact {int(exact)} round {int(round_out)}"] = fn
    for N in NS:
        seed += 1
        g = torch.Generator(device="cuda").manual_seed(seed)
        qkv = torch.randn(B * N, 3 * HEADS * 64, device="cuda", generator=g).half()
        dout = (torch.randn(B * N, HEADS * 64, device="cuda", generator=g) * 64).half()

        def fn_f16(qkv=qkv, dout=dout, N=N):
            o, lse = ops.attention_f16_fwd(qkv, B, N, HEADS, 64, 0.125)
            return [o, lse, ops.attention_f16_bwd(qkv, o, lse, dout, B, N, HEADS, 64, 0.125)]

        out[f"fp16 dh 64 N {N}"] = fn_f16
    return out


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
def test_attention_bits_match_previous_library():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    with open(GOLDEN) as fh:
        want = json.load(fh)
    got = digests()
    assert set(got) == set(want)
    bad = [k for k in want if got[k] != want[k]]
    assert not bad, f"attention forms whose bits changed: {bad}"


if __name__ == "__main__":
    print(json.dumps(digests(), indent=1))
